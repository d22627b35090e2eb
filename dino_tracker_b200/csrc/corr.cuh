// Internal interface of corr.cu / head.cu (not part of the C ABI).
#pragma once
#include "common.cuh"

namespace dtk {

constexpr int STREAM_MAX_M = 8;  // groups with at most this many descriptors use the streaming kernel

struct FeatView {
  const float* tpc; const float* norms; const void* hi; const void* lo;
  int T, C, P;
  const void* q8; const float* q_fac; const float* q_rho;   // int8 coarse operands (optional, dinotrk_features)
  const void* hilo;   // [T][P][ceil(C / 32)][64] hi / lo interleaved per 32 channels (optional, with hi / lo)
  bool tensor() const { return hi != nullptr && lo != nullptr; }
  bool s8() const { return q8 != nullptr && q_fac != nullptr && q_rho != nullptr; }
};
static inline FeatView make_view(const dinotrk_features& f, const dinotrk_geom& g) {
  return FeatView{f.tpc, f.norms, f.hi, f.lo, f.T, f.C, g.h * g.w, f.q8, f.q_fac, f.q_rho, f.hi && f.lo ? f.hilo : nullptr};
}
// fp16 elements per row of the interleaved split: 64 per 32-channel block (the last one zero-padded)
__host__ __device__ inline int hilo_row(int C) { return 64 * ((C + 31) / 32); }
// The full-map GEMM runs on the interleaved split (TcMode::F16X3I) when the features carry it and C % 32 == 0 (the
// descriptors' interleaved rows then fill exactly the workspace of their separate halves).
static inline bool corr_hilo(const FeatView& fv) { return fv.hilo != nullptr && fv.C % 32 == 0; }

// Value of a correlation map entry from its accumulator: acc / max(|d| |F|, clamp), the reference's cosine with its 1e-8
// clamp (callers apply the ReLU).  Every kernel that forms such a value uses this, so that the exact-window head's values
// are bit for bit the full-map GEMM's.
__device__ __forceinline__ float corr_cos(float acc, float dn, float fn, float clamp = 1e-8f) {
  return __fdiv_rn(acc, fmaxf(__fmul_rn(dn, fn), clamp));
}

constexpr int CORR_TILE = 256;   // token tile of the tensor-core correlation GEMM (= TC_BN); unit of the tile maxima

// Optional by-products / shortcuts of one launch_corr_maps call (all members may stay zero):
//   tkeys       [total_maps][cdiv(P, CORR_TILE)]: per map and 256-token tile, (bits of the tile maximum) << 32 |
//               (0x7fffffff - first token holding it), written by the GEMM epilogue: the maximum over a map's keys is its
//               first arg-max.  Maps of thin groups (streaming kernel) get ~0 in tile 0 = "no keys".  Only produced on
//               the tensor path (fv.tensor()).
//   zero_word   an int the plan kernel sets to 0 (the head's counter of uncertified maps: saves a launch)
//   split_ready the fp16 hi/lo copies of `desc` are already in split_ws (written by the sampler): skip the split kernel.
//               With corr_hilo(fv) they must be interleaved ([rows][2 C], dinotrk_split_hilo's layout), else hi rows then
//               lo rows at the next 256-byte boundary
//   no_thin     the caller knows that no group has <= STREAM_MAX_M descriptors: skip the streaming kernel launch
struct CorrAssist {
  unsigned long long* tkeys = nullptr;
  int* zero_word = nullptr;
  bool split_ready = false;
  bool no_thin = false;
  bool all_wide = false;   // no streaming kernel: groups of any size > 0 are GEMM tiles
  bool small_tiles = false;   // tensor path: 128-row single-CTA tiles instead of 256-row CTA-pair tiles (many tiny groups)
};

size_t corr_tc_workspace_bytes(int total_rows, int C);
// The separate-halves split of `rows` descriptor rows of C channels in a split workspace (corr_tc_workspace_bytes): hi rows,
// then lo rows at the next 256-byte boundary.
struct DescSplit {
  char* hi; char* lo;
  DescSplit(void* ws, size_t rows, int C) : hi(static_cast<char*>(ws)), lo(hi + align_up(rows * C * 2, 256)) {}
};
// workspace of launch_corr_maps: the GEMM tile plan of n_groups groups and the split of `rows` descriptor rows
struct CorrMapsWs {
  int* plan; float* split;
  CorrMapsWs(Arena& ar, int rows, int n_groups, int C)
      : plan(ar.take<int>(n_groups + 1)), split(ar.take<float>(corr_tc_workspace_bytes(rows, C) / 4)) {}
};
// desc_rows = number of rows of the desc array (bounds of its tensor map); split_ws: corr_tc_workspace_bytes
// (only touched when fv.tensor()).
int launch_corr_maps(const FeatView& fv, const float* desc, int desc_rows, const float* desc_norm,
                     const int* grp_frame, const int* grp_row0, const int* grp_m, const int* grp_map0, int n_groups,
                     int total_maps, int max_group_m, float* maps, int map_stride, int* tile_start, float* split_ws,
                     cudaStream_t st, const CorrAssist& assist = CorrAssist());
int launch_corr_gemm_tc(const void* tpc_hi, const void* tpc_lo, const float* norms, int T, int C, int P,
                        const float* desc, int desc_rows, const float* desc_norm, const int* grp_frame,
                        const int* grp_row0, const int* grp_m, const int* grp_map0, const int* tile_start, int n_groups,
                        int max_tiles, float* maps, int map_stride, float* desc_split_ws, cudaStream_t st,
                        unsigned long long* tkeys, bool split_ready,
                        int tile_rows /* TC2_BM: CTA-pair (two-CTA cluster) kernel; TC_BM: single-CTA kernel */,
                        bool relu = true /* false: signed cosines (no tile keys) */,
                        const float* clamp = nullptr /* [desc_rows]: per-row replacement of the norm product's 1e-8 (signed only) */,
                        const void* tpc_hilo = nullptr /* interleaved features (corr_hilo): the F16X3I GEMM; a ready split in
                                                          desc_split_ws is then interleaved too */);
int launch_split_f16(const float* x, void* hi, void* lo, size_t n, cudaStream_t st);
int launch_split_hilo(const float* x, void* hilo, size_t rows, int C, cudaStream_t st);

// Faithful range of the fp16 hi/lo split (DESIGN.md 3.1).  Per element, x - hi - lo is at most 2^-22 |x| while lo is an fp16
// normal and at most 2^-25 (half the smallest subnormal step) otherwise, so the split contraction's cosine error is
//   <= 2^-21 + 2^-25 sqrt(C) (1 / |d| + 1 / |F|).
// Norms >= 2^-3 sqrt(C) keep the absolute part <= 2^-22 per operand.  Elements above the largest fp16 (65504) make hi = inf.
// A video is in range when every |x| <= SPLIT_MAX_ABS and every token norm is 0 (an exact zero splits exactly) or
// >= split_min_norm(C).
constexpr float SPLIT_MAX_ABS = 65504.f;
__host__ __device__ inline float split_min_norm(int C) { return 0.125f * sqrtf((float)C); }

int launch_head(const float* maps, int n_maps, int map_stride, const dinotrk_geom& g,
                const dinotrk_head_weights& hw, const int* out_index, float* out, int out_stride, int out_mode,
                int* aux, int* scratch /* n_maps + 1 ints, or NULL: full-map kernel for every map */, cudaStream_t st,
                const unsigned long long* tkeys = nullptr /* tile keys of launch_corr_maps */, bool counter_zeroed = false,
                int parts = 3 /* bit 0: fast path over all maps, bit 1: full-map kernel over the uncertified ones */);

}  // namespace dtk

// Coarse pass + exact window: the anchor phase's correlation + head without ever writing a correlation map.
// Internal interface of xwin.cu (not part of the C ABI).
//
//   models/tracker.py:158-180 + models/networks/tracker_head.py:68-121 produce, per (descriptor, frame) map, ONE point:
//   the disc-masked soft-argmax around the map's arg-max.  That point depends on (i) which token is the arg-max,
//   (ii) the map values on the 15 x 15 window around it (11 x 11 logits <- 13 x 13 hidden <- 15 x 15 inputs) and (iii) an
//   upper bound on everything else (certificate that the stability branch, tracker_head.py:87-94, stays off).
//
//   1. coarse GEMM   one wgmma pass, int8 (per-token scales, the default) or fp16 over the `hi` halves; the epilogue keeps
//                    per map and 128-token tile only (largest value, its first token, second largest value).  |coarse -
//                    exact| <= eps for every token: XW_EPS for fp16 (rounding of both operands + fp32 accumulation), the
//                    per-map xw_eps_s8 for int8 (relative quantisation residuals of the map's two operands, see DESIGN.md).
//   2. plan          per map: the tokens that can be the exact arg-max (coarse >= max - 2 eps); a map whose candidates
//                    are not all tile maxima is "ambiguous".  Maps come in CELLS = the <= 128 source frames of one (query,
//                    anchor frame) pair: their arg-maxes cluster around the query's position in the anchor frame, so one
//                    21 x 21 token box around the cell's median arg-max holds every map's window.
//   3. exact GEMM    per cell, the fp32-faithful split-precision contraction (lo*hi + hi*lo + hi*hi, same operation
//                    sequence as the full-map GEMM) of the cell's descriptors against the tokens of its tight extent
//                    only: the union of its fitting maps' candidate windows, 225 to 441 of the box's tokens (2.8 to 5.4 %
//                    of the map).  Raw accumulators go to a [map][448] buffer laid out as the whole box (1.8 KB per map
//                    instead of 32 KB); the head reads nothing outside the extent.
//   4. head          one kernel, two maps per warp (a half-warp each, lane = refiner channel): exact arg-max among the
//                    candidates, the exact 15 x 15 window built in shared memory and m_out; the refiner one hidden row at a
//                    time, kept in registers; softmax sums on the 11 x 11 box, certificate with the bound from (1); writes
//                    the track point.  The next pair's window loads land while a pair is refined.
//   Maps that are ambiguous, do not fit their cell's box or fail the certificate are queued and re-done by the full-map
//   path (split-precision GEMM over all tokens + head kernels of head.cu) -- results never depend on the coarse values.
#pragma once
#include <type_traits>

#include "common.cuh"
#include "corr.cuh"

namespace dtk {

constexpr float XW_EPS = 1.1e-3f;     // bound on |coarse - exact| in cosine units (2^-10 + accumulation, rounded up)
constexpr int XW_BOX = 21;            // box side (tokens); windows of maps whose arg-max lies within +-3 of the centre fit
constexpr int XW_SLACK = 3;
constexpr int XW_COLS = 448;                                     // accumulator row pitch per map (441 box tokens, row-major)
constexpr int XW_MAX_CELL = 128;      // maps (source frames) per cell = wgmma M rows (64 or 128)
constexpr int XW_MAX_CAND = 4;
constexpr float XW_MIN_NORM = 1e-4f;  // guard of the coarse epilogue's reciprocal norms only.  XW_EPS holds when both norms are
                                      // >= split_min_norm(C) (corr.cuh): a smaller descriptor norm makes the map ambiguous, a
                                      // smaller token norm anywhere in the video sends the whole call to the full-map pipeline
constexpr int XW_TILE = 128;          // tokens per coarse key (half of the coarse GEMM's N tile: two keys per tile)

// ---- int8 coarse operands.  Per row x (token or descriptor): s = max|x_k| / 127, q = rint(x / s) in [-127, 127],
// fac = s / max(|x|, XW_MIN_NORM) (the coarse epilogue's factor), rho = |x - s q| / |x| rounded up (0 for x = 0).
// The coarse value of a map is <q_d, q_x> fac_d fac_x (int32 accumulation: exact while C 127^2 < 2^31; its conversion to
// float, cvt.rn.f32.s32, is exact while C 127^2 < 2^24, i.e. C <= 1040, and above that rounds by <= 2^-24 |<q_d, q_x>|).
// |<d, x> - <s_d q_d, s_x q_x>| <= |<d - d^, x>| + |<d^, x - x^>| <= (rho_d + (1 + rho_d) rho_x) |d| |x|, so in cosine
// units |coarse - exact| <= xw_eps_s8(rho_d, rho_F, xw_s8_slack(C)) with rho_F the largest rho_x of the map's frame.
// The slack covers the exact split path's own error -- 2^-21 from the operand split plus one truncating accumulator add
// (<= 2^-23 of the running magnitude) per wgmma, three wgmma (lo hi, hi lo, hi hi) per 16 channels: 3 ceil(C / 16) adds,
// DESIGN.md 3.1 -- the epilogue's four fp32 roundings and, above C = 1040, the accumulator's conversion:
// |<q_d, q_x>| s_d s_x <= |d^| |x^| <= (1 + rho_d)(1 + rho_x) |d| |x|, so <= 2^-24 (1 + rho_d)(1 + rho_F) in cosine units,
// with rho <= sqrt(C) / 254 (each residual is <= s / 2 and |x| >= 127 s).
//   C <= 1040: 2^-21 + 195 x 2^-23 + 4 x 2^-24 x 1.27 = 2.4e-5 <= XW_S8_SLACK = 2^-15 = 3.05e-5.
//   C > 1040:  XW_S8_SLACK + 3 ceil(C / 16) 2^-23: the adds explicitly, and 2^-15 for the rest (2^-21 + 5 x 2^-24 x 1.39
//              = 8.9e-7 at C = 2048).
constexpr float XW_S8_SLACK = 3.0518e-5f;   // 2^-15
constexpr int XW_S8_EXACT_C = 1040;         // C 127^2 < 2^24: the conversion is exact and XW_S8_SLACK alone suffices
// the widest feature the ViT stage writes (dinotrk_vit_forward: dim <= 2048; ViT-g/14: 1536)
constexpr int XW_S8_MAX_C = 2048;
// slack of xw_eps_s8 for C channels (see above), rounded up to float; exactly XW_S8_SLACK for C <= XW_S8_EXACT_C
inline float xw_s8_slack(int C) {
  if (C <= XW_S8_EXACT_C) return XW_S8_SLACK;
  const double s = (double)XW_S8_SLACK + 3.0 * (double)((C + 15) / 16) * 0x1p-23;
  const float f = (float)s;
  return (double)f < s ? nextafterf(f, INFINITY) : f;
}
// rho_F above which the automatic mode runs the fp16 coarse pass: eps ~ 2 rho_F, and 2 eps is the candidate margin.  At
// 0.03 (twice the largest token residual of Gaussian-like features at C = 1024, 0.0132) the margin stays below ~0.13,
// under the typical gap between a map's maximum and the next value of another tile; features with outlier channels
// (max |x| / rms far above Gaussian) exceed it and keep the fp16 pass.
constexpr float XW_S8_RHO_MAX = 0.03f;
__device__ __forceinline__ float xw_eps_s8(float rho_d, float rho_f, float slack) {
  return __fadd_ru(__fadd_ru(rho_d, __fmul_ru(__fadd_ru(1.f, rho_d), rho_f)), slack);
}

// One warp quantises row x (element k = ld(k), C % 4 == 0) with fp32 norm `norm` (the exact path's): writes q[C], *fac
// and returns rho (every lane).
template <class Load>
__device__ __forceinline__ float xw_quant_row(const Load& ld, int C, float norm, int8_t* __restrict__ q, float* __restrict__ fac) {
  const int lane = threadIdx.x & 31;
  float mx = 0.f;
  for (int k = 4 * lane; k < C; k += 128) {
    const float4 v = ld(k);
    mx = fmaxf(mx, fmaxf(fmaxf(fabsf(v.x), fabsf(v.y)), fmaxf(fabsf(v.z), fabsf(v.w))));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
  const float s = __fdiv_rn(mx, 127.f);
  double r2 = 0.0, x2 = 0.0;
  for (int k = 4 * lane; k < C; k += 128) {
    const float4 v = ld(k);
    const float vv[4] = {v.x, v.y, v.z, v.w};
    char4 o;
    signed char* oc = reinterpret_cast<signed char*>(&o);
#pragma unroll
    for (int e = 0; e < 4; ++e) {
      const float qf = s > 0.f ? fminf(fmaxf(rintf(__fdiv_rn(vv[e], s)), -127.f), 127.f) : 0.f;
      oc[e] = (signed char)qf;
      const double d = (double)vv[e] - (double)s * (double)qf;   // exact: s q has <= 32 significant bits
      r2 = fma(d, d, r2);
      x2 = fma((double)vv[e], (double)vv[e], x2);
    }
    *reinterpret_cast<char4*>(q + k) = o;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    r2 += __shfl_xor_sync(0xffffffffu, r2, o);
    x2 += __shfl_xor_sync(0xffffffffu, x2, o);
  }
  if (lane == 0) *fac = __fdiv_rn(s, fmaxf(norm, XW_MIN_NORM));
  // upward at every step (the double sums' own rounding, ~C 2^-53 relative, is far below the last float ulp)
  return x2 > 0.0 ? __double2float_ru(__ddiv_ru(__dsqrt_ru(r2), __dsqrt_rd(x2))) : 0.f;
}

// column of box token (by, bx) in a map's accumulator row
__host__ __device__ inline int xw_col(int by, int bx) { return by * XW_BOX + bx; }

struct XwChunk {          // device buffers of one chunk in flight (all sized for chunk_maps maps)
  unsigned long long* key1;   // [maps][n_tiles]  coarse maximum of a XW_TILE-token tile << 32 | (0x7fffffff - first token)
  float* max2;                // [maps][n_tiles]  second largest coarse value of the tile
  int* cand;                  // [maps][XW_MAX_CAND] candidate tokens (-1 = none)
  int* pinfo;                 // [maps] coarse arg-max token, or -1 - token for an ambiguous map (plan scratch)
  int* stat;                  // [maps] 0: exact-window path, 1: full-map path
  int* cell_of;               // [maps] cell index
  int2* box_org;              // [cells] (first box row, first box column); y = INT_MIN: skip the cell
  int4* box_ext;              // [cells] tight extent {first row, first column, rows, columns} relative to box_org: the union
                              // of the fitting maps' candidate windows, rows and columns in [15, 21] (set when box_org is)
  float* xbox;                // [maps][XW_COLS] raw split-precision accumulators of the box tokens
  int* slow_cnt;              // [n_groups + 4] per group count of queued maps; [n_groups] = total, [n_groups + 1] = of
                              // those queued by the certificate, [n_groups + 2] = extent tokens, [n_groups + 3] = cells
  int* slow_list;             // [maps] group g's queue lives at [grp_map0[g], grp_map0[g] + slow_cnt[g])
  XwChunk() = default;
  // every buffer of a chunk of `maps` maps, `cells` cells and n_groups groups, n_tiles coarse tiles per map
  XwChunk(Arena& ar, size_t maps, size_t cells, int n_tiles, int n_groups) {
    key1 = ar.take<unsigned long long>(maps * n_tiles);
    max2 = ar.take<float>(maps * n_tiles);
    cand = ar.take<int>(maps * XW_MAX_CAND);
    stat = ar.take<int>(maps);
    pinfo = ar.take<int>(maps);
    cell_of = ar.take<int>(maps);
    slow_list = ar.take<int>(maps);
    box_org = ar.take<int2>(cells);
    box_ext = ar.take<int4>(cells);
    xbox = ar.take<float>(maps * XW_COLS);
    slow_cnt = ar.take<int>((size_t)n_groups + 4);
  }
};

struct XwCells {          // host-planned, device-resident description of a chunk's cells
  const int* row0;     // [cells] first map of the cell (chunk-local: indexes the per-map arrays)
  const int* arow;     // [cells] first descriptor row of the cell in the GEMM's A arrays (consecutive rows, like its maps)
  const int* m;        // [cells] rows
  const int* frame;    // [cells] anchor frame
  const int* group;    // [cells] group index (for the slow queues)
  int n_cells, max_m;
};

// Coarse GEMM over the chunk's groups (tile_start: prefix of ceil(m / 256) per group, all groups wide): the int8 pass when
// desc_q8 is given (desc_fac = the rows' factors, fv's int8 features), else fp16 over desc_hi and fv.hi.
int launch_xw_coarse(const FeatView& fv, const void* desc_hi, int desc_rows, const float* desc_norm, const int* grp_frame,
                     const int* grp_row0, const int* grp_m, const int* grp_map0, const int* tile_start, int n_groups,
                     int max_tiles, const XwChunk& xc, cudaStream_t st, const float* rnorms, const void* desc_q8 = nullptr,
                     const float* desc_fac = nullptr);
// rnorms = 1 / |F| for the coarse epilogue; *min_bits = bit pattern of the smallest token norm of the video
int launch_xw_rnorms(const FeatView& fv, float* rnorms, unsigned* min_bits, cudaStream_t st);
// eps: per-map bound on |coarse - exact| of the int8 pass (xw_eps_s8), nullptr for the fp16 pass (XW_EPS)
int launch_xw_plan(const XwCells& cells, const float* desc_norm, int n_groups, const dinotrk_geom& g, const XwChunk& xc,
                   cudaStream_t st, int n_maps, float min_norm, const float* eps);
// box tokens from fv.hilo (128-byte rows) when given, else from fv.hi / fv.lo (64-byte rows)
int launch_xw_gemm(const FeatView& fv, const dinotrk_geom& g, const void* desc_hi, const void* desc_lo, int desc_rows,
                   const XwCells& cells, const XwChunk& xc, cudaStream_t st);
int launch_xw_head(const FeatView& fv, const dinotrk_geom& g, const dinotrk_head_weights& hw, const XwCells& cells,
                   const float* desc_norm, const int* grp_map0, int n_maps, const int* out_index, float* out, int out_stride,
                   int out_mode, const XwChunk& xc, cudaStream_t st, int n_groups, const float* eps);
// Appends the queued maps' descriptor rows (fp32 optional, hi, lo, norm, out_index) to compact arrays at row_base and their
// group arrays ([frame | row0 | m | map0] x gcap, entries grp_base ..) to cgrp.  n_slow = host copy of slow_cnt[n_groups].
// arow[map] = the map's row in desc / desc_hi / desc_lo (nullptr: the map index); norm and out_index are per map.
// hilo: the fp16 rows go to c_hi interleaved per 32 channels (the full-map GEMM's F16X3I operand; c_lo unused).
int launch_xw_compact(const float* desc, const void* desc_hi, const void* desc_lo, const int* arow, const float* desc_norm,
                      const int* out_index, int C, const int* grp_frame, const int* grp_map0, int n_groups, int n_slow,
                      const XwChunk& xc, float* c_desc, void* c_hi, void* c_lo, float* c_norm, int* c_out_index, int* cgrp,
                      int gcap, cudaStream_t st, int row_base = 0, int grp_base = 0, bool hilo = false);

}  // namespace dtk

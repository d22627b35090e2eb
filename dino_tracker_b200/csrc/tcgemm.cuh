// Persistent, warp-specialised wgmma GEMM for sm_90a:   D[m][n] = sum_k A[m][k] * B[n][k]
// (both operands K-major: A = [rows][K], B = [batch][N][K]), 128 x BN output tiles, operands staged by TMA into
// 128B-swizzled shared memory through an mbarrier ring, accumulators in registers.
//
//   warpgroup 0     : TMA producer (one elected lane; its registers are handed to the consumers)
//   warpgroups 1, 2 : wgmma on 64 rows each (m64nBN), then the epilogue of those rows: 32-column blocks of the
//                     accumulator go through shared memory so that the Epi functor sees one row per thread (or, for
//                     coalesced epilogues, 4 consecutive columns per thread with lanes running along the rows); fragment
//                     epilogues take the accumulator registers directly
// The producer runs ahead into the next tile while the consumers are in the epilogue.
//
// Pair variant (tc_gemm_pair_kernel, a cluster of two CTAs): the two CTAs compute the two 128-row halves of a 256 x BN
// tile; each loads half of the B tile and multicasts it to both, which halves the B operand traffic from L2 per CTA.
//
// Modes:
//   F16X3  : fp32-faithful split-precision: operands pre-split into fp16 hi + fp16 lo (x = hi + lo up to 2^-22),
//            lo*hi + hi*lo + hi*hi on the f16 tensor pipe (twice the TF32 rate), fp32 accumulation
//   F16X3I : F16X3 on operands whose hi and lo are interleaved per 32 channels ([rows][ceil(K / 32)][64] fp16, one
//            128-byte row = [hi 32 | lo 32], dinotrk_split_hilo): K blocks of 32 channels, one TMA per operand and stage,
//            hi read at 0 / 32 bytes into the row and lo at 64 / 96.  The same wgmma sequence as F16X3 (bit-identical
//            results) on half the bytes per stage, so twice the stages fit.  The "hi" operands carry the interleaved arrays
//   TF32X3 : the same scheme with TF32 parts (fp32 storage)
//   TF32   : single pass on fp32 data (the tensor core reads the top 19 bits)
//   BF16   : single pass on bf16 data
//   F16    : single pass on fp16 data (11-bit significand like TF32, twice its rate)
//   S8     : single pass on signed 8-bit data (twice the F16 rate), exact int32 accumulators; BN = 256 and fragment
//            epilogues only (they receive the int32 accumulators)
// Work = grouped tiles: group g covers A rows [row0[g], row0[g] + m[g]) against B batch item batch[g];
// m-tiles are numbered through the prefix array tile_start[] (device), n-tiles cover N.
#pragma once
#include <cuda_fp16.h>

#include <type_traits>

#include "common.cuh"
#include "tc05.cuh"

namespace dtk {

enum class TcMode { TF32X3 = 0, TF32 = 1, BF16 = 2, F16X3 = 3, F16 = 4, S8 = 5, F16X3I = 6 };

constexpr int TC_BM = 128, TC_BN = 256;   // TC_BN: default N tile (template parameter BN overrides it)
constexpr int TC2_BM = 256;               // M tile of a CTA pair
constexpr int TC_THREADS = 384;
constexpr int TC_EPI_PITCH = 36;          // floats per row of a consumer warpgroup's 64 x 32 epilogue block
constexpr int TC_SMEM_MAX = 227 * 1024;

template <TcMode MODE, int BN = TC_BN>
struct TcCfg {
  static_assert(BN == 64 || BN == 128 || BN == 256, "N tile must be 64, 128 or 256");
  static constexpr bool kIL = MODE == TcMode::F16X3I;             // hi / lo interleaved in each 128-byte row
  static constexpr int kElem = MODE == TcMode::S8 ? 1 : (MODE == TcMode::BF16 || MODE == TcMode::F16X3 || MODE == TcMode::F16 || kIL) ? 2 : 4;
  static constexpr int kRowElems = 128 / kElem;                   // elements per 128-byte swizzle row
  static constexpr int kBK = kIL ? kRowElems / 2 : kRowElems;     // K (channels) per K block
  static constexpr int kOps = (MODE == TcMode::TF32X3 || MODE == TcMode::F16X3) ? 2 : 1;   // hi (+ lo) tiles per operand
  static constexpr int kMmaK = 32 / kElem;                        // K per wgmma
  static constexpr int kABytes = TC_BM * 128, kBBytes = BN * 128;
  static constexpr int kStageBytes = kOps * (kABytes + kBBytes);
  static constexpr int kEpiBytes = 2 * 64 * TC_EPI_PITCH * 4;
  static constexpr int kFixed = kEpiBytes + 1024 /*align slack*/ + 256 /*barriers*/;
  static constexpr int kStages = (TC_SMEM_MAX - kFixed) / kStageBytes > 6 ? 6 : (TC_SMEM_MAX - kFixed) / kStageBytes;
  static_assert(kStages >= 2, "shared memory ring too shallow");
  static constexpr int kSmem = kStages * kStageBytes + kFixed;
  static constexpr bool kTF32 = (MODE == TcMode::TF32X3 || MODE == TcMode::TF32);
  static constexpr bool kS8 = MODE == TcMode::S8;
  using Acc = std::conditional_t<kS8, int, float>;                // accumulator element
  static_assert(!kS8 || BN == 256, "8-bit mode: m64n256k32 only");
};

// ---- scaled hi / lo split of gradient operands (delta_train.cu, contrastive.cu) ----
// power of two that puts max |g| in [2^13, 2^14) (1 for an all-zero tensor); exponents clamped to keep 2^e finite
__device__ __forceinline__ int grad_exp(unsigned amax_bits) {
  const float m = __uint_as_float(amax_bits);
  if (!(m > 0.f)) return 0;
  int e;
  frexpf(m, &e);
  e = 14 - e;
  return e > 126 ? 126 : (e < -126 ? -126 : e);
}

__device__ __forceinline__ void split16(float v, __half& h, __half& l) {
  h = __float2half_rn(v);
  l = __float2half_rn(v - __half2float(h));
}

// Epilogues that declare `static constexpr bool kCoalesced = true` are called as vec4(g, row, col, float4) with lanes
// running along a row; they also provide `bool direct(int col0)` to keep the thread-per-row call for selected column ranges.
template <class E, class = void> struct EpiCoalesced { static constexpr bool value = false; };
template <class E> struct EpiCoalesced<E, std::enable_if_t<E::kCoalesced>> { static constexpr bool value = true; };

// Read-modify-write epilogues (`static constexpr bool kPrefetch = true`) additionally provide
// `float4 fetch(g, row, col)` and `vec4(g, row, col, acc, fetched)`: the coalesced loop then issues a thread's reads of a
// block before its first write (through one pointer the compiler must otherwise keep every load behind the previous store).
template <class E, class = void> struct EpiPrefetch { static constexpr bool value = false; };
template <class E> struct EpiPrefetch<E, std::enable_if_t<E::kPrefetch>> { static constexpr bool value = true; };

// One output tile as the producer decoded it: group g, first row m0 inside the group and first column n0 of the tile, and
// the group's B batch item, first A row and row count (rows >= m are padding)
struct TcTile { int g, m0, n0, batch, row0, m; };

// Fragment epilogues (`static constexpr bool kFragment = true`) skip the shared-memory round trip.  The producer writes
// each tile's TcTile into shared memory next to the tile's first K block, so the consumers neither decode the tile nor
// read the group tables.  Once that K block has landed (before the tile's first wgmma) consumer thread t of each
// warpgroup calls
//   Pre begin(tile, t, r)
// (r: the thread's first accumulator row, below): it issues the tile's global reads, which are then in flight during the
// K loop.  Pre has a member `float2 col`, the tile's per-column values for columns n0 + t (.x) and n0 + t + 128 (.y); the
// body stages them in cols[c] (shared memory, c < BN = 256) so that the epilogue reads them with constant offsets.  Right
// after the tile's last wgmma has completed, every consumer thread calls
//   fragment(tile, r, fc, acc, cols, pre)
// with its own accumulator registers (float, or int in S8 mode; the epilogue may overwrite them): acc[4 i + {0, 1}] are
// row r, acc[4 i + {2, 3}] row r + 8 (rows inside the group), columns n0 + 8 i + fc + {0, 1}.  The 4 lanes of a quad
// (lane & 3) hold the same two rows.
template <class E, class = void> struct EpiFragment { static constexpr bool value = false; };
template <class E> struct EpiFragment<E, std::enable_if_t<E::kFragment>> { static constexpr bool value = true; };
template <class E, class = void> struct PreOf { struct type {}; };
template <class E> struct PreOf<E, std::enable_if_t<EpiFragment<E>::value>> { using type = typename E::Pre; };

struct TcProblem {
  const int* grp_batch;    // [n_groups] B batch item (frame) of each group
  const int* grp_row0;     // [n_groups] first A row
  const int* grp_m;        // [n_groups] number of A rows
  const int* tile_start;   // [n_groups + 1] prefix of ceil(m / M tile)  (M tile: TC_BM, or TC2_BM for the pair kernel)
  int n_groups;
  int N, K;                // B rows per batch item, reduction length
};

// Epi must provide a per-thread `State` plus
//   tile_begin(State&)                                                      once per (row, tile)
//   operator()(State&, int g, int r_in_group, int col0, const float (&v)[32], int ncols_valid)
//                                                                           per 32 consecutive columns, in column order
//   tile_end(State&, int g, int r_in_group, int n_tile)                     once per (row, tile)
template <TcMode MODE, class Epi, int BN, bool PAIR>
__device__ __forceinline__ void tc_gemm_body(const CUtensorMap& tmA_hi, const CUtensorMap& tmA_lo, const CUtensorMap& tmB_hi,
                                             const CUtensorMap& tmB_lo, const TcProblem& pb, const Epi& epi) {
  using Cfg = TcCfg<MODE, BN>;
  static_assert(!Cfg::kS8 || EpiFragment<Epi>::value, "8-bit mode: fragment epilogues only");
  constexpr int TM = PAIR ? TC2_BM : TC_BM;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);   // [kStages]
  uint64_t* empty = full + Cfg::kStages;                                                    // [kStages]
  float* epi_scratch = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes + 256);
  static_assert(2 * Cfg::kStages * 8 <= 256, "barrier block");

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const uint32_t rank = PAIR ? tc::cluster_ctarank() : 0u;
  const int unit = PAIR ? (int)(blockIdx.x >> 1) : (int)blockIdx.x, n_units = PAIR ? (int)(gridDim.x >> 1) : (int)gridDim.x;
  const int n_tiles_n = (pb.N + BN - 1) / BN;
  const int total_tiles = pb.tile_start[pb.n_groups] * n_tiles_n;
  const int KB = (pb.K + Cfg::kBK - 1) / Cfg::kBK;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&tmA_hi); tc::prefetch_tmap(&tmB_hi);
    if (Cfg::kOps == 2) { tc::prefetch_tmap(&tmA_lo); tc::prefetch_tmap(&tmB_lo); }
    // empty: one arrival per consumer warpgroup of every CTA whose B half lands in this CTA's slot
    for (int s = 0; s < Cfg::kStages; ++s) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], PAIR ? 4 : 2); }
    tc::mbar_fence_init();
  }
  if (PAIR) tc::cluster_sync_all(); else __syncthreads();

  // tile id -> (group, m0, n0): m-tile index is the slow dimension so that CTAs that run together share
  // the same B rows (frame) in L2
  auto decode = [&](int tile, int& g, int& m0, int& n0) {
    int mt = tile / n_tiles_n;
    n0 = (tile - mt * n_tiles_n) * BN;
    g = last_le(pb.n_groups, mt, pb.tile_start);
    m0 = (mt - pb.tile_start[g]) * TM + (int)rank * TC_BM;
  };
  // fragment epilogues: the record of the tile whose first K block is in ring slot s (written by the producer before it
  // arms full[s], read by the consumers before they release the slot)
  TcTile* recs = reinterpret_cast<TcTile*>(epi_scratch + 4 * BN);
  static_assert(!EpiFragment<Epi>::value || 4 * BN * 4 + Cfg::kStages * (int)sizeof(TcTile) <= Cfg::kEpiBytes,
                "fragment epilogue: column buffers and tile records");

  if (wg == 0) {
    // ===================== TMA producer =====================
    tc::regs_dealloc<40>();
    if (warp == 0 && tc::elect_one()) {
      int stage = 0, phase = 0;
      for (int tile = unit; tile < total_tiles; tile += n_units) {
        int g, m0, n0;
        decode(tile, g, m0, n0);
        const int row0 = pb.grp_row0[g], arow = row0 + m0, batch = pb.grp_batch[g];
        for (int kb = 0; kb < KB; ++kb) {
          tc::mbar_wait(&empty[stage], phase ^ 1);
          if constexpr (EpiFragment<Epi>::value)   // (the arrive below releases this store to the consumers)
            if (kb == 0) recs[stage] = TcTile{g, m0, n0, batch, row0, pb.grp_m[g]};
          uint8_t* st = smem + stage * Cfg::kStageBytes;
          tc::mbar_expect_tx(&full[stage], Cfg::kStageBytes);
          const int k0 = kb * Cfg::kRowElems;   // (interleaved: 32 channels = one whole row)
          tc::tma_load_2d(&tmA_hi, &full[stage], st, k0, arow);
          if (Cfg::kOps == 2) tc::tma_load_2d(&tmA_lo, &full[stage], st + Cfg::kABytes, k0, arow);
          uint8_t* sb = st + Cfg::kOps * Cfg::kABytes;
          if constexpr (PAIR) {   // this CTA's half of the B rows, into both CTAs
            const int off = (int)rank * (BN / 2);
            tc::tma_load_3d_mc(&tmB_hi, &full[stage], sb + off * 128, k0, n0 + off, batch, 3);
            if (Cfg::kOps == 2) tc::tma_load_3d_mc(&tmB_lo, &full[stage], sb + Cfg::kBBytes + off * 128, k0, n0 + off, batch, 3);
          } else {
            tc::tma_load_3d(&tmB_hi, &full[stage], sb, k0, n0, batch);
            if (Cfg::kOps == 2) tc::tma_load_3d(&tmB_lo, &full[stage], sb + Cfg::kBBytes, k0, n0, batch);
          }
          if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue: warpgroup cw owns rows [64 cw, 64 cw + 64) of the tile =====================
    tc::regs_alloc<232>();
    const int cw = wg - 1;
    float* sw = epi_scratch + cw * 64 * TC_EPI_PITCH;
    const int fr = (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);   // accumulator fragment: rows fr, fr + 8
    auto release = [&](int s) {
      if (t == 0) {
        if constexpr (PAIR) { tc::mbar_arrive_cluster(&empty[s], 0); tc::mbar_arrive_cluster(&empty[s], 1); }
        else tc::mbar_arrive(&empty[s]);
      }
    };
    int stage = 0, phase = 0;
    typename Cfg::Acc acc[BN / 2];
    if constexpr (EpiFragment<Epi>::value) {
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) acc[i] = 0;
    }
    // fragment epilogues: the warpgroup's per-column values of the tile in one of two buffers, used by alternate tiles (a
    // thread rewrites a buffer only after the next tile's barrier, which every thread passes after its epilogue's reads)
    int cbuf = 0;
    static_assert(!EpiFragment<Epi>::value || (BN == 256 && 4 * BN * 4 <= Cfg::kEpiBytes), "fragment epilogue: column buffers");
    for (int tile = unit; tile < total_tiles; tile += n_units) {
      int g, m0, n0;
      TcTile tl;
      typename PreOf<Epi>::type pre;
      if constexpr (EpiFragment<Epi>::value) {
        tc::mbar_wait(&full[stage], phase);
        tl = recs[stage];
        g = tl.g; m0 = tl.m0; n0 = tl.n0;
        pre = epi.begin(tl, t, m0 + cw * 64 + fr);
      } else {
        decode(tile, g, m0, n0);
      }
      // fragment epilogues: the tile's first wgmma ignores the accumulators (scale-d 0) instead of a zeroing pass over
      // them while the tensor pipe waits
      if constexpr (!EpiFragment<Epi>::value) {
#pragma unroll
        for (int i = 0; i < BN / 2; ++i) acc[i] = 0;
      }
      int prev = -1;
      for (int kb = 0; kb < KB; ++kb) {
        tc::mbar_wait(&full[stage], phase);
        tc::wgmma_fence();
        const uint32_t sa = tc::smem_u32(smem + stage * Cfg::kStageBytes) + cw * 64 * 128;
        const uint32_t sb = tc::smem_u32(smem + stage * Cfg::kStageBytes) + Cfg::kOps * Cfg::kABytes;
#pragma unroll
        for (int ks = 0; ks < Cfg::kBK / Cfg::kMmaK; ++ks) {
          const uint32_t koff = ks * 32;  // bytes inside the 128-byte swizzle row
          const uint64_t a_hi = tc::smem_desc_sw128(sa + koff), b_hi = tc::smem_desc_sw128(sb + koff);
          const uint32_t sd = EpiFragment<Epi>::value && kb == 0 && ks == 0 ? 0u : 1u;
          if constexpr (Cfg::kS8) {
            tc::wgmma_ss_s8<BN>(acc, a_hi, b_hi, sd);
          } else if constexpr (Cfg::kIL) {   // lo 64 bytes after hi in the same row; F16X3's product order
            const uint64_t a_lo = tc::smem_desc_sw128(sa + 64 + koff), b_lo = tc::smem_desc_sw128(sb + 64 + koff);
            tc::wgmma_ss<false, BN>(acc, a_lo, b_hi, 1u);
            tc::wgmma_ss<false, BN>(acc, a_hi, b_lo, 1u);
            tc::wgmma_ss<false, BN>(acc, a_hi, b_hi, 1u);
          } else if (Cfg::kOps == 2) {
            const uint64_t a_lo = tc::smem_desc_sw128(sa + Cfg::kABytes + koff);
            const uint64_t b_lo = tc::smem_desc_sw128(sb + Cfg::kBBytes + koff);
            // small terms first, then the dominant hi*hi
            tc::wgmma_ss<Cfg::kTF32, BN>(acc, a_lo, b_hi, 1u);
            tc::wgmma_ss<Cfg::kTF32, BN>(acc, a_hi, b_lo, 1u);
            tc::wgmma_ss<Cfg::kTF32, BN>(acc, a_hi, b_hi, 1u);
          } else {
            tc::wgmma_ss<Cfg::kTF32, BN>(acc, a_hi, b_hi, sd);
          }
        }
        tc::wgmma_commit();
        tc::wgmma_wait<1>();            // the previous K-block's MMAs are done: its slot may be refilled
        if (prev >= 0) release(prev);
        prev = stage;
        if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
      }
      tc::wgmma_wait<0>();
      tc::reg_fence(acc);
      if (prev >= 0) release(prev);

      const int rbase = m0 + cw * 64;        // row (inside the group) of the warpgroup's first row
      if constexpr (EpiFragment<Epi>::value) {
        float* cols = epi_scratch + (2 * cw + cbuf) * BN;
        cbuf ^= 1;
        cols[t] = pre.col.x;
        cols[t + 128] = pre.col.y;
        tc::named_sync(1 + cw, 128);
        epi.fragment(tl, rbase + fr, fc, acc, cols, pre);
      } else if constexpr (!Cfg::kS8) {
        // ---- epilogue: 32-column blocks through shared memory ----
        const int r = rbase + t;
        const bool row_ok = t < 64 && r < pb.grp_m[g];
        typename Epi::State est;
        epi.tile_begin(est);
#pragma unroll
        for (int c = 0; c < BN; c += 32) {
#pragma unroll
          for (int ii = 0; ii < 4; ++ii) {
            const int i = c / 8 + ii;
            *reinterpret_cast<float2*>(sw + fr * TC_EPI_PITCH + ii * 8 + fc) = make_float2(acc[4 * i], acc[4 * i + 1]);
            *reinterpret_cast<float2*>(sw + (fr + 8) * TC_EPI_PITCH + ii * 8 + fc) = make_float2(acc[4 * i + 2], acc[4 * i + 3]);
          }
          tc::named_sync(1 + cw, 128);
          const int ncols = min(32, pb.N - (n0 + c));
          bool done = false;
          if constexpr (EpiCoalesced<Epi>::value) {
            if (!epi.direct(n0 + c)) {
              // thread (r4, c4) owns 4 consecutive columns of rows it * 16 + r4 -> 8 threads cover 128 contiguous bytes
              const int c4 = (t & 7) * 4, r4 = t >> 3;
              if (c4 < ncols) {
                if constexpr (EpiPrefetch<Epi>::value) {
                  float4 pre[4];
#pragma unroll
                  for (int it = 0; it < 4; ++it) {
                    const int rr = it * 16 + r4;
                    pre[it] = rbase + rr < pb.grp_m[g] ? epi.fetch(g, rbase + rr, n0 + c + c4) : make_float4(0.f, 0.f, 0.f, 0.f);
                  }
#pragma unroll
                  for (int it = 0; it < 4; ++it) {
                    const int rr = it * 16 + r4;
                    if (rbase + rr < pb.grp_m[g])
                      epi.vec4(g, rbase + rr, n0 + c + c4, *reinterpret_cast<const float4*>(sw + rr * TC_EPI_PITCH + c4), pre[it]);
                  }
                } else {
#pragma unroll
                  for (int it = 0; it < 4; ++it) {
                    const int rr = it * 16 + r4;
                    if (rbase + rr < pb.grp_m[g])
                      epi.vec4(g, rbase + rr, n0 + c + c4, *reinterpret_cast<const float4*>(sw + rr * TC_EPI_PITCH + c4));
                  }
                }
              }
              done = true;
            }
          }
          if (!done && row_ok && ncols > 0) {
            float f[32];
#pragma unroll
            for (int i = 0; i < 32; i += 4) {
              const float4 v = *reinterpret_cast<const float4*>(sw + t * TC_EPI_PITCH + i);
              f[i] = v.x; f[i + 1] = v.y; f[i + 2] = v.z; f[i + 3] = v.w;
            }
            epi(est, g, r, n0 + c, f, ncols);
          }
          tc::named_sync(1 + cw, 128);
        }
        if (row_ok) epi.tile_end(est, g, r, n0 / BN);
      }
    }
  }
  if (PAIR) tc::cluster_sync_all();   // no CTA may exit while its peer can still multicast into it or arrive on its barriers
}

template <TcMode MODE, class Epi, int BN = TC_BN>
__global__ void __launch_bounds__(TC_THREADS, 1)
tc_gemm_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
               const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo, TcProblem pb,
               Epi epi) {
  tc_gemm_body<MODE, Epi, BN, false>(tmA_hi, tmA_lo, tmB_hi, tmB_lo, pb, epi);
}

// pb.tile_start: prefix of ceil(m / TC2_BM) per group; B tensor maps with boxes of BN / 2 rows; even grid.
template <TcMode MODE, class Epi, int BN = TC_BN>
__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(TC_THREADS, 1)
tc_gemm_pair_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                    const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo, TcProblem pb,
                    Epi epi) {
  tc_gemm_body<MODE, Epi, BN, true>(tmA_hi, tmA_lo, tmB_hi, tmB_lo, pb, epi);
}

// ---- host side ----
// Device group tables of a TcProblem
struct TcPlan {
  int* batch; int* row0; int* m; int* tile_start;
  TcProblem problem(int n_groups, int N, int K) const { return {batch, row0, m, tile_start, n_groups, N, K}; }
};

// Uniform tables: group g = `rows` A rows from row_base + g * row_stride against B batch item batch_base + g, in M tiles of
// tile_rows (TC_BM, or TC2_BM for the pair kernel).  One single-thread launch (corr_tc.cu).
int launch_tc_plan(const TcPlan& pl, int n_groups, int rows, int row_stride, int row_base, int batch_base, int tile_rows,
                   cudaStream_t st);

// *amax = max(*amax, max |x|) as the bits of a non-negative float, for grad_exp (corr_tc.cu; 256 threads per block)
int launch_amax(const float* x, size_t n, unsigned* amax, unsigned grid, cudaStream_t st);

// Operands: A [a_rows][K], B [b_batch][N][K], row pitches lda / ldb in elements (0: dense).  The lo parts are read in the
// split modes only (TcCfg::kOps == 2).  F16X3I: a_hi / b_hi are the interleaved arrays, rows of 64 ceil(K / 32) elements.
struct TcOperands {
  const void* a_hi; const void* a_lo; uint64_t a_rows, lda;
  const void* b_hi; const void* b_lo; uint64_t b_batch, ldb;
};

// One launch of tc_gemm_kernel (or tc_gemm_pair_kernel when PAIR) on pb.  m_tiles bounds the M tiles of the plan (TC_BM
// rows, TC2_BM for pairs); the grid is one CTA (pair) per output tile up to one per SM, at least one.  prof >= 0 times the
// launch under that profile class.
template <TcMode MODE, class Epi, int BN = TC_BN, bool PAIR = false>
int tc_launch(const TcOperands& op, const TcProblem& pb, int m_tiles, const Epi& epi, cudaStream_t st, int prof = -1) {
  using Cfg = TcCfg<MODE, BN>;
  constexpr int elem = MODE == TcMode::S8 ? TMAP_S8 : MODE == TcMode::BF16 ? TMAP_BF16 : Cfg::kElem == 2 ? TMAP_F16 : TMAP_F32;
  CUtensorMap ta[2], tb[2];
  const uint64_t cols = Cfg::kIL ? 64 * (uint64_t)((pb.K + 31) / 32) : (uint64_t)pb.K;   // elements per operand row
  for (int i = 0; i < Cfg::kOps; ++i) {   // single-pass modes pass the hi maps twice
    if (int rc = make_tmap_2d(&ta[i], i ? op.a_lo : op.a_hi, op.a_rows, cols, TC_BM, Cfg::kRowElems, elem, op.lda)) return rc;
    if (int rc = make_tmap_3d(&tb[i], i ? op.b_lo : op.b_hi, op.b_batch, pb.N, cols, PAIR ? BN / 2 : BN, Cfg::kRowElems, elem,
                              op.ldb))
      return rc;
  }
  const auto kern = [] {   // if constexpr: only the kernel launched here is instantiated
    if constexpr (PAIR) return tc_gemm_pair_kernel<MODE, Epi, BN>;
    else return tc_gemm_kernel<MODE, Epi, BN>;
  }();
  static PerDev<bool> attr_dev;   // one per instantiation
  bool& attr = attr_dev.get();
  if (!attr) {
    DTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, Cfg::kSmem));
    attr = true;
  }
  const int units = PAIR ? num_sms() / 2 : num_sms();
  long long n = (long long)m_tiles * cdiv(pb.N, BN);
  if (n > units) n = units;
  const int grid = (PAIR ? 2 : 1) * (n < 1 ? 1 : (int)n);
  ProfRange pr(prof, st);
  kern<<<grid, TC_THREADS, Cfg::kSmem, st>>>(ta[0], ta[Cfg::kOps - 1], tb[0], tb[Cfg::kOps - 1], pb, epi);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// N tile by N: 64, 128 or 256
inline int tc_bn(int N) { return N <= 64 ? 64 : N <= 128 ? 128 : 256; }

template <TcMode MODE, class Epi>
int tc_launch_bn(const TcOperands& op, const TcProblem& pb, int m_tiles, const Epi& epi, cudaStream_t st, int prof = -1) {
  switch (tc_bn(pb.N)) {
    case 64: return tc_launch<MODE, Epi, 64>(op, pb, m_tiles, epi, st, prof);
    case 128: return tc_launch<MODE, Epi, 128>(op, pb, m_tiles, epi, st, prof);
    default: return tc_launch<MODE, Epi, 256>(op, pb, m_tiles, epi, st, prof);
  }
}

}  // namespace dtk

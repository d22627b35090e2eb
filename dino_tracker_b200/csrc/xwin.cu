// Coarse pass + exact window (see xwin.cuh): kernels and launchers.
#include <cuda_fp16.h>

#include "common.cuh"
#include "corr.cuh"
#include "head.cuh"
#include "tcgemm.cuh"
#include "xwin.cuh"

namespace dtk {

// ====================================================================================================== 1. coarse GEMM
// Epilogue of the single-pass GEMM (int8 operands, or fp16 over the `hi` halves): nothing is stored per token.  Per (map, 128-token tile), two
// per 256-column GEMM tile: key1 = bits(max) << 32 | (0x7fffffff - first token holding it), max2 = second largest value
// (>= 0).  Values are the same expression as the exact path, relu(acc / max(|d| |F|, 1e-8)), with a fast division (its
// error is part of XW_EPS).  The int8 pass forms the same statistics of acc * fac_x * fac_d from its exact int32
// accumulators (their conversion to float is exact up to C = 1040; above, eps's slack covers its rounding, xwin.cuh).
//
// A fragment epilogue (tcgemm.cuh): it works on the accumulator registers of all eight consumer warps; the tile's token
// factors come from shared memory, where the GEMM body staged them (begin()).  Per element only u = acc * (1 / |F|) is
// formed; the row's positive factor 1 / |d| (and the ReLU) are applied to the two statistics at the end -- multiplication by a positive constant does not change which token holds
// the maximum.  The statistics -- the maximum, the first token holding it, the second largest value of the multiset -- do
// not depend on the order the values are folded in: a thread folds its 32 values per (row, key tile) into the maximum and
// the second value on min / max alone, the 4 lanes of the quad merge theirs by shuffles, and only then does each lane look
// for the quad's maximum among its values; the smallest of the four lanes' first columns holding it is the token.
constexpr int XW_GEMM_BN = 2 * XW_TILE;   // N tile of the coarse GEMM (m64n256 per consumer warpgroup)

template <class Acc>   // float: fp16 pass, int: int8 pass
struct CoarseEpi {
  static constexpr bool kFragment = true;
  static constexpr bool kS8 = std::is_same<Acc, int>::value;
  const float* rnorms;     // [T][P] token factor: 1 / |F[t][p]| (xw_rnorm_kernel; every norm is >= XW_MIN_NORM on this
                           // path), int8 pass: s_x / |F| (q_fac)
  const float* desc_norm;  // row factor 1 / max(|d|, XW_MIN_NORM) (fp16 pass), desc_norm[row] itself (int8 pass: s_d / |d|)
  const int* grp_map0;
  unsigned long long* key1;
  float* max2;
  int n_tiles, P;

  // per tile, read when the tile starts: the token factors of columns n0 + t and n0 + t + 128 (0 past the end of the map),
  // and for the row this thread writes (r + 8 (q >> 1), below) its row factor and its first map
  struct Pre { float2 col; float dv; int map0; };
  __device__ __forceinline__ Pre begin(const TcTile& tl, int t, int r) const {
    const float* rn = rnorms + (size_t)tl.batch * P;
    const int c0 = tl.n0 + t, c1 = c0 + XW_TILE;
    const int rr = r + 8 * ((threadIdx.x & 3) >> 1);
    Pre p;
    p.col = make_float2(c0 < P ? __ldg(rn + c0) : 0.f, c1 < P ? __ldg(rn + c1) : 0.f);
    p.dv = rr < tl.m ? __ldg(desc_norm + tl.row0 + rr) : 0.f;
    p.map0 = __ldg(grp_map0 + tl.g);
    return p;
  }
  static __device__ __forceinline__ float as_float(Acc a) {
    if constexpr (kS8) return __int_as_float(a); else return a;
  }
  static __device__ __forceinline__ Acc from_float(float v) {
    if constexpr (kS8) return __float_as_int(v); else return v;
  }
  // Key tile kh of the thread's two rows, pass 1: forms the values, leaves them in acc as floats (int8 pass: their bits)
  // and folds their maximum into m1[h] (row r + 8 h).  cols: the tile's token factors.  EDGE: the GEMM tile reaches past
  // the end of the map
  template <bool EDGE>
  __device__ __forceinline__ void fold_max(float (&m1)[2], int kh, const float* cols, int n0, int fc,
                                           Acc (&acc)[XW_GEMM_BN / 2]) const {
#pragma unroll
    for (int ii = 0; ii < XW_TILE / 8; ++ii) {   // (constant trip count: acc must stay in registers)
      const int i = kh * XW_TILE / 8 + ii;
      const float2 rnv = tc::lds_f2(tc::smem_u32(cols + fc + 8 * i));
      const int col = n0 + 8 * i + fc;
      const bool ok0 = !EDGE || col < P, ok1 = !EDGE || col + 1 < P;   // columns past the end of the map never win
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        const float a = ok0 ? (float)acc[4 * i + 2 * h] * rnv.x : -INFINITY;
        const float b = ok1 ? (float)acc[4 * i + 2 * h + 1] * rnv.y : -INFINITY;
        acc[4 * i + 2 * h] = from_float(a);
        acc[4 * i + 2 * h + 1] = from_float(b);
        m1[h] = fmaxf(m1[h], fmaxf(a, b));
      }
    }
  }
  // Pass 2, once m1 is the quad's maximum of row r + 8 h: among the thread's values of key tile kh, m2 = the largest of
  // those below m1, and pos records the columns holding m1.  One compare per value; its predicate selects the other two
  // updates.  Matches come in decreasing column order c = 8 i + j, and each sets pos = pos / 512 + (c + 1) (a
  // predicated FFMA, kept on the FMA pipe, where a predicated move or add would become an ALU-pipe SEL): the integer
  // part of pos is 1 + the first column holding m1 (0: none), and pos has a fractional part iff m1 is held twice.
  // pos < 257, so pos / 512 < 0.51 and the fraction, >= 2^-9 once set, survives the rounding of the sum (ulp <= 2^-15).
  __device__ __forceinline__ void scan(float m1, int h, int kh, const Acc (&acc)[XW_GEMM_BN / 2], float& pos,
                                       float& m2) const {
    pos = 0.f;
    m2 = -INFINITY;
#pragma unroll
    for (int ii = XW_TILE / 8 - 1; ii >= 0; --ii) {
      const int i = kh * XW_TILE / 8 + ii;
#pragma unroll
      for (int j = 1; j >= 0; --j)
        asm("{\n\t.reg .pred p;\n\t"
            "setp.eq.f32 p, %2, %3;\n\t"
            "@p fma.rn.f32 %0, %0, 0f3B000000, %4;\n\t"
            "@!p max.f32 %1, %1, %2;\n\t}"
            : "+f"(pos), "+f"(m2)
            : "f"(as_float(acc[4 * i + 2 * h + j])), "f"(m1), "f"((float)(8 * i + j + 1)));
    }
  }
  __device__ __forceinline__ void fragment(const TcTile& tl, int r, int fc, Acc (&acc)[XW_GEMM_BN / 2], const float* cols,
                                           const Pre& pre) const {
    // after the quad's merge every lane holds all four results; lane q keeps and writes row r + 8 (q >> 1) of key tile
    // 2 (n0 / 256) + (q & 1)
    const int q = threadIdx.x & 3, n0 = tl.n0;
    const bool edge = n0 + XW_GEMM_BN > P;
    float o1, o2;
    int otok;
#pragma unroll
    for (int kh = 0; kh < 2; ++kh) {
      float m1[2] = {-INFINITY, -INFINITY};   // rows r, r + 8
      if (edge) fold_max<true>(m1, kh, cols, n0, fc, acc);
      else fold_max<false>(m1, kh, cols, n0, fc, acc);
#pragma unroll
      for (int h = 0; h < 2; ++h) {
#pragma unroll
        for (int sh = 1; sh <= 2; sh <<= 1) m1[h] = fmaxf(m1[h], __shfl_xor_sync(0xffffffffu, m1[h], sh));
        float pos, m2;
        scan(m1[h], h, kh, acc, pos, m2);
        const int ip = (int)pos;   // (truncates)
        int tok = ip ? n0 + fc + ip - 1 : 0x7fffffff;
        int cnt = (ip != 0) + ((float)ip != pos);   // 0, 1, or 2 for "at least two"
#pragma unroll
        for (int sh = 1; sh <= 2; sh <<= 1) {
          tok = min(tok, __shfl_xor_sync(0xffffffffu, tok, sh));
          cnt += __shfl_xor_sync(0xffffffffu, cnt, sh);
          m2 = fmaxf(m2, __shfl_xor_sync(0xffffffffu, m2, sh));
        }
        if ((q & 1) == kh && (q >> 1) == h) {
          o1 = m1[h];
          o2 = cnt > 1 ? m1[h] : m2;   // the maximum held twice is also the second value
          otok = tok;
        }
      }
    }
    const int rr = r + 8 * (q >> 1), nt = n0 / XW_TILE + (q & 1);
    if (rr >= tl.m || nt >= n_tiles) return;   // padding row, or a key tile lying completely past the end of the map
    const float rdn = kS8 ? pre.dv : __fdividef(1.f, fmaxf(pre.dv, XW_MIN_NORM));
    const size_t off = (size_t)(pre.map0 + rr) * n_tiles + nt;
    key1[off] = ((unsigned long long)__float_as_uint(fmaxf(o1 * rdn, 0.f)) << 32) | (unsigned)(0x7fffffff - otok);
    max2[off] = fmaxf(o2 * rdn, 0.f);
  }
};

// rnorms[i] = 1 / norms[i]; *min_bits = bit pattern of the smallest norm (norms are >= 0: the bit pattern orders like the value)
__global__ void xw_rnorm_kernel(const float* __restrict__ norms, float* __restrict__ rnorms, size_t n, unsigned* __restrict__ min_bits) {
  float mn = INFINITY;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) {
    const float v = norms[i];
    rnorms[i] = __fdiv_rn(1.f, fmaxf(v, XW_MIN_NORM));
    mn = fminf(mn, v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  if ((threadIdx.x & 31) == 0) atomicMin(min_bits, __float_as_uint(fmaxf(mn, 0.f)));
}

int launch_xw_rnorms(const FeatView& fv, float* rnorms, unsigned* min_bits, cudaStream_t st) {
  const size_t n = (size_t)fv.T * fv.P;
  DTK_CUDA(cudaMemsetAsync(min_bits, 0x7f, sizeof(unsigned), st));   // 0x7f7f7f7f: a huge positive float
  ProfRange pr(PROF_XW_PLAN, st);
  xw_rnorm_kernel<<<num_sms() * 4, 256, 0, st>>>(fv.norms, rnorms, n, min_bits);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int launch_xw_coarse(const FeatView& fv, const void* desc_hi, int desc_rows, const float* desc_norm, const int* grp_frame,
                     const int* grp_row0, const int* grp_m, const int* grp_map0, const int* tile_start, int n_groups,
                     int max_tiles, const XwChunk& xc, cudaStream_t st, const float* rnorms, const void* desc_q8,
                     const float* desc_fac) {
  static_assert(XW_GEMM_BN == 256 && XW_TILE == 128, "one m64n256 GEMM N tile = two 128-token key tiles (CoarseEpi::fragment)");
  TcProblem pb{grp_frame, grp_row0, grp_m, tile_start, n_groups, fv.P, fv.C};
  if (desc_q8) {
    DTK_CHECK_ARG(fv.s8() && fv.C % 16 == 0 && fv.C <= XW_S8_MAX_C, "int8 coarse pass: needs the int8 features, C %% 16 == 0 "
                  "and C <= %d", XW_S8_MAX_C);
    CoarseEpi<int> epi{fv.q_fac, desc_fac, grp_map0, xc.key1, xc.max2, cdiv(fv.P, XW_TILE), fv.P};
    return tc_launch<TcMode::S8, CoarseEpi<int>, XW_GEMM_BN, true>({desc_q8, nullptr, (uint64_t)desc_rows, 0, fv.q8, nullptr,
                                                                    (uint64_t)fv.T, 0}, pb, max_tiles, epi, st, PROF_XW_COARSE);
  }
  CoarseEpi<float> epi{rnorms, desc_norm, grp_map0, xc.key1, xc.max2, cdiv(fv.P, XW_TILE), fv.P};
  return tc_launch<TcMode::F16, CoarseEpi<float>, XW_GEMM_BN, true>({desc_hi, nullptr, (uint64_t)desc_rows, 0, fv.hi, nullptr,
                                                                     (uint64_t)fv.T, 0}, pb, max_tiles, epi, st, PROF_XW_COARSE);
}

// ====================================================================================================== 2. plan
// (a) one warp per MAP (lane = tile): global coarse maximum, candidate tiles (max1 >= gmax - 2 eps), ambiguity (some tile's
//     SECOND value is also within 2 eps: an arg-max candidate whose token is unknown).  Writes the candidate tokens and
//     pinfo[map] = coarse arg-max token, or -1 - token if the map is ambiguous.
// (b) one warp per CELL: the lower medians of the unambiguous maps' coarse arg-max row / column give the box centre; a map
//     fits if every candidate lies within +-XW_SLACK of it.  The cell's extent (box_ext) is the union of its fitting maps'
//     candidate windows: the only box tokens the head reads.  Its tokens and the cell are counted into box_cnt[0] / [1].
//     KPL = cdiv(n_tiles, 32) keys per lane, tile t = lane + 32 q: candidates are ranked in tile order for any KPL.
constexpr int PLAN_WARPS = 8;
template <int KPL>
__global__ void __launch_bounds__(PLAN_WARPS * 32)
xw_cand_kernel(int n_maps, const float* __restrict__ desc_norm, float min_norm, int n_groups, int n_tiles,
               const unsigned long long* __restrict__ key1, const float* __restrict__ eps_map,
               const float* __restrict__ max2, int* __restrict__ cand, int* __restrict__ pinfo, int* __restrict__ slow_cnt) {
  const int lane = threadIdx.x & 31;
  const int gw = blockIdx.x * PLAN_WARPS + (threadIdx.x >> 5), nw = gridDim.x * PLAN_WARPS;
  if (gw == 0)   // zero the queue counters of this chunk (n_groups per-group counts + the total + the uncertified count)
    for (int i = lane; i <= n_groups + 3; i += 32) slow_cnt[i] = 0;
  for (int map = gw; map < n_maps; map += nw) {
    const unsigned long long* k1 = key1 + (size_t)map * n_tiles;
    const float* k2 = max2 + (size_t)map * n_tiles;
    unsigned long long kk[KPL] = {};
    float v2[KPL] = {};
#pragma unroll
    for (int q = 0; q < KPL; ++q) {
      const int t = lane + 32 * q;
      if (t < n_tiles) { kk[q] = __ldg(k1 + t); v2[q] = __ldg(k2 + t); }
    }
    unsigned long long gk = kk[0];
#pragma unroll
    for (int q = 1; q < KPL; ++q) gk = gk > kk[q] ? gk : kk[q];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, gk, o); gk = t > gk ? t : gk; }
    const float gmax = __uint_as_float((unsigned)(gk >> 32));
    const int ptok = 0x7fffffff - (int)(gk & 0xffffffffu);
    const float eps = eps_map ? eps_map[map] : XW_EPS;
    const float th = gmax - 2.f * eps;
    bool amb = false;
    int ncand = 0;
#pragma unroll
    for (int q = 0; q < KPL; ++q) {
      const int t = lane + 32 * q;
      const bool in = t < n_tiles;
      const bool isc = in && __uint_as_float((unsigned)(kk[q] >> 32)) >= th;
      const unsigned cm = __ballot_sync(0xffffffffu, isc);
      amb = amb || __any_sync(0xffffffffu, in && v2[q] >= th);
      const int rank = ncand + __popc(cm & ((1u << lane) - 1u));
      if (isc && rank < XW_MAX_CAND) cand[(size_t)map * XW_MAX_CAND + rank] = 0x7fffffff - (int)(kk[q] & 0xffffffffu);
      ncand += __popc(cm);
    }
    // a (near-)zero map has no meaningful arg-max candidates; a descriptor below the split's faithful range voids the bound
    amb = amb || ncand > XW_MAX_CAND || !(gmax > 4.f * eps) || !(desc_norm[map] >= min_norm);
    if (lane >= ncand && lane < XW_MAX_CAND) cand[(size_t)map * XW_MAX_CAND + lane] = -1;
    if (lane == 0) pinfo[map] = amb ? -1 - ptok : ptok;
  }
}

__global__ void __launch_bounds__(PLAN_WARPS * 32)
xw_cell_kernel(XwCells cells, int w, const int* __restrict__ cand, const int* __restrict__ pinfo, int* __restrict__ stat,
               int* __restrict__ cell_of, int2* __restrict__ box_org, int4* __restrict__ box_ext, int* __restrict__ box_cnt) {
  __shared__ short s_r[PLAN_WARPS][XW_MAX_CELL], s_c[PLAN_WARPS][XW_MAX_CELL];
  __shared__ unsigned char s_ok[PLAN_WARPS][XW_MAX_CELL];
  const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  const int gw = blockIdx.x * PLAN_WARPS + wid, nw = gridDim.x * PLAN_WARPS;
  for (int cell = gw; cell < cells.n_cells; cell += nw) {
    const int row0 = cells.row0[cell], m = cells.m[cell];
    int nv = 0;
    for (int r = lane; r < m; r += 32) {
      const int pi = __ldg(pinfo + row0 + r);
      const int ptok = pi >= 0 ? pi : -1 - pi;
      s_r[wid][r] = (short)(ptok / w);
      s_c[wid][r] = (short)(ptok - (ptok / w) * w);
      s_ok[wid][r] = pi >= 0 ? 1 : 0;
      nv += pi >= 0 ? 1 : 0;
      cell_of[row0 + r] = cell;
    }
    __syncwarp();
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) nv += __shfl_xor_sync(0xffffffffu, nv, o);
    int med_r = -1, med_c = -1;
    if (nv > 0) {   // lower medians over the unambiguous maps
      const int want = (nv - 1) / 2;
      for (int r = lane; r < m; r += 32) {
        if (!s_ok[wid][r]) continue;
        int rk_r = 0, rk_c = 0;
        const int vr = s_r[wid][r], vc = s_c[wid][r];
        for (int q = 0; q < m; ++q) {
          if (!s_ok[wid][q]) continue;
          rk_r += (s_r[wid][q] < vr) || (s_r[wid][q] == vr && q < r);
          rk_c += (s_c[wid][q] < vc) || (s_c[wid][q] == vc && q < r);
        }
        if (rk_r == want) med_r = vr;
        if (rk_c == want) med_c = vc;
      }
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        med_r = max(med_r, __shfl_xor_sync(0xffffffffu, med_r, o));
        med_c = max(med_c, __shfl_xor_sync(0xffffffffu, med_c, o));
      }
    }
    // the fitting maps' candidates span rows [lo_r, hi_r] and columns [lo_c, hi_c]
    int n_fit = 0, lo_r = INT_MAX, hi_r = INT_MIN, lo_c = INT_MAX, hi_c = INT_MIN;
    for (int r = lane; r < m; r += 32) {
      const int map = row0 + r;
      bool fit = s_ok[wid][r] != 0;
      int mr0 = INT_MAX, mr1 = INT_MIN, mc0 = INT_MAX, mc1 = INT_MIN;
      if (fit) {
        const int4 cd = __ldg(reinterpret_cast<const int4*>(cand) + map);
        const int ct[4] = {cd.x, cd.y, cd.z, cd.w};
#pragma unroll
        for (int q = 0; q < XW_MAX_CAND; ++q)
          if (ct[q] >= 0) {
            const int tr = ct[q] / w, tc_ = ct[q] - tr * w;
            fit = fit && abs(tr - med_r) <= XW_SLACK && abs(tc_ - med_c) <= XW_SLACK;
            mr0 = min(mr0, tr); mr1 = max(mr1, tr); mc0 = min(mc0, tc_); mc1 = max(mc1, tc_);
          }
      }
      stat[map] = fit ? 0 : 1;
      n_fit += fit ? 1 : 0;
      if (fit) { lo_r = min(lo_r, mr0); hi_r = max(hi_r, mr1); lo_c = min(lo_c, mc0); hi_c = max(hi_c, mc1); }
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      n_fit += __shfl_xor_sync(0xffffffffu, n_fit, o);
      lo_r = min(lo_r, __shfl_xor_sync(0xffffffffu, lo_r, o)); hi_r = max(hi_r, __shfl_xor_sync(0xffffffffu, hi_r, o));
      lo_c = min(lo_c, __shfl_xor_sync(0xffffffffu, lo_c, o)); hi_c = max(hi_c, __shfl_xor_sync(0xffffffffu, hi_c, o));
    }
    if (lane == 0) {
      const int org_r = med_r - XW_BOX / 2, org_c = med_c - XW_BOX / 2;
      box_org[cell] = n_fit > 0 ? make_int2(org_r, org_c) : make_int2(0, INT_MIN);
      if (n_fit > 0) {   // every candidate lies within +-XW_SLACK of the centre: the extent lies inside the 21 x 21 box
        const int4 e = make_int4(lo_r - WM / 2 - org_r, lo_c - WM / 2 - org_c, hi_r - lo_r + WM, hi_c - lo_c + WM);
        box_ext[cell] = e;
        atomicAdd(box_cnt, e.z * e.w);
        atomicAdd(box_cnt + 1, 1);
      }
    }
    __syncwarp();
  }
}

int launch_xw_plan(const XwCells& cells, const float* desc_norm, int n_groups, const dinotrk_geom& g, const XwChunk& xc,
                   cudaStream_t st, int n_maps, float min_norm, const float* eps) {
  static_assert(XW_MAX_CAND == 4, "candidates are read as one int4");
  const int n_tiles = cdiv(g.h * g.w, XW_TILE);
  DTK_CHECK_GRID(g, "exact-window path");
  static_assert(DTK_GRID_MAX_TOKENS <= 256 * XW_TILE, "xw_cand_kernel keeps at most 8 keys per lane");
  DTK_CHECK_ARG(cells.max_m <= XW_MAX_CELL, "exact-window path: cell of %d rows", cells.max_m);
  if (cells.n_cells <= 0 || n_maps <= 0) return DINOTRK_OK;
  ProfRange pr(PROF_XW_PLAN, st);
  int grid = cdiv(n_maps, PLAN_WARPS);
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  auto cand_kernel = n_tiles <= 64 ? xw_cand_kernel<2> : n_tiles <= 128 ? xw_cand_kernel<4> : xw_cand_kernel<8>;
  cand_kernel<<<grid, PLAN_WARPS * 32, 0, st>>>(n_maps, desc_norm, min_norm, n_groups, n_tiles, xc.key1, eps, xc.max2, xc.cand, xc.pinfo, xc.slow_cnt);
  DTK_LAUNCHED();
  grid = cdiv(cells.n_cells, PLAN_WARPS);
  if (grid > num_sms() * 8) grid = num_sms() * 8;
  xw_cell_kernel<<<grid, PLAN_WARPS * 32, 0, st>>>(cells, g.w, xc.cand, xc.pinfo, xc.stat, xc.cell_of, xc.box_org, xc.box_ext,
                                                   xc.slow_cnt + n_groups + 2);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// ====================================================================================================== 3. exact box GEMM
// Persistent, warp-specialised (same roles as tc_gemm_kernel).  The cell's DESCRIPTORS are the wgmma M operand (64 rows per
// consumer warpgroup) and the tokens of its tight extent (XwChunk::box_ext: bh x bw tokens, 15..21 each) the N operand, in
// PARTS of whole extent rows, at most XW_PART_TOK = 128 tokens each (m64n128k16; the columns past a part's tokens are
// computed and never stored): rp = floor(128 / bw) rows per part at most (8 for bw <= 16, 6 at bw = 21), the rows shared
// out evenly.  A cell whose maps agree (15 x 15 or 16 x 16 tokens) is two parts; the whole 21 x 21 box is four.  A stage
// of a 128-token part is small, so the ring holds five or six stages: a stage's time is set by how many fills are in
// flight, not by its bytes (DESIGN.md 4.3).  Two layouts:
//   MB = 64   every cell of the call has <= 64 maps: the parts go in pairs (their count is rounded up to even), warpgroup 1
//             on the first and warpgroup 2 on the second of a pair.  A ring stage holds the descriptor K-block and both
//             parts of the pair, so the descriptors are loaded once per pair and each warpgroup drains its pipeline once
//             per pair.
//   MB = 128  cells of up to 128 maps: warpgroup 1 takes descriptor rows 0-63 and warpgroup 2 rows 64-127 of the same part;
//             the parts run one after the other, a stage holding the descriptor K-block and one part.
// K blocks of 32 channels.  Split precision: lo*hi + hi*lo + hi*hi per K step of 16, K ascending -- the full-map GEMM's
// sequence of products, whatever the extent and its parts.  The descriptor K-block is two tiles (hi, lo) of
// 64-byte-swizzled rows.  A part's tokens arrive as one 4-D TMA box {channels, bw columns, rows, 1 frame} of the feature
// video, zero-filled outside the token grid, landing at the start of the part's 1024-byte-aligned slot (part token (y, x)
// in slot row y bw + x).  The box's shape changes from cell to cell, so the kernel takes a table of tensor maps, one per
// (bw, rows) (XwTokMaps).  Token rows come in one of two layouts (HILO):
//   false  the separate hi and lo halves [T][h][w][C]: two boxes of 64-byte rows (32 channels) per part and K block.
//   true   the interleaved split [T][h][w][ceil(C / 32)][64] (FeatView::hilo): one box of 128-byte rows [hi 32 | lo 32] in
//          the 128-byte swizzle; a K step reads hi 0 / 32 and lo 64 / 96 bytes into the row.  Same bytes in half as many
//          rows: the TMA's cost per row, not the MMA, bounds the 64-byte layout (DESIGN.md 4.3).
// A MB = 64 stage is 40 KiB in either layout (five fit), a MB = 128 stage 32 KiB (six).
// Epilogue: from the accumulator fragment through a per-warp shared-memory tile (16 maps x 32 part tokens) to
// xbox[map][xw_col(row, column)] of the 21 x 21 box, one map's consecutive tokens per warp store.
constexpr int XW_EXT_MIN = WM;                          // smallest extent side: one candidate's window
constexpr int XW_NW = XW_BOX - XW_EXT_MIN + 1;          // extent widths 15 .. 21
constexpr int XW_PART_TOK = 128;                        // tokens of a part at most: its wgmma N
constexpr int XW_PART_ROWS = XW_PART_TOK / XW_EXT_MIN;  // rows of a part at most (8)
constexpr int XW_EPI_ROWS = 16;                         // maps of one consumer warp's fragment rows
constexpr int XW_EPI_PITCH = 40;                        // floats per staged map row: the quads' 8-byte writes are conflict-free

// the token boxes' tensor maps: [hi or the interleaved split, lo][bw - XW_EXT_MIN][rows - 1]
template <bool HILO>
struct XwTokMaps { CUtensorMap m[HILO ? 1 : 2][XW_NW][XW_PART_ROWS]; };

template <int MB, bool HILO>
struct XwCfg {
  static constexpr int kBK = 32;                                  // channels per K block
  static constexpr int kRow = 2 * kBK;                            // bytes per descriptor row of one half (64-byte swizzle)
  static constexpr int kTokRow = HILO ? 2 * kRow : kRow;          // bytes per token row of one TMA box
  static constexpr int kBoxes = HILO ? 1 : 2;                     // token boxes per part and K block
  static constexpr int kDescBytes = MB * kRow;                    // one operand half (hi or lo) of the descriptor K-block
  static constexpr int kSlotBytes = XW_PART_TOK * kTokRow;        // one token box's slot
  static constexpr int kParts = MB == 64 ? 2 : 1;                 // parts per stage
  // stage: [desc hi | desc lo | part boxes (| the second part's boxes, MB = 64)].  Every token box starts 1024-byte
  // aligned (the 128-byte swizzle's atom).
  static constexpr int kTokOff = 2 * kDescBytes;
  static constexpr int kStageBytes = kTokOff + kParts * kBoxes * kSlotBytes;
  static constexpr int kStages = MB == 64 ? 5 : 6;
  // after the ring and its barriers: one epilogue staging tile per consumer warp (its 16 maps x 32 part tokens)
  static constexpr int kBarBytes = 256;
  static constexpr int kEpiBytes = 8 * XW_EPI_ROWS * XW_EPI_PITCH * 4;
  static constexpr int kSmem = kStages * kStageBytes + 1024 + kBarBytes + kEpiBytes;
  static_assert(2 * kStages * 8 <= kBarBytes, "barriers");
  static_assert(kSmem <= 227 * 1024, "shared-memory ring too large");
  static_assert(kTokOff % 1024 == 0 && kSlotBytes % 1024 == 0 && kStageBytes % 1024 == 0,
                "token boxes must start 1024-byte aligned");
};

// A cell's extent and its parts.  Null box_ext: the whole 21 x 21 box.  An extent outside the box skips the cell.
template <int MB>
struct XwExt {
  int y, x, bh, bw, n;   // first box row / column, rows, columns, parts
  XwExt() = default;
  __device__ __forceinline__ XwExt(const int4* __restrict__ box_ext, int cell) {
    const int4 e = box_ext ? __ldg(box_ext + cell) : make_int4(0, 0, XW_BOX, XW_BOX);
    y = e.x; x = e.y; bh = e.z; bw = e.w;
    const int rp = XW_PART_TOK / max(bw, 1);
    n = ok() ? (bh + rp - 1) / rp : 0;
    if (MB == 64) n += n & 1;   // whole pairs
  }
  __device__ __forceinline__ bool ok() const {
    return y >= 0 && x >= 0 && bh >= XW_EXT_MIN && bw >= XW_EXT_MIN && y + bh <= XW_BOX && x + bw <= XW_BOX;
  }
  // part i: rows bh / n, one more for the first bh % n parts (so <= ceil(bh / n) <= rp rows, >= 1 since n <= 8 < bh)
  __device__ __forceinline__ int rows(int i) const { return bh / n + (i < bh % n ? 1 : 0); }
  __device__ __forceinline__ int row(int i) const { return y + i * (bh / n) + min(i, bh % n); }   // its first box row
};

// One part of a cell on one consumer warpgroup: the K loop over the ring, then rows [r0, r0 + 64) of the cell x the part's
// ntok tokens (rows of bw, from box column col0 = xw_col(first row, first column)) into xbox.  d_off / t_off: byte offsets
// of the warpgroup's descriptor rows / the part's token box(es) in a stage, t_half: distance from a token box's hi half to
// its lo half (separate halves only).
template <int MB, bool HILO>
__device__ __forceinline__ void xw_part(uint8_t* smem, uint64_t* full, uint64_t* empty, float* epi, int& stage, int& phase, int KB,
                                        uint32_t d_off, uint32_t t_off, uint32_t t_half, float* __restrict__ xbox, int map0,
                                        int r0, int m, int ntok, int bw, int col0) {
  using Cfg = XwCfg<MB, HILO>;
  constexpr int N = XW_PART_TOK;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, t = threadIdx.x & 127;
  float acc[N / 2];
#pragma unroll
  for (int i = 0; i < N / 2; ++i) acc[i] = 0.f;
  int prev = -1;
  for (int kb = 0; kb < KB; ++kb) {
    tc::mbar_wait(&full[stage], phase);
    tc::wgmma_fence();
    const uint32_t sd = tc::smem_u32(smem + stage * Cfg::kStageBytes) + d_off;
    const uint32_t st = tc::smem_u32(smem + stage * Cfg::kStageBytes) + t_off;
#pragma unroll
    for (int ks = 0; ks < Cfg::kBK / 16; ++ks) {
      const uint32_t koff = ks * 32;
      const uint64_t d_hi = tc::smem_desc_sw64(sd + koff), d_lo = tc::smem_desc_sw64(sd + Cfg::kDescBytes + koff);
      const uint64_t t_hi = HILO ? tc::smem_desc_sw128(st + koff) : tc::smem_desc_sw64(st + koff);
      const uint64_t t_lo = HILO ? tc::smem_desc_sw128(st + Cfg::kRow + koff) : tc::smem_desc_sw64(st + t_half + koff);
      tc::wgmma_ss<false, N>(acc, d_lo, t_hi, 1u);   // desc_lo * tok_hi, desc_hi * tok_lo, desc_hi * tok_hi:
      tc::wgmma_ss<false, N>(acc, d_hi, t_lo, 1u);   // the product order of tc_gemm_kernel (F16X3)
      tc::wgmma_ss<false, N>(acc, d_hi, t_hi, 1u);
    }
    tc::wgmma_commit();
    tc::wgmma_wait<1>();
    if (prev >= 0 && t == 0) tc::mbar_arrive(&empty[prev]);
    prev = stage;
    if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
  }
  tc::wgmma_wait<0>();
  tc::reg_fence(acc);
  if (prev >= 0 && t == 0) tc::mbar_arrive(&empty[prev]);
  // Fragment rows are maps, columns part tokens: acc[4 i + 2 h + {0, 1}] = map rw + fr + 8 h, tokens 8 i + fc + {0, 1}
  // (rw = the warp's first row).  Stored straight from the fragment, every warp store would write 4 lanes' values of 8
  // maps, half of each 32-byte sector; the partial sectors held a part's epilogue at about a quarter of a cell's time
  // with the ring idle (DESIGN.md 4.3).  So each warp passes its 16 maps through shared memory 32 tokens at a time, and
  // lane l stores token 32 q + l of one map per store: runs of bw consecutive floats.
  const int rw = r0 + (warp & 3) * 16, fr = lane >> 2, fc = 2 * (lane & 3);
  float* buf = epi + (warp & 7) * XW_EPI_ROWS * XW_EPI_PITCH;
  float* dst = xbox + (size_t)(map0 + rw) * XW_COLS + col0;
  const int nr = min(m - rw, XW_EPI_ROWS);   // the warp's maps (<= 0: none)
#pragma unroll
  for (int q = 0; q < N / 32; ++q) {
    if (32 * q >= ntok || nr <= 0) break;
#pragma unroll
    for (int ii = 0; ii < 4; ++ii)
#pragma unroll
      for (int h = 0; h < 2; ++h)
        *reinterpret_cast<float2*>(buf + (fr + 8 * h) * XW_EPI_PITCH + 8 * ii + fc) =
            make_float2(acc[4 * (4 * q + ii) + 2 * h], acc[4 * (4 * q + ii) + 2 * h + 1]);
    __syncwarp();
    const int j = 32 * q + lane, y = j / bw, off = y * XW_BOX + (j - y * bw);
    if (j < ntok)
      for (int k = 0; k < nr; ++k) dst[(size_t)k * XW_COLS + off] = buf[k * XW_EPI_PITCH + lane];
    __syncwarp();
  }
}

template <int MB, bool HILO>
__global__ void __launch_bounds__(TC_THREADS, 1)
xw_gemm_kernel(const __grid_constant__ CUtensorMap tmD_hi, const __grid_constant__ CUtensorMap tmD_lo,
               const __grid_constant__ XwTokMaps<HILO> tok, XwCells cells, const int2* __restrict__ box_org,
               const int4* __restrict__ box_ext, float* __restrict__ xbox, int K) {
  using Cfg = XwCfg<MB, HILO>;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t* full = reinterpret_cast<uint64_t*>(smem + Cfg::kStages * Cfg::kStageBytes);   // [kStages]
  uint64_t* empty = full + Cfg::kStages;                                                    // [kStages]
  float* epi = reinterpret_cast<float*>(smem + Cfg::kStages * Cfg::kStageBytes + Cfg::kBarBytes);

  const int warp = threadIdx.x >> 5, wg = threadIdx.x >> 7;
  const int KB = (K + Cfg::kBK - 1) / Cfg::kBK;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&tmD_hi); tc::prefetch_tmap(&tmD_lo);
    for (int s = 0; s < Cfg::kStages; ++s) { tc::mbar_init(&full[s], 1); tc::mbar_init(&empty[s], 2); }   // 2 consumer warpgroups
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (wg == 0) {
    // ===================== TMA producer =====================
    tc::regs_dealloc<40>();
    if (warp == 0 && tc::elect_one()) {
      int stage = 0, phase = 0;
      for (int cell = blockIdx.x; cell < cells.n_cells; cell += gridDim.x) {
        const int2 org = box_org[cell];
        if (org.y == INT_MIN) continue;            // every map of the cell takes the full-map path
        const XwExt<MB> e(box_ext, cell);
        const int drow = cells.arow[cell], frame = cells.frame[cell], col = org.y + e.x;   // first grid column
        const int wi = e.bw - XW_EXT_MIN;
        for (int p0 = 0; p0 < e.n; p0 += Cfg::kParts) {
          int tok_rows = 0;   // token rows of the stage's box(es)
          for (int q = 0; q < Cfg::kParts; ++q) tok_rows += e.rows(p0 + q) * e.bw;
          for (int kb = 0; kb < KB; ++kb) {
            const int k0 = kb * Cfg::kBK, kt = HILO ? 2 * k0 : k0;   // channel / token-row element of the K block
            tc::mbar_wait(&empty[stage], phase ^ 1);
            uint8_t* st = smem + stage * Cfg::kStageBytes;
            tc::mbar_expect_tx(&full[stage], 2 * Cfg::kDescBytes + Cfg::kBoxes * tok_rows * Cfg::kTokRow);
            for (int q = 0; q < Cfg::kParts; ++q) {
              uint8_t* s = st + Cfg::kTokOff + q * Cfg::kBoxes * Cfg::kSlotBytes;
              const int ri = e.rows(p0 + q) - 1, row = org.x + e.row(p0 + q);
              tc::tma_load_4d(&tok.m[0][wi][ri], &full[stage], s, kt, col, row, frame);
              if constexpr (!HILO) tc::tma_load_4d(&tok.m[1][wi][ri], &full[stage], s + Cfg::kSlotBytes, kt, col, row, frame);
            }
            tc::tma_load_2d(&tmD_hi, &full[stage], st, k0, drow);
            tc::tma_load_2d(&tmD_lo, &full[stage], st + Cfg::kDescBytes, k0, drow);
            if (++stage == Cfg::kStages) { stage = 0; phase ^= 1; }
          }
        }
      }
    }
  } else {
    // ===================== MMA + epilogue =====================
    tc::regs_alloc<232>();
    const int cw = wg - 1;
    int stage = 0, phase = 0;
    // a cell's description is loaded one cell ahead: its loads land while the cell before it runs, not between the two
    struct Meta { bool skip; XwExt<MB> e; int m, map0; };
    auto meta = [&](int cell) {
      return Meta{box_org[cell].y == INT_MIN, XwExt<MB>(box_ext, cell), cells.m[cell], cells.row0[cell]};
    };
    Meta cur;
    if (blockIdx.x < cells.n_cells) cur = meta(blockIdx.x);
    for (int cell = blockIdx.x; cell < cells.n_cells; cell += gridDim.x) {
      Meta nxt;
      if (cell + gridDim.x < cells.n_cells) nxt = meta(cell + gridDim.x);
      const XwExt<MB>& e = cur.e;
      const int m = cur.m, map0 = cur.map0;
      if (!cur.skip)
        for (int p0 = 0; p0 < e.n; p0 += Cfg::kParts) {
          if constexpr (MB == 64) {   // warpgroup cw: part p0 + cw of the pair, all 64 descriptor rows
            const int p = p0 + cw;
            xw_part<MB, HILO>(smem, full, empty, epi, stage, phase, KB, 0, Cfg::kTokOff + cw * Cfg::kBoxes * Cfg::kSlotBytes,
                              Cfg::kSlotBytes, xbox, map0, 0, m, e.rows(p) * e.bw, e.bw, xw_col(e.row(p), e.x));
          } else {                    // warpgroup cw: descriptor rows [64 cw, 64 cw + 64) of part p0
            xw_part<MB, HILO>(smem, full, empty, epi, stage, phase, KB, cw * 64 * Cfg::kRow, Cfg::kTokOff, Cfg::kSlotBytes,
                              xbox, map0, 64 * cw, m, e.rows(p0) * e.bw, e.bw, xw_col(e.row(p0), e.x));
          }
        }
      cur = nxt;
    }
  }
}

// The token boxes' tensor maps of a feature view, encoded once per (tensor, shape) and kept for the following launches
// (a chunk's launch would otherwise encode up to 112 maps).  One entry per device: it is rebuilt when the features change.
template <bool HILO>
static int xw_tok_maps(const FeatView& fv, const dinotrk_geom& g, const XwTokMaps<HILO>*& out) {
  struct Entry { const void* base[2]; uint64_t dims[4]; bool valid; XwTokMaps<HILO> maps; };
  static PerDev<Entry> cache;
  Entry& e = cache.get();
  const void* base[2] = {HILO ? fv.hilo : fv.hi, HILO ? nullptr : fv.lo};
  const uint64_t row = HILO ? (uint64_t)hilo_row(fv.C) : (uint64_t)fv.C;   // fp16 elements per token row
  const uint64_t dims[4] = {row, (uint64_t)g.w, (uint64_t)g.h, (uint64_t)fv.T};
  if (!e.valid || memcmp(e.base, base, sizeof(base)) != 0 || memcmp(e.dims, dims, sizeof(dims)) != 0) {
    e.valid = false;
    const uint64_t strides[3] = {row * 2, (uint64_t)g.w * row * 2, (uint64_t)fv.P * row * 2};
    constexpr int BK = XwCfg<64, HILO>::kBK;
    const uint32_t ib = HILO ? 2 * BK : BK, tsw = HILO ? 128 : 2 * BK;
    for (int o = 0; o < (HILO ? 1 : 2); ++o)
      for (int wi = 0; wi < XW_NW; ++wi)
        for (int ri = 0; ri < XW_PART_ROWS; ++ri) {
          const uint32_t box[4] = {ib, (uint32_t)(XW_EXT_MIN + wi), (uint32_t)(1 + ri), 1};
          if (int rc = make_tmap_4d(&e.maps.m[o][wi][ri], base[o], dims, strides, box, TMAP_F16, tsw)) return rc;
        }
    memcpy(e.base, base, sizeof(base));
    memcpy(e.dims, dims, sizeof(dims));
    e.valid = true;
  }
  out = &e.maps;
  return DINOTRK_OK;
}

template <int MB, bool HILO>
static int run_xw_gemm(const FeatView& fv, const dinotrk_geom& g, const CUtensorMap (&tmD)[2], const XwCells& cells,
                       const XwChunk& xc, cudaStream_t st) {
  const XwTokMaps<HILO>* tok;
  if (int rc = xw_tok_maps<HILO>(fv, g, tok)) return rc;
  static PerDev<bool> attr_dev;
  bool& attr = attr_dev.get();
  if (!attr) {
    DTK_CUDA(cudaFuncSetAttribute(xw_gemm_kernel<MB, HILO>, cudaFuncAttributeMaxDynamicSharedMemorySize, XwCfg<MB, HILO>::kSmem));
    attr = true;
  }
  const int sms = num_sms();
  const int grid = cells.n_cells < sms ? cells.n_cells : sms;
  ProfRange pr(PROF_XW_GEMM, st);
  xw_gemm_kernel<MB, HILO><<<grid, TC_THREADS, XwCfg<MB, HILO>::kSmem, st>>>(tmD[0], tmD[1], *tok, cells, xc.box_org, xc.box_ext,
                                                                              xc.xbox, fv.C);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int launch_xw_gemm(const FeatView& fv, const dinotrk_geom& g, const void* desc_hi, const void* desc_lo, int desc_rows,
                   const XwCells& cells, const XwChunk& xc, cudaStream_t st) {
  if (cells.n_cells <= 0) return DINOTRK_OK;
  DTK_CHECK_ARG(fv.C % 8 == 0 && cells.max_m <= XW_MAX_CELL, "exact-window GEMM: bad sizes");
  const bool small = cells.max_m <= 64, hilo = fv.hilo != nullptr;
  constexpr int BK = XwCfg<64, false>::kBK, SW = 2 * BK;   // 32-channel K blocks; descriptors in 64-byte swizzle
  CUtensorMap tmD[2];   // desc hi, desc lo
  int rc;
  if ((rc = make_tmap_2d(&tmD[0], desc_hi, desc_rows, fv.C, small ? 64 : 128, BK, TMAP_F16, 0, SW))) return rc;
  if ((rc = make_tmap_2d(&tmD[1], desc_lo, desc_rows, fv.C, small ? 64 : 128, BK, TMAP_F16, 0, SW))) return rc;
  if (hilo) return small ? run_xw_gemm<64, true>(fv, g, tmD, cells, xc, st) : run_xw_gemm<128, true>(fv, g, tmD, cells, xc, st);
  return small ? run_xw_gemm<64, false>(fv, g, tmD, cells, xc, st) : run_xw_gemm<128, false>(fv, g, tmD, cells, xc, st);
}

// ====================================================================================================== 4. head
// One kernel, two maps per warp: half-warp hf (lanes 16 hf .. 16 hf + 15) owns map 2 pair + hf, and its lane l is refiner
// channel l.  Per map:
//   window   exact values v = relu(acc / max(|d| |F|, 1e-8)) (the full-map GEMM's epilogue expression, corr_cos) formed from
//            xbox's raw accumulators at the candidates (-> exact first arg-max) and on the 15 x 15 window (lane l: window
//            column l), which goes to shared memory, with m_out = max(exact window values outside the 7 x 7 core,
//                                                                  per tile: (its max token inside the core ? second value : max) + eps).
//            Before the current pair is refined, the warp runs the next pair's arg-max chain: three levels of dependent
//            loads (state, cell, norm, candidates, eps and tile keys; box origin and frame; the values at the candidates),
//            which it waits for.  Only the window's 2 x 15 loads per lane (cp.async into shared memory) land while the
//            current pair is refined.
//   refiner  lane = channel c.  Hidden row j (13 values of channel c, from three window rows read as broadcasts) stays in
//            registers and goes at once into the three logit rows it is a tap row of: chain A0 of row j, A1 of row j - 1
//            (whose A0 + A1 is then complete) and A2 of row j - 2 (whose per-channel logit is then complete).  Every lane
//            works on every row, and no hidden window is stored.  The 16 channels' contributions to a finished logit row
//            meet in shared memory, where lane x adds them up in the tree of the pair-lane layout: (c, c + 8) first, then
//            the pair sums xor 4, xor 2, xor 1.
//   tail     softmax sums on the 11 x 11 box, the certificate of head.cuh, and either the track point or a place in the
//            group's full-map queue.
// Every hidden value, logit and softmax sum is the same sequence of fp32 operations as in the refiner's first form
// (xw_refine): relu((a0 + a1) + a2) with a0 an FMA chain from b1 and a1, a2 chains from a product, taps in (ky, kx) order.
constexpr int XH_WARPS = 8;
constexpr int XH_WP = 16;       // window row pitch (floats): 15 values and a zero
constexpr int XH_WIN = WM * XH_WP;   // 240 floats per map; 240 = 16 mod 32: the two maps' window rows lie in disjoint banks
constexpr int XH_RP = 20;       // row pitch of a channel-sum buffer: 8 lanes' 16-byte reads of consecutive rows hit distinct banks
constexpr int XH_RED = 240;     // one logit row's 11 x 16 channel contributions of one map (11 x 20, padded to 16 mod 32)
constexpr int XH_ZB = 128;      // the 121 logits of one map
// per warp: [windows: 2 maps | channel sums: 2 buffers x 2 maps | logits: 2 maps | gathered accumulators: 2 maps |
// gathered token norms: 2 maps]
constexpr int XH_RAW = 2 * XH_WIN + 4 * XH_RED + 2 * XH_ZB;
constexpr int XH_PER_WARP = XH_RAW + 4 * XH_WIN;
constexpr int XH_SMEM = XH_WARPS * XH_PER_WARP * 4;
static_assert(XH_WIN % 32 == 16 && XH_RED % 32 == 16 && WB * XH_RP <= XH_RED && WB * WB <= XH_ZB, "head buffer layout");

constexpr int XH_KEYS = 4;      // tile keys per lane loaded with the map's first loads (all of them up to 64 tiles)

struct XhGather {       // one map's gathers, lane l of its half-warp
  int amax;             // exact first arg-max token; -1: no map, or a map the plan queued
  float dn, mout;       // descriptor norm; the lane's share of m_out from the tile keys
  unsigned ok;          // bit y: window row y, column l lies inside the token grid
};

// 4-byte asynchronous copy global -> shared: a gathered value lands without holding a register while the pair before it
// is refined
__device__ __forceinline__ void xh_cp4(float* dst, const float* src) {
  asm volatile("cp.async.ca.shared.global [%0], [%1], 4;\n" ::"r"((unsigned)__cvta_generic_to_shared(dst)), "l"(src) : "memory");
}
__device__ __forceinline__ void xh_cp_wait() { asm volatile("cp.async.wait_all;\n" ::: "memory"); }

__device__ __forceinline__ void xh_gather(XhGather& gt, int map, int n_maps, int l, int h, int w, int P, int n_tiles,
                                          const float* __restrict__ norms, const float* __restrict__ desc_norm,
                                          const int* __restrict__ cell_frame, const int* __restrict__ cell_of,
                                          const int2* __restrict__ box_org, const int* __restrict__ stat,
                                          const int* __restrict__ cand, const unsigned long long* __restrict__ key1,
                                          const float* __restrict__ max2, const float* __restrict__ xbox,
                                          const float* __restrict__ eps_map, float* __restrict__ racc, float* __restrict__ rfn) {
  gt.amax = -1;
  gt.ok = 0;
  if (map >= n_maps) return;
  // The chain has three levels of dependent loads; everything that depends only on the map index is issued at the first:
  // the state, the cell, the norm, the candidates, eps and the tile keys of the first 16 XH_KEYS tiles.
  const int st = __ldg(stat + map), cell = __ldg(cell_of + map);
  const float dn = __ldg(desc_norm + map);
  const int4 cd = __ldg(reinterpret_cast<const int4*>(cand) + map);
  const float eps = eps_map ? __ldg(eps_map + map) : XW_EPS;
  const unsigned long long* k1 = key1 + (size_t)map * n_tiles;
  const float* k2 = max2 + (size_t)map * n_tiles;
  unsigned long long kk[XH_KEYS];
  float kv2[XH_KEYS];
#pragma unroll
  for (int q = 0; q < XH_KEYS; ++q) {
    const int t = l + 16 * q;
    kk[q] = t < n_tiles ? __ldg(k1 + t) : 0ull;
    kv2[q] = t < n_tiles ? __ldg(k2 + t) : 0.f;
  }
  if (st != 0) return;
  const int2 org = __ldg(box_org + cell);
  const float* fn = norms + (size_t)__ldg(cell_frame + cell) * P;
  const float* xr = xbox + (size_t)map * XW_COLS;
  // exact first arg-max among the candidates (every lane, redundantly: <= 4 loads)
  const int ct[4] = {cd.x, cd.y, cd.z, cd.w};
  float best = -1.f;
  int amax = -1;
#pragma unroll
  for (int q = 0; q < XW_MAX_CAND; ++q)
    if (ct[q] >= 0) {
      const int tr = ct[q] / w, tcn = ct[q] - tr * w;
      const float v = fmaxf(corr_cos(__ldg(xr + xw_col(tr - org.x, tcn - org.y)), dn, __ldg(fn + ct[q])), 0.f);
      if (v > best || (v == best && ct[q] < amax)) { best = v; amax = ct[q]; }
    }
  const int arow = amax / w, acol = amax - arow * w;
  // coarse bound on everything outside the window, from the tile keys
  float mout = 0.f;
  auto fold = [&](unsigned long long k, float m2) {
    const int tk = 0x7fffffff - (int)(k & 0xffffffffu);
    const int tr = tk / w, tcn = tk - tr * w;
    const bool in_core = abs(tr - arow) <= 3 && abs(tcn - acol) <= 3;
    mout = fmaxf(mout, (in_core ? m2 : __uint_as_float((unsigned)(k >> 32))) + eps);
  };
#pragma unroll
  for (int q = 0; q < XH_KEYS; ++q)
    if (l + 16 * q < n_tiles) fold(kk[q], kv2[q]);
  for (int t = l + 16 * XH_KEYS; t < n_tiles; t += 16) fold(__ldg(k1 + t), __ldg(k2 + t));
  // window column l: raw accumulators and token norms to racc / rfn (row y at y XH_WP + l), read when the pair is refined
  const int c = acol - 7 + l;
  const bool col_in = l < WM && c >= 0 && c < w;
  unsigned ok = 0;
#pragma unroll
  for (int y = 0; y < WM; ++y) {
    const int r = arow - 7 + y;
    if (col_in && r >= 0 && r < h) {
      xh_cp4(racc + y * XH_WP + l, xr + xw_col(r - org.x, c - org.y));
      xh_cp4(rfn + y * XH_WP + l, fn + r * w + c);
      ok |= 1u << y;
    }
  }
  gt.amax = amax;
  gt.dn = dn;
  gt.mout = mout;
  gt.ok = ok;
}

// Exact window column l into shared memory (zero outside the map) from the lane's gathers; returns its share of m_out.
__device__ __forceinline__ float xh_window(const XhGather& gt, const float* __restrict__ racc, const float* __restrict__ rfn,
                                           float* __restrict__ win, int l) {
  xh_cp_wait();
  float mout = gt.mout;
#pragma unroll
  for (int y = 0; y < WM; ++y) {
    float v = 0.f;
    if ((gt.ok >> y) & 1u) {
      v = fmaxf(corr_cos(racc[y * XH_WP + l], gt.dn, rfn[y * XH_WP + l]), 0.f);
      if (!(abs(y - 7) <= 3 && abs(l - 7) <= 3)) mout = fmaxf(mout, v);
    }
    win[y * XH_WP + l] = v;
  }
  return mout;
}

// k-th tap row (ky) chain of a 3-tap kernel row over three consecutive values: a product, then two FMAs
__device__ __forceinline__ float xh_tap3(const float* wk, float v0, float v1, float v2) {
  return __fmaf_rn(wk[2], v2, __fmaf_rn(wk[1], v1, __fmul_rn(wk[0], v0)));
}

// Hidden row j of channel l, and what it completes: in A0in / Sin the A0 chains of logit row j - 1 and the A0 + A1 sums
// of row j - 2; out A0out / Sout those of rows j and j - 1; the logits of row j - 2 go to zb.  red: this half's first
// channel-sum buffer (the second lies 2 XH_RED further; rows alternate between them, so one warp barrier per row suffices).
template <bool INTERIOR>
__device__ __forceinline__ void xh_step(int j, const float (&A0in)[WB], const float (&Sin)[WB], float (&A0out)[WB],
                                        float (&Sout)[WB], const float* __restrict__ win, float* __restrict__ red,
                                        float* __restrict__ zb, const float (&w1)[9], float b1, const float (&w2)[9], float b2,
                                        bool row_in, unsigned cmask, int l) {
  float in[3][16];
#pragma unroll
  for (int ky = 0; ky < 3; ++ky)
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const float4 v = *reinterpret_cast<const float4*>(win + (j + ky) * XH_WP + 4 * q);
      in[ky][4 * q] = v.x; in[ky][4 * q + 1] = v.y; in[ky][4 * q + 2] = v.z; in[ky][4 * q + 3] = v.w;
    }
  float hr[WH];
#pragma unroll
  for (int x = 0; x < WH; ++x) {
    // three short chains per output (one per input row) instead of one chain of nine dependent FMAs
    float a0 = __fmaf_rn(w1[0], in[0][x], b1), a1 = __fmul_rn(w1[3], in[1][x]), a2 = __fmul_rn(w1[6], in[2][x]);
    a0 = __fmaf_rn(w1[1], in[0][x + 1], a0); a1 = __fmaf_rn(w1[4], in[1][x + 1], a1); a2 = __fmaf_rn(w1[7], in[2][x + 1], a2);
    a0 = __fmaf_rn(w1[2], in[0][x + 2], a0); a1 = __fmaf_rn(w1[5], in[1][x + 2], a1); a2 = __fmaf_rn(w1[8], in[2][x + 2], a2);
    const float a = __fadd_rn(__fadd_rn(a0, a1), a2);
    hr[x] = INTERIOR || (row_in && ((cmask >> x) & 1u)) ? fmaxf(a, 0.f) : 0.f;
  }
  if (j < WB) {
#pragma unroll
    for (int x = 0; x < WB; ++x) A0out[x] = xh_tap3(w2, hr[x], hr[x + 1], hr[x + 2]);
  }
  if (j >= 1 && j <= WB) {
#pragma unroll
    for (int x = 0; x < WB; ++x) Sout[x] = __fadd_rn(A0in[x], xh_tap3(w2 + 3, hr[x], hr[x + 1], hr[x + 2]));
  }
  if (j >= 2) {
    float* rb = red + (j & 1) * (2 * XH_RED);
#pragma unroll
    for (int x = 0; x < WB; ++x) rb[x * XH_RP + l] = __fadd_rn(Sin[x], xh_tap3(w2 + 6, hr[x], hr[x + 1], hr[x + 2]));
    __syncwarp();
    if (l < WB) {
      float p[16];
#pragma unroll
      for (int q = 0; q < 4; ++q) {
        const float4 v = *reinterpret_cast<const float4*>(rb + l * XH_RP + 4 * q);
        p[4 * q] = v.x; p[4 * q + 1] = v.y; p[4 * q + 2] = v.z; p[4 * q + 3] = v.w;
      }
      float v[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) v[i] = __fadd_rn(p[i], p[i + 8]);
      const float t = __fadd_rn(__fadd_rn(__fadd_rn(v[0], v[4]), __fadd_rn(v[2], v[6])),
                                __fadd_rn(__fadd_rn(v[1], v[5]), __fadd_rn(v[3], v[7])));
      zb[(j - 2) * WB + l] = __fadd_rn(t, b2);
    }
  }
}

// Refiner of one map per half-warp: the 121 logits into zb.  INTERIOR: both maps' 15 x 15 windows lie inside the token
// grid (no hidden value is forced to zero -- the common case away from the frame border).
template <bool INTERIOR>
__device__ __forceinline__ void xh_refine(const float* __restrict__ win, float* __restrict__ red, float* __restrict__ zb,
                                          const float (&w1)[9], float b1, const float (&w2)[9], float b2, int arow, int acol,
                                          int h, int w, int l) {
  unsigned cmask = 0;
#pragma unroll
  for (int x = 0; x < WH; ++x) cmask |= (acol - 6 + x >= 0 && acol - 6 + x < w) ? 1u << x : 0u;
  float A0a[WB], Sa[WB], A0b[WB], Sb[WB];
#pragma unroll
  for (int x = 0; x < WB; ++x) { A0a[x] = 0.f; Sa[x] = 0.f; }
#pragma unroll 1
  for (int j = 0; j < WH; j += 2) {
    xh_step<INTERIOR>(j, A0a, Sa, A0b, Sb, win, red, zb, w1, b1, w2, b2, arow - 6 + j >= 0 && arow - 6 + j < h, cmask, l);
    if (j + 1 < WH)
      xh_step<INTERIOR>(j + 1, A0b, Sb, A0a, Sa, win, red, zb, w1, b1, w2, b2, arow - 5 + j >= 0 && arow - 5 + j < h, cmask, l);
  }
}

// Softmax sums on the box / the disc.  Lane l takes pixels l + 16 k: even k are the pixels l + 32 q lane l of a whole warp
// would take, odd k lane l + 16's, each in its own accumulator; adding the two is the xor-16 step of warp_sum, and the
// xor 8 .. 1 steps follow -- the sums of the one-map-per-warp form, bit for bit.
__device__ __forceinline__ void xh_sums(const HeadParams& hp, const float* __restrict__ zb, int arow, int acol, int l,
                                        float& zmax, float (&tot)[5]) {
  float z[8];
  bool valid[8];
  zmax = -INFINITY;
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int p = l + 16 * k;
    const int y = p / WB, x = p - y * WB, r = arow - 5 + y, c = acol - 5 + x;
    valid[k] = p < WB * WB && r >= 0 && r < hp.h && c >= 0 && c < hp.w;
    z[k] = valid[k] ? zb[p] : -INFINITY;
    zmax = fmaxf(zmax, z[k]);
  }
#pragma unroll
  for (int o = 8; o > 0; o >>= 1) zmax = fmaxf(zmax, __shfl_xor_sync(0xffffffffu, zmax, o));
  float s[2][5] = {};
#pragma unroll
  for (int k = 0; k < 8; ++k) {
    const int p = l + 16 * k;
    const int y = p / WB, x = p - y * WB, r = arow - 5 + y, c = acol - 5 + x;
    const float e = valid[k] ? expf(z[k] - zmax) : 0.f;
    float (&t)[5] = s[k & 1];
    t[0] += e;
    if (valid[k] && in_disc(hp, r, c, arow, acol)) {
      t[1] += e; t[2] = fmaf(token_px(hp, c), e, t[2]); t[3] = fmaf(token_px(hp, r), e, t[3]);
    }
    t[4] += valid[k] ? 1.f : 0.f;
  }
#pragma unroll
  for (int i = 0; i < 5; ++i) {
    float v = s[0][i] + s[1][i];
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    tot[i] = v;
  }
}

// REFINE = false: the window part alone (arg-max, window, m_out; m_out goes to the map's output x), which only
// tools/bench_xw_head.py --split runs, to time the two parts of the kernel apart
template <bool REFINE>
__global__ void __launch_bounds__(XH_WARPS * 32, 2)
xw_head_kernel(int n_maps, HeadParams hp, dinotrk_head_weights wts, int n_tiles, const float* __restrict__ norms,
               const float* __restrict__ desc_norm, const int* __restrict__ cell_frame, const int* __restrict__ cell_group,
               const int* __restrict__ cell_of, const int2* __restrict__ box_org, const int* __restrict__ stat,
               const int* __restrict__ cand, const unsigned long long* __restrict__ key1, const float* __restrict__ max2,
               const float* __restrict__ xbox, const float* __restrict__ eps_map, const int* __restrict__ grp_map0,
               const int* __restrict__ out_index, float* __restrict__ out, int* __restrict__ slow_cnt,
               int* __restrict__ slow_list, int n_groups) {
  extern __shared__ __align__(16) float xh_smem[];
  // (the warp index through a shuffle: the compiler then knows that everything derived from it -- the pair index, the
  // loop trip count, the branches on the pair's state -- is warp-uniform and keeps the shuffles plain SHFLs)
  const int lane = threadIdx.x & 31, wid = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0);
  const int hf = lane >> 4, l = lane & 15;
  float* ws = xh_smem + wid * XH_PER_WARP;
  float* win = ws + hf * XH_WIN;
  float* red = ws + 2 * XH_WIN + hf * XH_RED;
  float* zb = ws + 2 * XH_WIN + 4 * XH_RED + hf * XH_ZB;
  float* racc = ws + XH_RAW + hf * XH_WIN;
  float* rfn = racc + 2 * XH_WIN;
  float w1[9], w2[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) { w1[k] = wts.w1[l][k]; w2[k] = wts.w2[l][k]; }
  const float b1 = wts.b1[l];
  const int h = hp.h, w = hp.w;
  const int n_pairs = (n_maps + 1) >> 1, stride = gridDim.x * XH_WARPS;

  int pair = blockIdx.x * XH_WARPS + wid;
  XhGather gt;
  if (pair < n_pairs)
    xh_gather(gt, 2 * pair + hf, n_maps, l, h, w, hp.P, n_tiles, norms, desc_norm, cell_frame, cell_of, box_org, stat, cand,
              key1, max2, xbox, eps_map, racc, rfn);
  for (; pair < n_pairs; pair += stride) {
    const int map = 2 * pair + hf, amax = gt.amax;
    const bool exact = amax >= 0;
    const int arow = exact ? amax / w : 7, acol = exact ? amax - arow * w : 7;
    float mout = xh_window(gt, racc, rfn, win, l);
#pragma unroll
    for (int o = 8; o > 0; o >>= 1) mout = fmaxf(mout, __shfl_xor_sync(0xffffffffu, mout, o));
    const bool any = __any_sync(0xffffffffu, exact);
    const bool interior = __all_sync(0xffffffffu, !exact || (arow >= 7 && arow + 7 < h && acol >= 7 && acol + 7 < w));
    if (pair + stride < n_pairs)   // the next pair's arg-max chain; its window's loads land while this pair is refined
      xh_gather(gt, 2 * (pair + stride) + hf, n_maps, l, h, w, hp.P, n_tiles, norms, desc_norm, cell_frame, cell_of, box_org,
                stat, cand, key1, max2, xbox, eps_map, racc, rfn);
    __syncwarp();
    if constexpr (!REFINE) {
      if (l == 0 && exact) out[(size_t)(out_index ? out_index[map] : map) * hp.out_stride] = mout;
      continue;
    }
    float zmax = 0.f;
    float tot[5] = {0.f, 0.f, 0.f, 0.f, 0.f};
    if (any) {
      if (interior) xh_refine<true>(win, red, zb, w1, b1, w2, wts.b2, arow, acol, h, w, l);
      else xh_refine<false>(win, red, zb, w1, b1, w2, wts.b2, arow, acol, h, w, l);
      __syncwarp();
      xh_sums(hp, zb, arow, acol, l, zmax, tot);
    }
    if (l == 0 && map < n_maps) {
      if (exact && head_certified(hp, wts, mout, zmax, tot)) {
        head_store_point(hp, __fdiv_rn(tot[2], tot[1]), __fdiv_rn(tot[3], tot[1]), out_index, out, map);
      } else {
        const int g = cell_group[cell_of[map]];
        const int pos = atomicAdd(slow_cnt + g, 1);
        slow_list[grp_map0[g] + pos] = map;
        atomicAdd(slow_cnt + n_groups, 1);
        if (exact) atomicAdd(slow_cnt + n_groups + 1, 1);   // (statistics: queued by the certificate, not by the plan)
      }
    }
    __syncwarp();
  }
}

static int g_xw_head_window_only = 0;   // dinotrk_xw_head_set_window_only

int launch_xw_head(const FeatView& fv, const dinotrk_geom& g, const dinotrk_head_weights& hw, const XwCells& cells,
                   const float* desc_norm, const int* grp_map0, int n_maps, const int* out_index, float* out, int out_stride,
                   int out_mode, const XwChunk& xc, cudaStream_t st, int n_groups, const float* eps) {
  if (n_maps <= 0) return DINOTRK_OK;
  DTK_CHECK_ARG(disc_fits_box(g), "exact-window path: disc radius %d exceeds 5 tokens", g.radius);
  const HeadParams hp = make_head_params(g, hw, dinotrk_map_stride(&g), out_stride, out_mode);
  const int sms = num_sms();
  int grid = cdiv(cdiv(n_maps, 2), XH_WARPS);
  if (grid > sms * 2) grid = sms * 2;
  static PerDev<bool> attr_dev;
  bool& attr = attr_dev.get();
  if (!attr) {
    DTK_CUDA(cudaFuncSetAttribute(xw_head_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, XH_SMEM));
    DTK_CUDA(cudaFuncSetAttribute(xw_head_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, XH_SMEM));
    attr = true;
  }
  ProfRange pr(PROF_XW_HEAD, st);
  (g_xw_head_window_only ? xw_head_kernel<false> : xw_head_kernel<true>)<<<grid, XH_WARPS * 32, XH_SMEM, st>>>(n_maps, hp, hw, cdiv(hp.P, XW_TILE), fv.norms, desc_norm, cells.frame,
                                                       cells.group, xc.cell_of, xc.box_org, xc.stat, xc.cand, xc.key1, xc.max2,
                                                       xc.xbox, eps, grp_map0, out_index, out, xc.slow_cnt, xc.slow_list,
                                                       n_groups);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// ====================================================================================================== 5. full-map queue
// One block per queued map: copies its descriptor (fp32 + fp16 hi / lo), norm and output slot to compact row b; block 0
// also writes the compact group arrays.  Rows of a group keep their queue order (arbitrary, results do not depend on it).
// HILO: the fp16 row goes to c_hi interleaved per 32 channels ([rows][2 C], C % 32 == 0; c_lo unused).
template <bool HILO>
__global__ void __launch_bounds__(128)
xw_compact_kernel(const float4* __restrict__ desc, const uint4* __restrict__ dhi, const uint4* __restrict__ dlo,
                  const int* __restrict__ arow, const float* __restrict__ desc_norm, const int* __restrict__ out_index, int C, const int* __restrict__ grp_frame,
                  const int* __restrict__ grp_map0, int n_groups, const int* __restrict__ slow_cnt,
                  const int* __restrict__ slow_list, float4* __restrict__ c_desc, uint4* __restrict__ c_hi, uint4* __restrict__ c_lo,
                  float* __restrict__ c_norm, int* __restrict__ c_out_index, int* __restrict__ cgrp, int gcap, int row_base,
                  int grp_base) {
  __shared__ int s_g, s_pos;
  const int bb = blockIdx.x;
  if (threadIdx.x == 0) {
    int pre = 0, gsel = -1, psel = 0;
    for (int g = 0; g < n_groups; ++g) {
      const int c = slow_cnt[g];
      if (bb == 0) {
        cgrp[grp_base + g] = grp_frame[g]; cgrp[gcap + grp_base + g] = row_base + pre; cgrp[2 * gcap + grp_base + g] = c;
        cgrp[3 * gcap + grp_base + g] = row_base + pre;
      }
      if (gsel < 0 && bb < pre + c) { gsel = g; psel = bb - pre; }
      pre += c;
    }
    s_g = gsel; s_pos = psel;
  }
  __syncthreads();
  if (s_g < 0) return;
  const int b = row_base + bb;
  const int src = slow_list[grp_map0[s_g] + s_pos];
  const size_t srow = arow ? arow[src] : src;
  if (desc != nullptr)   // (the fp32 copy only feeds the non-tensor GEMMs)
    for (int i = threadIdx.x; i < C / 4; i += blockDim.x) c_desc[(size_t)b * (C / 4) + i] = desc[srow * (C / 4) + i];
  if (dhi != nullptr)
    for (int i = threadIdx.x; i < C / 8; i += blockDim.x) {
      if (HILO) {   // 8 channels = a quarter of a 32-channel block: hi at uint4 (i / 4) 8 + i % 4, lo 4 further
        const size_t o = (size_t)b * (C / 4) + (i >> 2) * 8 + (i & 3);
        c_hi[o] = dhi[srow * (C / 8) + i];
        c_hi[o + 4] = dlo[srow * (C / 8) + i];
      } else {
        c_hi[(size_t)b * (C / 8) + i] = dhi[srow * (C / 8) + i];
        c_lo[(size_t)b * (C / 8) + i] = dlo[srow * (C / 8) + i];
      }
    }
  if (threadIdx.x == 0) { c_norm[b] = desc_norm[src]; c_out_index[b] = out_index[src]; }
}

int launch_xw_compact(const float* desc, const void* desc_hi, const void* desc_lo, const int* arow, const float* desc_norm,
                      const int* out_index, int C, const int* grp_frame, const int* grp_map0, int n_groups, int n_slow,
                      const XwChunk& xc, float* c_desc, void* c_hi, void* c_lo, float* c_norm, int* c_out_index, int* cgrp,
                      int gcap, cudaStream_t st, int row_base, int grp_base, bool hilo) {
  if (n_slow <= 0) return DINOTRK_OK;
  DTK_CHECK_ARG(!hilo || C % 32 == 0, "xw_compact: interleaved rows need C %% 32 == 0");
  ProfRange pr(PROF_MISC, st);
  (hilo ? xw_compact_kernel<true> : xw_compact_kernel<false>)<<<n_slow, 128, 0, st>>>(reinterpret_cast<const float4*>(desc), reinterpret_cast<const uint4*>(desc_hi),
                                            reinterpret_cast<const uint4*>(desc_lo), arow, desc_norm, out_index, C, grp_frame, grp_map0,
                                            n_groups, xc.slow_cnt, xc.slow_list, reinterpret_cast<float4*>(c_desc),
                                            reinterpret_cast<uint4*>(c_hi), reinterpret_cast<uint4*>(c_lo), c_norm, c_out_index, cgrp,
                                            gcap, row_base, grp_base);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// tile_start[g] = sum over groups before g of ceil(m / TC2_BM) (one warp; the coarse GEMM's M-tile prefix)
__global__ void xw_tile_prefix_kernel(const int* __restrict__ grp_m, int n_groups, int* __restrict__ tile_start) {
  const int lane = threadIdx.x;
  int base = 0;
  for (int g0 = 0; g0 < n_groups; g0 += 32) {
    const int g = g0 + lane;
    const int v = g < n_groups ? (grp_m[g] + TC2_BM - 1) / TC2_BM : 0;
    int inc = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
      const int u = __shfl_up_sync(0xffffffffu, inc, o);
      if (lane >= o) inc += u;
    }
    if (g < n_groups) tile_start[g] = base + inc - v;
    base += __shfl_sync(0xffffffffu, inc, 31);
  }
  if (lane == 0) tile_start[n_groups] = base;
}

// workspace of the coarse-keys entry points: 1 / |F| of the T P tokens, the GEMM's tile prefix, the smallest token norm
struct XwKeysWs {
  float* rnorms; int* tile_start; unsigned* min_bits;
  XwKeysWs(Arena& ar, size_t tokens, int n_groups) {
    rnorms = ar.take<float>(tokens);
    tile_start = ar.take<int>(n_groups + 1);
    min_bits = ar.take<unsigned>(1);
  }
};

// eps[row] = xw_eps_s8(rho[row], rho_f[frame], slack) over the rows of group blockIdx.x
__global__ void xw_eps_kernel(const int* __restrict__ grp_frame, const int* __restrict__ grp_row0, const int* __restrict__ grp_m,
                              const float* __restrict__ rho, const float* __restrict__ rho_f, float slack, float* __restrict__ eps) {
  const int g = blockIdx.x, r0 = grp_row0[g];
  const float rf = rho_f[grp_frame[g]];
  for (int r = threadIdx.x; r < grp_m[g]; r += blockDim.x) eps[r0 + r] = xw_eps_s8(rho[r0 + r], rf, slack);
}

}  // namespace dtk

using namespace dtk;

extern "C" {

size_t dinotrk_xw_coarse_keys_workspace_bytes(int T, int n_groups, const dinotrk_geom* g) {
  return align_up(layout_end<XwKeysWs>((size_t)T * (g ? (size_t)g->h * g->w : 0), n_groups), 256) + 1024;
}

int dinotrk_xw_coarse_keys(const dinotrk_features* feat, const dinotrk_geom* g, const void* desc_hi, int desc_rows,
                           const float* desc_norm, const int* grp_frame, const int* grp_row0, const int* grp_m, int n_groups,
                           unsigned long long* key1, float* max2, void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(feat && feat->norms && feat->hi && g && desc_hi && desc_norm && grp_frame && grp_row0 && grp_m && key1 && max2,
                "xw_coarse_keys: null pointer (the fp16 split of the features is required)");
  DTK_CHECK_ARG(feat->T > 0 && feat->C > 0 && feat->C % 8 == 0 && desc_rows > 0 && n_groups >= 0,
                "xw_coarse_keys: bad sizes (C must be a multiple of 8)");
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_xw_coarse_keys_workspace_bytes(feat->T, n_groups, g),
                "xw_coarse_keys: workspace too small");
  if (n_groups == 0) return DINOTRK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const FeatView fv = make_view(*feat, *g);
  Arena ar(workspace);
  const XwKeysWs ws(ar, (size_t)fv.T * fv.P, n_groups);
  int rc = launch_xw_rnorms(fv, ws.rnorms, ws.min_bits, st);
  if (rc) return rc;
  {
    ProfRange pr(PROF_MISC, st);
    xw_tile_prefix_kernel<<<1, 32, 0, st>>>(grp_m, n_groups, ws.tile_start);
    DTK_LAUNCHED();
  }
  XwChunk xc{};
  xc.key1 = key1;
  xc.max2 = max2;
  return launch_xw_coarse(fv, desc_hi, desc_rows, desc_norm, grp_frame, grp_row0, grp_m, grp_row0, ws.tile_start, n_groups,
                          desc_rows / TC2_BM + n_groups, xc, st, ws.rnorms);
}

int dinotrk_xw_coarse_keys_i8(const dinotrk_features* feat, const dinotrk_geom* g, const void* desc_q8, const float* desc_fac,
                              const float* desc_rho, int desc_rows, const int* grp_frame, const int* grp_row0, const int* grp_m,
                              int n_groups, unsigned long long* key1, float* max2, float* eps, void* workspace,
                              size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(feat && feat->norms && feat->q8 && feat->q_fac && feat->q_rho && g && desc_q8 && desc_fac && desc_rho &&
                grp_frame && grp_row0 && grp_m && key1 && max2, "xw_coarse_keys_i8: null pointer (the int8 features are required)");
  DTK_CHECK_ARG(feat->T > 0 && feat->C > 0 && feat->C % 16 == 0 && feat->C <= XW_S8_MAX_C && desc_rows > 0 && n_groups >= 0,
                "xw_coarse_keys_i8: bad sizes (C must be a multiple of 16, <= %d)", XW_S8_MAX_C);
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_xw_coarse_keys_workspace_bytes(feat->T, n_groups, g),
                "xw_coarse_keys_i8: workspace too small");
  if (n_groups == 0) return DINOTRK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const FeatView fv = make_view(*feat, *g);
  Arena ar(workspace);
  const XwKeysWs ws(ar, (size_t)fv.T * fv.P, n_groups);   // rnorms and min_bits unused: the int8 epilogue needs no 1 / |F|
  {
    ProfRange pr(PROF_MISC, st);
    xw_tile_prefix_kernel<<<1, 32, 0, st>>>(grp_m, n_groups, ws.tile_start);
    DTK_LAUNCHED();
    if (eps) {
      xw_eps_kernel<<<n_groups, 128, 0, st>>>(grp_frame, grp_row0, grp_m, desc_rho, fv.q_rho, xw_s8_slack(fv.C), eps);
      DTK_LAUNCHED();
    }
  }
  XwChunk xc{};
  xc.key1 = key1;
  xc.max2 = max2;
  return launch_xw_coarse(fv, nullptr, desc_rows, nullptr, grp_frame, grp_row0, grp_m, grp_row0, ws.tile_start, n_groups,
                          desc_rows / TC2_BM + n_groups, xc, st, nullptr, desc_q8, desc_fac);
}

int dinotrk_xw_head_set_window_only(int on) {
  DTK_CHECK_ARG(on == 0 || on == 1, "xw_head_set_window_only: 0 or 1");
  g_xw_head_window_only = on;
  return DINOTRK_OK;
}

int dinotrk_xw_box_gemm_ext(const dinotrk_features* feat, const dinotrk_geom* g, const void* desc_hi, const void* desc_lo,
                            int desc_rows, const int* cell_row0, const int* cell_m, const int* cell_frame, const int* box_org,
                            const int* box_ext, int n_cells, int max_m, float* xbox, void* stream) {
  DTK_CHECK_ARG(feat && feat->hi && feat->lo && g && desc_hi && desc_lo && cell_row0 && cell_m && cell_frame && box_org && xbox,
                "xw_box_gemm: null pointer (the fp16 split of the features is required)");
  DTK_CHECK_ARG(feat->T > 0 && feat->C > 0 && feat->C % 8 == 0 && desc_rows > 0 && n_cells >= 0 && max_m > 0 &&
                max_m <= XW_MAX_CELL, "xw_box_gemm: bad sizes (C must be a multiple of 8, cells of 1..%d rows)", XW_MAX_CELL);
  DTK_CHECK_ARG(reinterpret_cast<uintptr_t>(box_org) % 8 == 0, "xw_box_gemm: box_org must be 8-byte aligned");
  DTK_CHECK_ARG(reinterpret_cast<uintptr_t>(box_ext) % 16 == 0, "xw_box_gemm: box_ext must be 16-byte aligned");
  const FeatView fv = make_view(*feat, *g);
  const XwCells cells{cell_row0, cell_row0, cell_m, cell_frame, nullptr, n_cells, max_m};
  XwChunk xc{};
  xc.box_org = reinterpret_cast<int2*>(const_cast<int*>(box_org));
  xc.box_ext = reinterpret_cast<int4*>(const_cast<int*>(box_ext));
  xc.xbox = xbox;
  return launch_xw_gemm(fv, *g, desc_hi, desc_lo, desc_rows, cells, xc, (cudaStream_t)stream);
}

int dinotrk_xw_box_gemm(const dinotrk_features* feat, const dinotrk_geom* g, const void* desc_hi, const void* desc_lo,
                        int desc_rows, const int* cell_row0, const int* cell_m, const int* cell_frame, const int* box_org,
                        int n_cells, int max_m, float* xbox, void* stream) {
  return dinotrk_xw_box_gemm_ext(feat, g, desc_hi, desc_lo, desc_rows, cell_row0, cell_m, cell_frame, box_org, nullptr, n_cells,
                                 max_m, xbox, stream);
}

}  // extern "C"

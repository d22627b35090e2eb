// Best-buddy contrastive losses of the training step (dino_tracker.py:332-344, get_bb_pairs_contrastive_loss) for all
// pairs of one loss in one call.  Rows are grouped by pair: group g owns rows [row0_g, row0_g + b_g) of the source / target
// descriptors S, U [B][C] and the frames s_g, t_g of the token-major frame set E [N][P][C].  Per row r of group g
//   bb[r]     = cos(S_r, U_r)
//   cst[r][n] = cos(S_r, E[t_g][n]),  cts[r][n] = cos(U_r, E[s_g][n])          (cos(a, b) = <a, b> / max(|a| |b|, 1e-8))
//   lse_st[r] = log sum_n exp(cst[r][n] / tau),  loss_st[r] = lse_st[r] - bb[r] / tau   (and the same for ts)
//
// Forward: the 2B x P cosines run through the grouped F16X3 wgmma GEMM of the correlation maps (corr_tc.cu, signed
// epilogue) on operands scaled by powers of two (the frame set as a whole, each descriptor row on its own), with the
// reference's clamp applied to the unscaled norm product (the clamp constant carries the same factors), and are KEPT for the backward (8.3 MB per 256 rows at P = 8107): recomputing
// them would repeat the forward's GEMM, the largest cost of the node.  Log-sum-exp and row sums are max-shifted block reductions in a fixed order.
//
// Backward, with D[R][n] the gradient reaching cosine (R, n) (softmax term + the constant of the mean), the clamp folded
// into Deff[R][n] = D |a_R| |E_n| / max(|a_R| |E_n|, 1e-8) (= D where the clamp is not hit):
//   dX_R  = (1 / |a_R|) sum_n Deff[R][n] Ê_n      - a_R / |a_R|^2 sum_n D cos u          (GEMM 1, K = P)
//   dE_n += (1 / |E_n|) sum_R Deff[R][n] â_R      - E_n / |E_n|^2 sum_R D cos u          (GEMM 2, K = rows of the frame)
// (u = 1 where the clamp is not hit; zero rows and zero tokens, whose cosines are all clamped, get their term in plain
// fp32 loops).  Both GEMMs run on wgmma with Deff split hi / lo after the power of two that puts its
// max |.| in [2^13, 2^14) (delta_train.cu's rule; the epilogue multiplies by the inverse), so the result does not depend on
// the gradient's scale.  Each accumulated K chain is at most 2048 long; chains and the correction terms are summed in a
// fixed order with no atomics on values: two runs give the same bits.
#include <cuda_fp16.h>

#include <algorithm>
#include <vector>

#include "common.cuh"
#include "corr.cuh"
#include "tcgemm.cuh"

namespace dtk {

constexpr int CL_THREADS = 256;
constexpr int CL_K_CHUNK = 2048;   // longest K chain of one wgmma accumulation (delta_train.cu: GEMM_K_CHUNK)

// The unit vectors Ê, â (the backward GEMMs' B operands, entries ~C^-1/2) are split after a fixed 2^13, so that their lo
// halves stay fp16 normals (2^-22 relative per element); the epilogues undo it with the gradient's scale.
constexpr int CL_UNIT_EXP = 13;

static int pad8(int x) { return (x + 7) & ~7; }

// one row's norm and cosine terms -------------------------------------------------------------------------------------
__global__ void cl_norms_kernel(const float* __restrict__ x, size_t rows, int C, float* __restrict__ norms) {
  const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= rows) return;
  const float* r = x + w * C;
  float s = 0.f;
  for (int c = lane; c < C; c += 32) s = fmaf(r[c], r[c], s);
  s = warp_sum(s);
  if (lane == 0) norms[w] = sqrtf(s);
}

// bb[r] = cos(S_r, U_r) for every row (rows of no group included: they are ignored downstream)
__global__ void cl_bb_kernel(const float* __restrict__ desc, const float* __restrict__ dn, int B, int C, float* __restrict__ bb) {
  const int r = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (r >= B) return;
  const float* s = desc + (size_t)r * C;
  const float* u = desc + (size_t)(B + r) * C;
  float d = 0.f;
  for (int c = lane; c < C; c += 32) d = fmaf(s[c], u[c], d);
  d = warp_sum(d);
  if (lane == 0) bb[r] = corr_cos(d, dn[r], dn[B + r]);
}

// fixed-order block reduction (sum or max) of one value per thread
template <bool kMax>
__device__ __forceinline__ float block_reduce(float v, float* sh) {
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const float t = __shfl_xor_sync(0xffffffffu, v, o);
    v = kMax ? fmaxf(v, t) : v + t;
  }
  __syncthreads();
  if (lane == 0) sh[warp] = v;
  __syncthreads();
  float a = sh[0];
  for (int k = 1; k < CL_THREADS / 32; ++k) a = kMax ? fmaxf(a, sh[k]) : a + sh[k];
  return a;
}

// block per row R of [2B]: max-shifted log-sum-exp and row sum of the cosine row; the loss of the row
// out = [7][B]: bb, lse_st, lse_ts, loss_st, loss_ts, rsum_st, rsum_ts
__global__ void __launch_bounds__(CL_THREADS)
cl_lse_kernel(const float* __restrict__ cosm, int P, int ld, int B, float inv_tau, const int* __restrict__ row_grp,
              float* __restrict__ out) {
  __shared__ float sh[CL_THREADS / 32];
  const int R = blockIdx.x, r = R < B ? R : R - B, dir = R < B ? 0 : 1;
  if (row_grp[r] < 0) return;
  const float* c = cosm + (size_t)R * ld;
  float mx = -INFINITY, rs = 0.f;
  for (int n = threadIdx.x; n < P; n += CL_THREADS) { mx = fmaxf(mx, c[n]); rs += c[n]; }
  mx = block_reduce<true>(mx, sh);
  rs = block_reduce<false>(rs, sh);
  const float m = mx * inv_tau;
  float se = 0.f;
  for (int n = threadIdx.x; n < P; n += CL_THREADS) se += expf(fmaf(c[n], inv_tau, -m));
  se = block_reduce<false>(se, sh);
  if (threadIdx.x == 0) {
    const float lse = m + logf(se);
    out[(size_t)(1 + dir) * B + r] = lse;
    out[(size_t)(3 + dir) * B + r] = lse - out[r] * inv_tau;
    out[(size_t)(5 + dir) * B + r] = rs;
  }
}

// ---- backward ----------------------------------------------------------------------------------------------------------
struct ClGrad {
  const float* cosm; int ld;      // [2B][ld] saved cosines
  const float* out;               // forward rows [7][B]
  const float* g_st; const float* g_ts;          // [B]
  const float* g_cmean;           // [n_groups]
  const int* row_grp; const int* grp_rows;       // [B], [n_groups]
  const float* dn;                // [2B] descriptor norms
  const float* en;                // [N][P] token norms
  const int* row_frame;           // [2B] frame of the row's cosines
  int B, P;
  float inv_tau;
  // D of cosine (R, n)
  __device__ __forceinline__ float grad(int R, int n) const {
    const int r = R < B ? R : R - B, g = row_grp[r];
    const float c = cosm[(size_t)R * ld + n];
    const float lse = out[(size_t)(R < B ? 1 : 2) * B + r];
    const float gr = R < B ? g_st[r] : g_ts[r];
    return fmaf(gr * inv_tau, expf(fmaf(c, inv_tau, -lse)), g_cmean[g] / (2.f * (float)grp_rows[g] * (float)P));
  }
  // (D cos u, Deff) of cosine (R, n)
  __device__ __forceinline__ void at(int R, int n, float& dcu, float& deff) const {
    const float c = cosm[(size_t)R * ld + n];
    const float d = grad(R, n);
    const float prod = __fmul_rn(dn[R], en[(size_t)row_frame[R] * P + n]);
    const bool u = prod >= 1e-8f;
    dcu = u ? d * c : 0.f;
    deff = u ? d : __fdiv_rn(d * prod, 1e-8f);
  }
};

// block per row R: Deff row (zero past P) into dbuf [2B][Pp], sum_n D cos u into rcorr[R], max |Deff| into amax
__global__ void __launch_bounds__(CL_THREADS)
cl_drow_kernel(ClGrad gr, int Pp, float* __restrict__ dbuf, float* __restrict__ rcorr, unsigned* __restrict__ amax) {
  __shared__ float sh[CL_THREADS / 32];
  const int R = blockIdx.x, r = R < gr.B ? R : R - gr.B;
  float* drow = dbuf + (size_t)R * Pp;
  if (gr.row_grp[r] < 0) {
    for (int n = threadIdx.x; n < Pp; n += CL_THREADS) drow[n] = 0.f;
    if (threadIdx.x == 0) rcorr[R] = 0.f;
    return;
  }
  float s = 0.f;
  unsigned m = 0u;
  for (int n = threadIdx.x; n < Pp; n += CL_THREADS) {
    float dcu = 0.f, deff = 0.f;
    if (n < gr.P) gr.at(R, n, dcu, deff);
    drow[n] = deff;
    s += dcu;
    m = max(m, __float_as_uint(fabsf(deff)));
  }
  s = block_reduce<false>(s, sh);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(amax, m);   // a max: the same bits in any order
  if (threadIdx.x == 0) rcorr[R] = s;
}

// Descriptor rows of the forward GEMM, warp per row: each row split after its own power of two (max |.| in [2^13, 2^14)),
// its norm scaled alike, and the reference's 1e-8 clamp carried to the scaled product of the row's and the frame set's
// norms (same decisions, same quotients as the unscaled product).
__global__ void cl_desc_split_kernel(const float* __restrict__ desc, const float* __restrict__ dn, size_t rows, int C,
                                     const unsigned* __restrict__ amax_e, __half* __restrict__ hi, __half* __restrict__ lo,
                                     float* __restrict__ dn_s, float* __restrict__ eps) {
  const size_t r = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= rows) return;
  const float* x = desc + r * C;
  unsigned m = 0u;
  for (int c = lane; c < C; c += 32) m = max(m, __float_as_uint(fabsf(x[c])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  const int e = grad_exp(m);
  const float s = ldexpf(1.f, e);
  for (int c = lane; c < C; c += 32) split16(x[c] * s, hi[r * C + c], lo[r * C + c]);
  if (lane == 0) {
    const int ee = e + grad_exp(*amax_e);
    dn_s[r] = dn[r] * s;
    eps[r] = ldexpf(1e-8f, ee < 150 ? ee : 150);
  }
}

// y = x * 2^grad_exp(amax) (exact)
__global__ void cl_scale_kernel(const float* __restrict__ x, const unsigned* __restrict__ amax, float* __restrict__ y, size_t n) {
  const float s = ldexpf(1.f, grad_exp(*amax));
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x) y[i] = x[i] * s;
}

// A of GEMM 1: Deff * 2^e split, [2B][Pp] (also the forward's scaled operands)
__global__ void cl_split_rows_kernel(const float* __restrict__ d, const unsigned* __restrict__ amax, __half* __restrict__ hi,
                                     __half* __restrict__ lo, size_t n) {
  const float s = ldexpf(1.f, grad_exp(*amax));
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    split16(d[i] * s, hi[i], lo[i]);
}

// 32 x 32 transposing split: out[z][c][k] = (in(z, k, c) * scale(z, k)) split, for k < kn, c < cn (zero where the source
// is absent).  Used for the three transposed operands below through the `Src` functor.
template <class Src>
__global__ void cl_transpose_split_kernel(Src src, int kn, int cn, int ld_out, __half* __restrict__ hi, __half* __restrict__ lo) {
  __shared__ float tile[32][33];
  const int z = blockIdx.z, k0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int k = k0 + i, c = c0 + threadIdx.x;
    tile[i][threadIdx.x] = (k < kn && c < cn) ? src(z, k, c) : 0.f;
  }
  __syncthreads();
  for (int i = threadIdx.y; i < 32; i += blockDim.y) {
    const int c = c0 + i, k = k0 + threadIdx.x;
    if (c < cn && k < ld_out) {
      __half h, l;
      split16(tile[threadIdx.x][i], h, l);
      const size_t o = ((size_t)z * cn + c) * ld_out + k;
      hi[o] = h; lo[o] = l;
    }
  }
}

// B of GEMM 1: Ê^T [N][C][Pp]
struct SrcEhatT {
  const float* E; const float* en; int P, C;
  __device__ __forceinline__ float operator()(int f, int n, int c) const {
    if (n >= P) return 0.f;
    const float nr = en[(size_t)f * P + n];
    return nr > 0.f ? ldexpf(__fdiv_rn(E[((size_t)f * P + n) * C + c], nr), CL_UNIT_EXP) : 0.f;
  }
};
// A of GEMM 2: (Deff * 2^e)^T per frame, [N][Pp][Kx]: out[f][n][k] = Deff[rows_f[k]][n]
struct SrcDT {
  const float* d; const int* frame_rows; const unsigned* amax; int Pp, Kx;
  __device__ __forceinline__ float operator()(int f, int k, int n) const {
    const int R = frame_rows[(size_t)f * Kx + k];
    return R < 0 ? 0.f : d[(size_t)R * Pp + n] * ldexpf(1.f, grad_exp(*amax));
  }
};
// B of GEMM 2: â^T per frame, [N][C][Kx]: out[f][c][k] = desc[rows_f[k]][c] / |desc|
struct SrcDescT {
  const float* desc; const float* dn; const int* frame_rows; int C, Kx;
  __device__ __forceinline__ float operator()(int f, int k, int c) const {
    const int R = frame_rows[(size_t)f * Kx + k];
    if (R < 0) return 0.f;
    const float nr = dn[R];
    return nr > 0.f ? ldexpf(__fdiv_rn(desc[(size_t)R * C + c], nr), CL_UNIT_EXP) : 0.f;
  }
};

// GEMM 1 epilogue: dX[R][col] (+)= acc 2^-e / |a_R|  (R < B: dS, else dU)
struct EpiDesc {
  float* dS; float* dU; const float* dn; const int* grp_row0; const unsigned* amax; int B, C, accumulate;
  struct State { float inv; };
  __device__ __forceinline__ void tile_begin(State& s) const { s.inv = ldexpf(1.f, -grad_exp(*amax) - CL_UNIT_EXP); }
  __device__ __forceinline__ void tile_end(State&, int, int, int) const {}
  __device__ __forceinline__ void operator()(State& s, int g, int r, int col0, const float (&f)[32], int ncols) const {
    const int R = grp_row0[g] + r;
    const float nr = dn[R];
    float* o = (R < B ? dS + (size_t)R * C : dU + (size_t)(R - B) * C) + col0;
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (i < ncols) {
        const float v = nr > 0.f ? __fdiv_rn(f[i] * s.inv, nr) : 0.f;
        o[i] = accumulate ? o[i] + v : v;
      }
  }
};

// GEMM 2 epilogue: dE[f][n][col] += acc 2^-e / |E_n|
struct EpiTok {
  float* dE; const float* en; const int* grp_batch; const unsigned* amax; int P, C;
  struct State { float inv; };
  __device__ __forceinline__ void tile_begin(State& s) const { s.inv = ldexpf(1.f, -grad_exp(*amax) - CL_UNIT_EXP); }
  __device__ __forceinline__ void tile_end(State&, int, int, int) const {}
  __device__ __forceinline__ void operator()(State& s, int g, int n, int col0, const float (&f)[32], int ncols) const {
    const size_t tok = (size_t)grp_batch[g] * P + n;
    const float nr = en[tok];
    float* o = dE + tok * C + col0;
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (i < ncols && nr > 0.f) o[i] += __fdiv_rn(f[i] * s.inv, nr);
  }
};

// warp per row R: dX_R += - a_R / |a_R|^2 rcorr[R] + g_bb[r] dcos(S_r, U_r) / dX_R.  A zero row (every cosine of it
// clamped, no direction for GEMM 1) gets its full-frame term sum_n D E_n / 1e-8 here, tokens in order.
__global__ void cl_row_finish_kernel(ClGrad gr, const float* __restrict__ E, const float* __restrict__ desc,
                                     const float* __restrict__ dn, const float* __restrict__ rcorr,
                                     const float* __restrict__ out, const float* __restrict__ g_st, const float* __restrict__ g_ts,
                                     const float* __restrict__ g_bbmean, const int* __restrict__ row_grp,
                                     const int* __restrict__ grp_rows, int B, int C, float inv_tau, float* __restrict__ dS,
                                     float* __restrict__ dU) {
  const int R = (int)(((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5);
  const int lane = threadIdx.x & 31;
  if (R >= 2 * B) return;
  const int r = R < B ? R : R - B, g = row_grp[r];
  float* o = R < B ? dS + (size_t)r * C : dU + (size_t)r * C;
  if (g < 0) {
    for (int c = lane; c < C; c += 32) o[c] = 0.f;
    return;
  }
  const float na = dn[R], nb = dn[R < B ? R + B : R - B];
  const float* a = desc + (size_t)R * C;
  const float* b = desc + (size_t)(R < B ? R + B : R - B) * C;
  const float prod = __fmul_rn(na, nb);
  const bool ub = prod >= 1e-8f;
  const float den = fmaxf(prod, 1e-8f);
  const float gbb = -(g_st[r] + g_ts[r]) * inv_tau + g_bbmean[g] / (float)grp_rows[g];
  const float bbv = out[r];
  const bool ua = na > 0.f;
  const float ca = ua ? rcorr[R] / (na * na) : 0.f;            // rcorr only gathers unclamped terms: 0 when |a| = 0
  const float cb = ub ? gbb * bbv / (na * na) : 0.f;
  for (int c = lane; c < C; c += 32) o[c] += gbb * __fdiv_rn(b[c], den) - (ca + cb) * a[c];
  if (!ua) {
    const float* ef = E + (size_t)gr.row_frame[R] * gr.P * C;
    for (int n = 0; n < gr.P; ++n) {
      const float d = __fdiv_rn(gr.grad(R, n), 1e-8f);
      for (int c = lane; c < C; c += 32) o[c] = fmaf(d, ef[(size_t)n * C + c], o[c]);
    }
  }
}

// warp per token (f, n): dE[f][n] -= E_n / |E_n|^2 sum over the frame's rows of D cos u  (rows in frame_rows order)
__global__ void cl_tok_corr_kernel(ClGrad gr, const float* __restrict__ E, const float* __restrict__ desc,
                                   const int* __restrict__ frame_rows,
                                   const int* __restrict__ frame_k, int N, int Kx, int C, float* __restrict__ dE) {
  const size_t w = ((size_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (w >= (size_t)N * gr.P) return;
  const int f = (int)(w / gr.P), n = (int)(w - (size_t)f * gr.P);
  const int K = frame_k[f];
  if (K == 0) return;
  float s = 0.f;
  for (int k = lane; k < K; k += 32) {
    float dcu, deff;
    gr.at(frame_rows[(size_t)f * Kx + k], n, dcu, deff);
    s += dcu;
  }
  s = warp_sum(s);
  const float nr = gr.en[w];
  float* o = dE + w * C;
  if (!(nr > 0.f)) {   // a zero token: no direction for GEMM 2, its term sum_R D a_R / 1e-8 here, rows in order
    for (int k = 0; k < K; ++k) {
      const int R = frame_rows[(size_t)f * Kx + k];
      const float d = __fdiv_rn(gr.grad(R, n), 1e-8f);
      for (int c = lane; c < C; c += 32) o[c] = fmaf(d, desc[(size_t)R * C + c], o[c]);
    }
    return;
  }
  const float coef = s / (nr * nr);
  const float* e = E + w * C;
  for (int c = lane; c < C; c += 32) o[c] -= coef * e[c];
}

// ---- host-side plan --------------------------------------------------------------------------------------------------
// Directional groups: k = g (S rows against frame t_g) and k = G + g (U rows, stored at B + row, against frame s_g).
struct ClPlan {
  int G2;                                  // 2 * n_groups
  std::vector<int> frame, row0, m, tile_start, zero;   // the directional groups' GEMM tables (tile_start: 128-row tiles)
  std::vector<int> row_grp;                // [B] group of a row, -1 if none
  std::vector<int> row_frame;              // [2B]
  std::vector<int> frame_k;                // [N] rows whose cosines are against frame f
  int Kx;                                  // pad8(max frame_k)
  std::vector<int> frame_rows;             // [N][Kx] those rows, directional-group order (-1 padding)
  std::vector<int> f_batch, f_row0, f_m, f_tiles;      // GEMM 2 groups: one per frame (frames without rows have m = 0)
  int tiles1, tiles2;
};

static int cl_check(int N, int P, int C, int B, const int* grp_src, const int* grp_tgt, const int* grp_row0,
                    const int* grp_rows, int n_groups, float tau) {
  DTK_CHECK_ARG(N > 0 && P > 0 && B >= 0 && n_groups >= 0, "bb_contrastive: bad sizes");
  DTK_CHECK_ARG(C > 0 && C % 8 == 0, "bb_contrastive: C must be a positive multiple of 8 (got %d)", C);
  DTK_CHECK_ARG(tau > 0.f, "bb_contrastive: temperature must be positive");
  DTK_CHECK_ARG(n_groups == 0 || (grp_src && grp_tgt && grp_row0 && grp_rows), "bb_contrastive: null group table");
  std::vector<char> used(B > 0 ? B : 1, 0);
  for (int g = 0; g < n_groups; ++g) {
    DTK_CHECK_ARG(grp_src[g] >= 0 && grp_src[g] < N && grp_tgt[g] >= 0 && grp_tgt[g] < N,
                  "bb_contrastive: group %d has frame slots (%d, %d) outside [0, %d)", g, grp_src[g], grp_tgt[g], N);
    DTK_CHECK_ARG(grp_rows[g] >= 0 && grp_row0[g] >= 0 && (long long)grp_row0[g] + grp_rows[g] <= B,
                  "bb_contrastive: group %d rows [%d, +%d) outside [0, %d)", g, grp_row0[g], grp_rows[g], B);
    for (int r = grp_row0[g]; r < grp_row0[g] + grp_rows[g]; ++r) {
      DTK_CHECK_ARG(!used[r], "bb_contrastive: row %d belongs to two groups", r);
      used[r] = 1;
    }
  }
  return DINOTRK_OK;
}

static ClPlan cl_plan(int N, int P, int B, const int* grp_src, const int* grp_tgt, const int* grp_row0, const int* grp_rows,
                      int G) {
  ClPlan p;
  p.G2 = 2 * G;
  int acc = 0;
  for (int k = 0; k < p.G2; ++k) {
    const int g = k % G, dir = k / G;
    p.frame.push_back(dir ? grp_src[g] : grp_tgt[g]);
    p.row0.push_back(grp_row0[g] + dir * B);
    p.m.push_back(grp_rows[g]);
    p.zero.push_back(0);
    p.tile_start.push_back(acc);
    acc += cdiv(grp_rows[g], TC_BM);
  }
  p.tile_start.push_back(acc);
  p.tiles1 = acc;
  p.row_grp.assign(B, -1);
  p.row_frame.assign(2 * B, 0);
  p.frame_k.assign(N, 0);
  for (int k = 0; k < p.G2; ++k) {
    for (int r = 0; r < p.m[k]; ++r) {
      if (k < G) p.row_grp[grp_row0[k] + r] = k;
      p.row_frame[p.row0[k] + r] = p.frame[k];
    }
    p.frame_k[p.frame[k]] += p.m[k];
  }
  int kmax = 0;
  for (int f = 0; f < N; ++f) kmax = p.frame_k[f] > kmax ? p.frame_k[f] : kmax;
  p.Kx = pad8(kmax > 0 ? kmax : 1);
  p.frame_rows.assign((size_t)N * p.Kx, -1);
  std::vector<int> fill(N, 0);
  for (int k = 0; k < p.G2; ++k)
    for (int r = 0; r < p.m[k]; ++r) p.frame_rows[(size_t)p.frame[k] * p.Kx + fill[p.frame[k]]++] = p.row0[k] + r;
  const int Pp = pad8(P);
  acc = 0;
  for (int f = 0; f < N; ++f) {
    p.f_batch.push_back(f);
    p.f_row0.push_back(f * Pp);
    p.f_m.push_back(p.frame_k[f] ? P : 0);
    p.f_tiles.push_back(acc);
    acc += p.frame_k[f] ? cdiv(P, TC_BM) : 0;
  }
  p.f_tiles.push_back(acc);
  p.tiles2 = acc;
  return p;
}

template <class T>
static void upload(T* d, const std::vector<T>& v, cudaStream_t st, int* rc) {
  if (!v.empty() && cudaMemcpyAsync(d, v.data(), v.size() * sizeof(T), cudaMemcpyHostToDevice, st) != cudaSuccess) {
    set_error("bb_contrastive: table upload failed");
    *rc = DINOTRK_ECUDA;
  }
}

// The plan tables are carved at the bounds the plan can reach from the shapes (the group tables at 2 n_groups + 1).
struct ClFwdWs {
  __half* e_hi; __half* e_lo; float* en; float* desc; float* dn; float* split_ws; float* en_s; float* dn_s; unsigned* amax;
  float* eps_s; int* frame; int* row0; int* m; int* tile_start; int* spare; int* row_grp;
  ClFwdWs(Arena& ar, int N, int P, int C, int B, int n_groups) {
    e_hi = ar.take<__half>((size_t)N * P * C);
    e_lo = ar.take<__half>((size_t)N * P * C);
    en = ar.take<float>((size_t)N * P);                   // token norms
    desc = ar.take<float>((size_t)2 * B * C);             // [S; U]
    dn = ar.take<float>((size_t)2 * B);                   // their norms
    split_ws = ar.take<float>(corr_tc_workspace_bytes(2 * B, C) / sizeof(float));
    en_s = ar.take<float>((size_t)N * P);                 // scaled token norms
    dn_s = ar.take<float>((size_t)2 * B);                 // scaled descriptor norms
    amax = ar.take<unsigned>(1);                          // max |E|
    eps_s = ar.take<float>((size_t)2 * B);                // per-row clamp of the scaled norm products
    frame = ar.take<int>(2 * n_groups + 1);
    row0 = ar.take<int>(2 * n_groups + 1);
    m = ar.take<int>(2 * n_groups + 1);
    tile_start = ar.take<int>(2 * n_groups + 1);
    spare = ar.take<int>(2 * n_groups + 1);               // unused; part of the size callers allocate
    row_grp = ar.take<int>(B > 0 ? B : 1);
  }
};

struct ClBwdWs {
  float* en; float* desc; float* dn; float* rcorr; unsigned* amax; float* dbuf;
  __half *a1_hi, *a1_lo, *b1_hi, *b1_lo, *a2_hi, *a2_lo, *b2_hi, *b2_lo;
  int *frame, *row0, *m, *tile_start, *row_grp, *row_frame, *frame_k, *frame_rows, *f_batch, *f_row0, *f_m, *f_tiles, *grows;
  ClBwdWs(Arena& ar, int N, int P, int C, int B, const ClPlan& pl) {
    const size_t Pp = pad8(P);
    en = ar.take<float>((size_t)N * P);                   // token norms
    desc = ar.take<float>((size_t)2 * B * C);             // [S; U]
    dn = ar.take<float>((size_t)2 * B);                   // norms
    rcorr = ar.take<float>((size_t)2 * B);                // row corrections
    amax = ar.take<unsigned>(1);
    dbuf = ar.take<float>((size_t)2 * B * Pp);            // Deff
    a1_hi = ar.take<__half>((size_t)2 * B * Pp);
    a1_lo = ar.take<__half>((size_t)2 * B * Pp);
    b1_hi = ar.take<__half>((size_t)N * C * Pp);
    b1_lo = ar.take<__half>((size_t)N * C * Pp);
    a2_hi = ar.take<__half>((size_t)N * Pp * pl.Kx);
    a2_lo = ar.take<__half>((size_t)N * Pp * pl.Kx);
    b2_hi = ar.take<__half>((size_t)N * C * pl.Kx);
    b2_lo = ar.take<__half>((size_t)N * C * pl.Kx);
    frame = ar.take<int>(pl.G2 + 1);
    row0 = ar.take<int>(pl.G2 + 1);
    m = ar.take<int>(pl.G2 + 1);
    tile_start = ar.take<int>(pl.G2 + 1);
    row_grp = ar.take<int>(B > 0 ? B : 1);
    row_frame = ar.take<int>(2 * (size_t)B + 1);
    frame_k = ar.take<int>(N);
    frame_rows = ar.take<int>((size_t)N * pl.Kx);
    f_batch = ar.take<int>(N + 1);
    f_row0 = ar.take<int>(N + 1);
    f_m = ar.take<int>(N + 1);
    f_tiles = ar.take<int>(N + 1);
    grows = ar.take<int>(pl.G2 > 0 ? pl.G2 / 2 : 1);   // rows per group
  }
};

}  // namespace dtk

using namespace dtk;

extern "C" {

int dinotrk_bb_contrastive_cos_stride(int P) { return pad8(P); }

size_t dinotrk_bb_contrastive_forward_workspace_bytes(int N, int P, int C, int B, int n_groups) {
  return layout_end<ClFwdWs>(N, P, C, B, n_groups) + 256;
}

int dinotrk_bb_contrastive_forward(const float* E, int N, int P, int C, const float* S, const float* U, int B,
                                   const int* grp_src, const int* grp_tgt, const int* grp_row0, const int* grp_rows, int n_groups,
                                   float tau, float* cosm, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = cl_check(N, P, C, B, grp_src, grp_tgt, grp_row0, grp_rows, n_groups, tau)) return rc;
  DTK_CHECK_ARG(E && (B == 0 || (S && U && cosm && out)), "bb_contrastive_forward: null pointer");
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_bb_contrastive_forward_workspace_bytes(N, P, C, B, n_groups),
                "bb_contrastive_forward: workspace too small");
  ClPlan pl = cl_plan(N, P, B, grp_src, grp_tgt, grp_row0, grp_rows, n_groups);
  if (pl.tiles1 == 0) return DINOTRK_OK;   // every group empty
  cudaStream_t st = (cudaStream_t)stream;
  ProfRange pr(PROF_CONTRASTIVE, st);
  Arena ar(workspace);
  const ClFwdWs ws(ar, N, P, C, B, n_groups);
  int rc = DINOTRK_OK;
  upload(ws.frame, pl.frame, st, &rc);
  upload(ws.row0, pl.row0, st, &rc);
  upload(ws.m, pl.m, st, &rc);
  upload(ws.tile_start, pl.tile_start, st, &rc);
  upload(ws.row_grp, pl.row_grp, st, &rc);
  if (rc) return rc;
  DTK_CUDA(cudaMemcpyAsync(ws.desc, S, (size_t)B * C * 4, cudaMemcpyDeviceToDevice, st));
  DTK_CUDA(cudaMemcpyAsync(ws.desc + (size_t)B * C, U, (size_t)B * C * 4, cudaMemcpyDeviceToDevice, st));
  const size_t toks = (size_t)N * P;
  cl_norms_kernel<<<(unsigned)((toks * 32 + 255) / 256), 256, 0, st>>>(E, toks, C, ws.en);
  DTK_LAUNCHED();
  cl_norms_kernel<<<(unsigned)((2 * (size_t)B * 32 + 255) / 256), 256, 0, st>>>(ws.desc, 2 * (size_t)B, C, ws.dn);
  DTK_LAUNCHED();
  cl_bb_kernel<<<(unsigned)(((size_t)B * 32 + 255) / 256), 256, 0, st>>>(ws.desc, ws.dn, B, C, out);
  DTK_LAUNCHED();
  // E is split after the power of two that puts its max |.| in [2^13, 2^14), every descriptor row after its own, and the
  // epilogue's norms and clamp carry the same factors: the cosines do not depend on the inputs' scale, and a row far below
  // the others keeps its precision.
  DTK_CUDA(cudaMemsetAsync(ws.amax, 0, sizeof(unsigned), st));
  const unsigned ge = (unsigned)std::min<size_t>((toks * C + 255) / 256, (size_t)num_sms() * 16);
  if ((rc = launch_amax(E, toks * C, ws.amax, ge, st))) return rc;
  cl_split_rows_kernel<<<ge, 256, 0, st>>>(E, ws.amax, ws.e_hi, ws.e_lo, toks * C);
  DTK_LAUNCHED();
  const DescSplit d(ws.split_ws, 2 * (size_t)B, C);   // launch_corr_gemm_tc's layout of a ready split
  __half* d_hi = reinterpret_cast<__half*>(d.hi);
  __half* d_lo = reinterpret_cast<__half*>(d.lo);
  cl_desc_split_kernel<<<(unsigned)cdiv(2 * B * 32, 256), 256, 0, st>>>(ws.desc, ws.dn, 2 * (size_t)B, C, ws.amax, d_hi, d_lo, ws.dn_s,
                                                                         ws.eps_s);
  DTK_LAUNCHED();
  cl_scale_kernel<<<(unsigned)std::min<size_t>((toks + 255) / 256, (size_t)num_sms() * 16), 256, 0, st>>>(ws.en, ws.amax, ws.en_s, toks);
  DTK_LAUNCHED();
  if ((rc = launch_corr_gemm_tc(ws.e_hi, ws.e_lo, ws.en_s, N, C, P, ws.desc, 2 * B, ws.dn_s, ws.frame, ws.row0, ws.m, ws.row0, ws.tile_start, pl.G2,
                                pl.tiles1, cosm, pad8(P), ws.split_ws, st, nullptr, true, TC_BM, false, ws.eps_s)))
    return rc;
  cl_lse_kernel<<<2 * B, CL_THREADS, 0, st>>>(cosm, P, pad8(P), B, 1.f / tau, ws.row_grp, out);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

size_t dinotrk_bb_contrastive_backward_workspace_bytes(int N, int P, int C, int B, const int* grp_src, const int* grp_tgt,
                                                       const int* grp_row0, const int* grp_rows, int n_groups) {
  if (cl_check(N, P, C, B, grp_src, grp_tgt, grp_row0, grp_rows, n_groups, 1.f)) return 0;
  return layout_end<ClBwdWs>(N, P, C, B, cl_plan(N, P, B, grp_src, grp_tgt, grp_row0, grp_rows, n_groups)) + 256;
}

int dinotrk_bb_contrastive_backward(const float* E, int N, int P, int C, const float* S, const float* U, int B,
                                    const int* grp_src, const int* grp_tgt, const int* grp_row0, const int* grp_rows,
                                    int n_groups, float tau, const float* cosm, const float* out, const float* g_st,
                                    const float* g_ts, const float* g_bbmean, const float* g_cmean, float* dS, float* dU,
                                    float* dE, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = cl_check(N, P, C, B, grp_src, grp_tgt, grp_row0, grp_rows, n_groups, tau)) return rc;
  DTK_CHECK_ARG(E && dE && (B == 0 || (S && U && cosm && out && g_st && g_ts && dS && dU)) &&
                    (n_groups == 0 || (g_bbmean && g_cmean)),
                "bb_contrastive_backward: null pointer");
  ClPlan pl = cl_plan(N, P, B, grp_src, grp_tgt, grp_row0, grp_rows, n_groups);
  DTK_CHECK_ARG(workspace && workspace_bytes >= layout_end<ClBwdWs>(N, P, C, B, pl) + 256, "bb_contrastive_backward: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  if (pl.tiles1 == 0) {   // every group empty: zero descriptor gradients, nothing into dE
    if (B > 0) {
      DTK_CUDA(cudaMemsetAsync(dS, 0, (size_t)B * C * 4, st));
      DTK_CUDA(cudaMemsetAsync(dU, 0, (size_t)B * C * 4, st));
    }
    return DINOTRK_OK;
  }
  ProfRange pr(PROF_CONTRASTIVE, st);
  const int Pp = pad8(P), Kx = pl.Kx;
  Arena ar(workspace);
  const ClBwdWs ws(ar, N, P, C, B, pl);
  int rc = DINOTRK_OK;
  upload(ws.frame, pl.frame, st, &rc);
  upload(ws.row0, pl.row0, st, &rc);
  upload(ws.m, pl.m, st, &rc);
  upload(ws.tile_start, pl.tile_start, st, &rc);
  upload(ws.row_grp, pl.row_grp, st, &rc);
  upload(ws.row_frame, pl.row_frame, st, &rc);
  upload(ws.frame_k, pl.frame_k, st, &rc);
  upload(ws.frame_rows, pl.frame_rows, st, &rc);
  upload(ws.f_batch, pl.f_batch, st, &rc);
  upload(ws.f_row0, pl.f_row0, st, &rc);
  upload(ws.f_m, pl.f_m, st, &rc);
  upload(ws.f_tiles, pl.f_tiles, st, &rc);
  std::vector<int> grows(n_groups);
  for (int g = 0; g < n_groups; ++g) grows[g] = grp_rows[g];
  upload(ws.grows, grows, st, &rc);
  if (rc) return rc;
  DTK_CUDA(cudaMemcpyAsync(ws.desc, S, (size_t)B * C * 4, cudaMemcpyDeviceToDevice, st));
  DTK_CUDA(cudaMemcpyAsync(ws.desc + (size_t)B * C, U, (size_t)B * C * 4, cudaMemcpyDeviceToDevice, st));
  DTK_CUDA(cudaMemsetAsync(ws.amax, 0, sizeof(unsigned), st));
  const size_t toks = (size_t)N * P;
  cl_norms_kernel<<<(unsigned)((toks * 32 + 255) / 256), 256, 0, st>>>(E, toks, C, ws.en);
  DTK_LAUNCHED();
  cl_norms_kernel<<<(unsigned)((2 * (size_t)B * 32 + 255) / 256), 256, 0, st>>>(ws.desc, 2 * (size_t)B, C, ws.dn);
  DTK_LAUNCHED();
  ClGrad gr{cosm, Pp, out, g_st, g_ts, g_cmean, ws.row_grp, ws.grows, ws.dn, ws.en, ws.row_frame, B, P, 1.f / tau};
  cl_drow_kernel<<<2 * B, CL_THREADS, 0, st>>>(gr, Pp, ws.dbuf, ws.rcorr, ws.amax);
  DTK_LAUNCHED();
  {
    const size_t n = (size_t)2 * B * Pp;
    unsigned grid = (unsigned)((n + 255) / 256);
    if (grid > (unsigned)num_sms() * 16) grid = num_sms() * 16;
    cl_split_rows_kernel<<<grid, 256, 0, st>>>(ws.dbuf, ws.amax, ws.a1_hi, ws.a1_lo, n);
    DTK_LAUNCHED();
  }
  const dim3 tb(32, 8);
  cl_transpose_split_kernel<<<dim3(cdiv(Pp, 32), cdiv(C, 32), N), tb, 0, st>>>(SrcEhatT{E, ws.en, P, C}, Pp, C, Pp, ws.b1_hi, ws.b1_lo);
  DTK_LAUNCHED();
  cl_transpose_split_kernel<<<dim3(cdiv(Kx, 32), cdiv(Pp, 32), N), tb, 0, st>>>(SrcDT{ws.dbuf, ws.frame_rows, ws.amax, Pp, Kx}, Kx, Pp,
                                                                                  Kx, ws.a2_hi, ws.a2_lo);
  DTK_LAUNCHED();
  cl_transpose_split_kernel<<<dim3(cdiv(Kx, 32), cdiv(C, 32), N), tb, 0, st>>>(SrcDescT{ws.desc, ws.dn, ws.frame_rows, C, Kx}, Kx, C,
                                                                                 Kx, ws.b2_hi, ws.b2_lo);
  DTK_LAUNCHED();
  // GEMM 1: dS / dU over K = P in chains of CL_K_CHUNK, the first chain overwrites; one launch per chain [k0, k0 + kc)
  for (int k0 = 0; k0 < P; k0 += CL_K_CHUNK) {
    EpiDesc epi{dS, dU, ws.dn, ws.row0, ws.amax, B, C, k0 > 0};
    const TcProblem pb{ws.frame, ws.row0, ws.m, ws.tile_start, pl.G2, C, std::min(CL_K_CHUNK, P - k0)};
    if ((rc = tc_launch_bn<TcMode::F16X3>({ws.a1_hi + k0, ws.a1_lo + k0, (uint64_t)2 * B, (uint64_t)Pp, ws.b1_hi + k0, ws.b1_lo + k0,
                                           (uint64_t)N, (uint64_t)Pp}, pb, pl.tiles1, epi, st)))
      return rc;
  }
  cl_row_finish_kernel<<<(unsigned)((2 * (size_t)B * 32 + 255) / 256), 256, 0, st>>>(
      gr, E, ws.desc, ws.dn, ws.rcorr, out, g_st, g_ts, g_bbmean, ws.row_grp, ws.grows, B, C, 1.f / tau, dS, dU);
  DTK_LAUNCHED();
  // dE: the norm correction, then GEMM 2 over the frame's rows in chains of CL_K_CHUNK
  cl_tok_corr_kernel<<<(unsigned)((toks * 32 + 255) / 256), 256, 0, st>>>(gr, E, ws.desc, ws.frame_rows, ws.frame_k, N, Kx, C, dE);
  DTK_LAUNCHED();
  if (pl.tiles2 > 0) {
    EpiTok epi{dE, ws.en, ws.f_batch, ws.amax, P, C};
    for (int k0 = 0; k0 < Kx; k0 += CL_K_CHUNK) {
      const TcProblem pb{ws.f_batch, ws.f_row0, ws.f_m, ws.f_tiles, N, C, std::min(CL_K_CHUNK, Kx - k0)};
      if ((rc = tc_launch_bn<TcMode::F16X3>({ws.a2_hi + k0, ws.a2_lo + k0, (uint64_t)N * Pp, (uint64_t)Kx, ws.b2_hi + k0, ws.b2_lo + k0,
                                             (uint64_t)N, (uint64_t)Kx}, pb, pl.tiles2, epi, st)))
        return rc;
    }
  }
  return DINOTRK_OK;
}

}  // extern "C"

// Delta-DINO's training step (models/networks/delta_dino.py:22-61 with gradients, models/tracker.py:113-129):
//   forward  : per layer the convolution on tensor cores (delta.cu's im2col + F16X3 GEMM, conv bias, no ReLU), BatchNorm
//              on the batch statistics (train) or the running statistics (eval), ReLU + BlurPool (layers 1-3), and for
//              the last layer the bilinear alignment onto the token grid.  The pre-BN conv outputs and the per-channel
//              mean / 1/sigma are kept for the reverse pass.
//   backward : alignment adjoint, BatchNorm backward, ReLU mask, BlurPool adjoint, and per convolution the weight
//              gradient dW = dY^T im2col(x) and the input gradient (zero-padded im2col of dY times the flipped weights on
//              the padded domain, then the reflect-pad band folded back), both as F16X3 wgmma GEMMs.
// Every reduction runs in a fixed order (no atomics on values): two runs give the same bits.
//
// Gradient operands span many decades (1e-6 .. 1e-9 in a real step, below fp16's normal range): before the hi / lo
// split, every dY is multiplied by the power of two that puts its max |.| in [2^13, 2^14), and the GEMM epilogue
// multiplies by the inverse.  Both steps are exact, so the result does not depend on the gradient's scale.
#include <cuda_fp16.h>

#include "common.cuh"
#include "delta.cuh"
#include "tcgemm.cuh"

namespace dtk {

// ---- per-chunk geometry -------------------------------------------------------------------------------------------
struct TrainGeom {
  int B, H[4], W[4], cin[4], cout[4], dil[4], Kp[4];   // conv l: input H[l] x W[l] x cin[l] (cin[0] = 4, padded RGB)
  size_t M(int l) const { return (size_t)B * H[l] * W[l]; }
  int Hc() const { return H[3]; }
  int Wc() const { return W[3]; }
};

static TrainGeom train_geom(int B, int H, int W, const int* ch) {
  TrainGeom g;
  g.B = B;
  const int d[4] = {1, 1, 1, 2};
  for (int l = 0; l < 4; ++l) {
    g.H[l] = H; g.W[l] = W;
    g.cin[l] = l == 0 ? 4 : ch[l];
    g.cout[l] = ch[l + 1];
    g.dil[l] = d[l];
    g.Kp[l] = (int)align_up((size_t)25 * g.cin[l], 8);
    if (l < 3) { H = (H - 1) / 2 + 1; W = (W - 1) / 2 + 1; }
  }
  return g;
}

constexpr int BN_MAX_BLOCKS = 512;   // row blocks of a per-channel reduction (fixed per shape: deterministic)
constexpr int WG_MAX_SPLITS = 256;   // pixel splits of a weight-gradient GEMM (groups of one launch)
// Longest K a gradient GEMM accumulates in the tensor core's fp32 accumulators before the epilogue takes over (in fp32 /
// float64 round-to-nearest sums, in a fixed order).  The wgmma accumulation does not round to nearest: at the shipped
// shapes, chains of ~2e4 pixels gave about twice the weight-gradient error of chains of 2048 (512 gained nothing more).
constexpr int GEMM_K_CHUNK = 2048;
constexpr int WG_TARGET_TILES = 264; // 2 x the SMs of an H100 SXM; a constant, so the summation order never depends on the card

static int bn_blocks(size_t M) { size_t n = (M + 255) / 256; return (int)(n < BN_MAX_BLOCKS ? n : BN_MAX_BLOCKS); }

struct SavedView {
  float* y[4];         // pre-BN conv outputs, NHWC
  double* mean[4];     // per-channel mean used by the forward (batch or running)
  double* invstd[4];   // 1 / sqrt(var + eps)
  SavedView(Arena& ar, const TrainGeom& g) {
    for (int l = 0; l < 4; ++l) {
      y[l] = ar.take<float>(g.M(l) * g.cout[l]);
      mean[l] = ar.take<double>(g.cout[l]);
      invstd[l] = ar.take<double>(g.cout[l]);
    }
  }
};

// ---- BatchNorm ------------------------------------------------------------------------------------------------------
// Per-channel sums over the M rows of an NHWC [M][C] tensor, in float64, block partials in a fixed order:
//   mode 0: (sum x, -)      mode 1: (sum (x - mean), sum (x - mean)^2)      mode 2: (sum g, sum g * xhat(x))
__global__ void bn_reduce_kernel(const float* __restrict__ x, const float* __restrict__ g, size_t M, int C, size_t rows_per_blk,
                                 const double* __restrict__ mean, const double* __restrict__ invstd, int mode,
                                 double2* __restrict__ part) {
  const int tx = threadIdx.x, ty = threadIdx.y;
  const int c = blockIdx.y * 32 + tx;
  const size_t r0 = blockIdx.x * rows_per_blk, r1 = r0 + rows_per_blk < M ? r0 + rows_per_blk : M;
  double s0 = 0.0, s1 = 0.0;
  if (c < C) {
    const double mu = mode ? mean[c] : 0.0, is = mode == 2 ? invstd[c] : 0.0;
    for (size_t m = r0 + ty; m < r1; m += 8) {
      const double v = x[m * C + c];
      if (mode == 0) {
        s0 += v;
      } else if (mode == 1) {
        const double d = v - mu;
        s0 += d; s1 = fma(d, d, s1);
      } else {
        const double gv = g[m * C + c];
        s0 += gv; s1 = fma(gv, (v - mu) * is, s1);
      }
    }
  }
  __shared__ double2 sh[8][32];
  sh[ty][tx] = make_double2(s0, s1);
  __syncthreads();
  if (ty == 0 && c < C) {
    double2 a = sh[0][tx];
    for (int t = 1; t < 8; ++t) { a.x += sh[t][tx].x; a.y += sh[t][tx].y; }
    part[(size_t)blockIdx.x * C + c] = a;
  }
}

__device__ __forceinline__ double2 bn_sum_parts(const double2* part, int nblk, int C, int c) {
  double2 a = make_double2(0.0, 0.0);
  for (int b = 0; b < nblk; ++b) { a.x += part[(size_t)b * C + c].x; a.y += part[(size_t)b * C + c].y; }
  return a;
}

__global__ void bn_mean_kernel(const double2* __restrict__ part, int nblk, int C, size_t M, double* __restrict__ mean) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) mean[c] = bn_sum_parts(part, nblk, C, c).x / (double)M;
}

// corrected two-pass variance; running statistics as torch.nn.BatchNorm2d (momentum, unbiased running_var)
__global__ void bn_var_kernel(const double2* __restrict__ part, int nblk, int C, size_t M, const double* __restrict__ mean,
                              double* __restrict__ invstd, float* __restrict__ run_mean, float* __restrict__ run_var,
                              double momentum, double eps) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double2 s = bn_sum_parts(part, nblk, C, c);
  const double n = (double)M;
  double var = (s.y - s.x * s.x / n) / n;
  var = var > 0.0 ? var : 0.0;
  invstd[c] = 1.0 / sqrt(var + eps);
  run_mean[c] = (float)((1.0 - momentum) * (double)run_mean[c] + momentum * mean[c]);
  run_var[c] = (float)((1.0 - momentum) * (double)run_var[c] + momentum * var * n / (n - 1.0));
}

__global__ void bn_eval_stats_kernel(const float* __restrict__ run_mean, const float* __restrict__ run_var, int C, double eps,
                                     double* __restrict__ mean, double* __restrict__ invstd) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) { mean[c] = run_mean[c]; invstd[c] = 1.0 / sqrt((double)run_var[c] + eps); }
}

// normalised value and the affine of one element (the forward and the reverse pass use this one function)
__device__ __forceinline__ float bn_xhat(float y, double mean, double invstd) { return (float)(((double)y - mean) * invstd); }
__device__ __forceinline__ float bn_affine(float y, double mean, double invstd, float gamma, float beta) {
  return fmaf(bn_xhat(y, mean, invstd), gamma, beta);
}

// BlurPool(stride 2, filt 4) of relu(BN(y)): reflect pad (1, 2, 1, 2), depthwise outer([1,3,3,1]) / 64
__global__ void bn_relu_blur_kernel(const float* __restrict__ y, const double* __restrict__ mean, const double* __restrict__ invstd,
                                    const float* __restrict__ gamma, const float* __restrict__ beta, float* __restrict__ out,
                                    int B, int H, int W, int C, int Ho, int Wo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t total = (size_t)B * Ho * Wo * C;
  if (i >= total) return;
  const int c = (int)(i % C);
  size_t p = i / C;
  const int ox = (int)(p % Wo);
  p /= Wo;
  const int oy = (int)(p % Ho), b = (int)(p / Ho);
  const float f[4] = {1.f / 8.f, 3.f / 8.f, 3.f / 8.f, 1.f / 8.f};
  const double mu = mean[c], is = invstd[c];
  const float ga = gamma[c], be = beta[c];
  float acc = 0.f;
#pragma unroll
  for (int ky = 0; ky < 4; ++ky) {
    const int sy = reflect(2 * oy + ky - 1, H);
#pragma unroll
    for (int kx = 0; kx < 4; ++kx) {
      const int sx = reflect(2 * ox + kx - 1, W);
      const float z = fmaxf(bn_affine(y[(((size_t)b * H + sy) * W + sx) * C + c], mu, is, ga, be), 0.f);
      acc = fmaf(z, f[ky] * f[kx], acc);
    }
  }
  out[i] = acc;
}

// bilinear weights of the token grid along one axis (grid_sample, border, align_corners=True): token i reads CNN
// columns x0 = floor(s[i]) with weight x0 + 1 - s[i], and x0 + 1 (if inside) with weight s[i] - x0
__device__ __forceinline__ void align_axis(float s, int n, int& x0, float& w0, float& w1, bool& ok1) {
  const float f = floorf(s);
  x0 = (int)f; w0 = f + 1.f - s; w1 = s - f; ok1 = x0 + 1 <= n - 1;
}

// residual[b][p][c] = sum over the bilinear corners of BN(y)  (last layer: no ReLU)
__global__ void bn_align_kernel(const float* __restrict__ y, const double* __restrict__ mean, const double* __restrict__ invstd,
                                const float* __restrict__ gamma, const float* __restrict__ beta, const float* __restrict__ ixs,
                                const float* __restrict__ iys, int Hc, int Wc, int C, int h, int w, float* __restrict__ res) {
  const int p = blockIdx.x, b = blockIdx.y;
  const int r = p / w, q = p - r * w;
  int x0, y0; float wx0, wx1, wy0, wy1; bool okx, oky;
  align_axis(ixs[q], Wc, x0, wx0, wx1, okx);
  align_axis(iys[r], Hc, y0, wy0, wy1, oky);
  // ATen grid_sampler_2d: nw = (ix_se - ix) * (iy_se - iy), ...
  const float wnw = wx0 * wy0, wne = wx1 * wy0, wsw = wx0 * wy1, wse = wx1 * wy1;
  const float* base = y + (size_t)b * Hc * Wc * C;
  const float* pnw = base + ((size_t)y0 * Wc + x0) * C;
  const float* pne = pnw + C;
  const float* psw = pnw + (size_t)Wc * C;
  const float* pse = psw + C;
  float* o = res + ((size_t)b * h * w + p) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    const double mu = mean[c], is = invstd[c];
    const float ga = gamma[c], be = beta[c];
    float acc = 0.f;
    acc = fmaf(bn_affine(pnw[c], mu, is, ga, be), wnw, acc);
    if (okx) acc = fmaf(bn_affine(pne[c], mu, is, ga, be), wne, acc);
    if (oky) acc = fmaf(bn_affine(psw[c], mu, is, ga, be), wsw, acc);
    if (okx && oky) acc = fmaf(bn_affine(pse[c], mu, is, ga, be), wse, acc);
    o[c] = acc;
  }
}

// ---- reverse pass: element-wise and gather kernels ------------------------------------------------------------------
// Adjoint of the alignment: dz[b][y][x][c] = sum over the tokens whose bilinear corners touch (y, x) of weight * g.
// The tables are per axis, so the touching tokens are (rows touching y) x (columns touching x); the weight is the
// forward's product (x factor) * (y factor).  Dynamic shared memory: (w + h) x (int + float).
__global__ void align_adjoint_kernel(const float* __restrict__ g, const float* __restrict__ ixs, const float* __restrict__ iys,
                                     int Hc, int Wc, int C, int h, int w, float* __restrict__ dz) {
  extern __shared__ float sh_align[];
  int* cols = reinterpret_cast<int*>(sh_align);
  float* fxs = sh_align + w;
  int* rows = reinterpret_cast<int*>(fxs + w);
  float* fys = fxs + w + h;
  __shared__ int n_cols, n_rows;
  const int x = blockIdx.x, y = blockIdx.y, b = blockIdx.z;
  if (threadIdx.x == 0) {
    int n = 0;
    for (int q = 0; q < w; ++q) {
      int x0; float w0, w1; bool ok1;
      align_axis(ixs[q], Wc, x0, w0, w1, ok1);
      if (x0 == x) { cols[n] = q; fxs[n++] = w0; }
      else if (ok1 && x0 + 1 == x) { cols[n] = q; fxs[n++] = w1; }
    }
    n_cols = n;
    n = 0;
    for (int r = 0; r < h; ++r) {
      int y0; float w0, w1; bool ok1;
      align_axis(iys[r], Hc, y0, w0, w1, ok1);
      if (y0 == y) { rows[n] = r; fys[n++] = w0; }
      else if (ok1 && y0 + 1 == y) { rows[n] = r; fys[n++] = w1; }
    }
    n_rows = n;
  }
  __syncthreads();
  const float* gb = g + (size_t)b * h * w * C;
  float* o = dz + (((size_t)b * Hc + y) * Wc + x) * C;
  for (int c = threadIdx.x; c < C; c += blockDim.x) {
    float acc = 0.f;
    for (int i = 0; i < n_rows; ++i)
      for (int j = 0; j < n_cols; ++j)
        acc = fmaf(fxs[j] * fys[i], gb[((size_t)rows[i] * w + cols[j]) * C + c], acc);
    o[c] = acc;
  }
}

// sum_dz / M and sum_dz*xhat / M for the train-mode dx; d gamma = sum dz*xhat, d beta = sum dz
__global__ void bn_grad_kernel(const double2* __restrict__ part, int nblk, int C, size_t M, double* __restrict__ m_dz,
                               double* __restrict__ m_dzx, float* __restrict__ d_gamma, float* __restrict__ d_beta) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= C) return;
  const double2 s = bn_sum_parts(part, nblk, C, c);
  d_beta[c] = (float)s.x;
  d_gamma[c] = (float)s.y;
  m_dz[c] = s.x / (double)M;
  m_dzx[c] = s.y / (double)M;
}

__global__ void chan_sum_kernel(const double2* __restrict__ part, int nblk, int C, float* __restrict__ out) {
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c < C) out[c] = (float)bn_sum_parts(part, nblk, C, c).x;
}

// in place: dz -> dy = gamma * invstd * (dz - mean(dz) - xhat * mean(dz * xhat))   (train)  |  gamma * invstd * dz  (eval)
__global__ void bn_backward_kernel(const float* __restrict__ y, float* __restrict__ g, size_t n, int C, const double* __restrict__ mean,
                                   const double* __restrict__ invstd, const float* __restrict__ gamma, const double* __restrict__ m_dz,
                                   const double* __restrict__ m_dzx, int train) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % C);
  const double k = (double)gamma[c] * invstd[c];
  double d = g[i];
  if (train) d = d - m_dz[c] - (double)bn_xhat(y[i], mean[c], invstd[c]) * m_dzx[c];
  g[i] = (float)(k * d);
}

// dgrad operand: zero-padded im2col of dY on the padded input domain (Hp = H + 4d, Wp = W + 4d), scaled and split.
// A[m = (b, py, px)][k = (ky*5 + kx)*C + co] = dY[b][py - ky d][px - kx d][co]  (0 outside the H x W output)
__global__ void col_dgrad_split_kernel(const float* __restrict__ dy, const unsigned* __restrict__ amax, __half* __restrict__ hi,
                                       __half* __restrict__ lo, int H, int W, int C, int dil, int Hp, int Wp, size_t m0,
                                       size_t m_count) {
  if (blockIdx.x >= m_count) return;
  const size_t m = m0 + blockIdx.x;
  const int HWp = Hp * Wp;
  const int b = (int)(m / HWp), rem = (int)(m - (size_t)b * HWp);
  const int py = rem / Wp, px = rem - py * Wp;
  const float s = ldexpf(1.f, grad_exp(*amax));
  const int K = 25 * C;
  __half* oh = hi + (size_t)blockIdx.x * K;
  __half* ol = lo + (size_t)blockIdx.x * K;
  for (int k4 = threadIdx.x * 4; k4 < K; k4 += blockDim.x * 4) {
    const int tap = k4 / C, co = k4 - tap * C;   // C % 8 == 0: the 4 elements share the tap
    const int ky = tap / 5, kx = tap - ky * 5;
    const int oy = py - ky * dil, ox = px - kx * dil;
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (oy >= 0 && oy < H && ox >= 0 && ox < W)
      v = __ldg(reinterpret_cast<const float4*>(dy + (((size_t)b * H + oy) * W + ox) * C + co));
    __half h0, h1, h2, h3, l0, l1, l2, l3;
    split16(v.x * s, h0, l0); split16(v.y * s, h1, l1); split16(v.z * s, h2, l2); split16(v.w * s, h3, l3);
    __half2 a = __halves2half2(h0, h1), c = __halves2half2(h2, h3), d = __halves2half2(l0, l1), e = __halves2half2(l2, l3);
    *reinterpret_cast<uint2*>(oh + k4) = make_uint2(*reinterpret_cast<unsigned*>(&a), *reinterpret_cast<unsigned*>(&c));
    *reinterpret_cast<uint2*>(ol + k4) = make_uint2(*reinterpret_cast<unsigned*>(&d), *reinterpret_cast<unsigned*>(&e));
  }
}

// wgrad A operand: dY^T of pixels [p0, p0 + S*Kc), scaled and split: out[s][co][j] = dY[p0 + s*Kc + j][co] (0 past M)
__global__ void dyT_split_kernel(const float* __restrict__ dy, const unsigned* __restrict__ amax, __half* __restrict__ hi,
                                 __half* __restrict__ lo, size_t M, int C, size_t p0, int Kc) {
  __shared__ float tile[32][33];
  const int s = blockIdx.z;
  const int j0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
  const float sc = ldexpf(1.f, grad_exp(*amax));
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const size_t p = p0 + (size_t)s * Kc + j0 + r;
    const int c = c0 + threadIdx.x;
    tile[r][threadIdx.x] = (j0 + r < Kc && p < M && c < C) ? dy[p * C + c] * sc : 0.f;
  }
  __syncthreads();
  for (int r = threadIdx.y; r < 32; r += blockDim.y) {
    const int c = c0 + r, j = j0 + threadIdx.x;
    if (c < C && j < Kc) {
      __half h, l;
      split16(tile[threadIdx.x][r], h, l);
      const size_t o = ((size_t)s * C + c) * Kc + j;
      hi[o] = h; lo[o] = l;
    }
  }
}

// wgrad B operand: transposed im2col (reflect pad, dilation) of the layer input, split:
// out[s][k][j] = x[reflect tap k of pixel p0 + s*Kc + j] for k < 25*Cin (0 for k in [25 Cin, Kp) and pixels past M)
constexpr int COLT_K = 32;
__global__ void colT_split_kernel(const float* __restrict__ x, __half* __restrict__ hi, __half* __restrict__ lo, int H, int W,
                                  int Cin, int dil, int Kp, size_t M, size_t p0, int Kc) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  const int s = blockIdx.z, k0 = blockIdx.y * COLT_K;
  if (j >= Kc) return;
  const size_t p = p0 + (size_t)s * Kc + j;
  const bool valid = p < M;
  const int HW = H * W;
  const int b = valid ? (int)(p / HW) : 0, rem = valid ? (int)(p - (size_t)b * HW) : 0;
  const int py = rem / W, px = rem - py * W;
  const int K = 25 * Cin;
  for (int k = k0; k < k0 + COLT_K && k < Kp; ++k) {
    float v = 0.f;
    if (valid && k < K) {
      const int tap = k / Cin, ci = k - tap * Cin;
      const int ky = tap / 5, kx = tap - ky * 5;
      const int sy = reflect(py + (ky - 2) * dil, H), sx = reflect(px + (kx - 2) * dil, W);
      v = x[(((size_t)b * H + sy) * W + sx) * Cin + ci];
    }
    __half h, l;
    split16(v, h, l);
    const size_t o = ((size_t)s * Kp + k) * Kc + j;
    hi[o] = h; lo[o] = l;
  }
}

// the padded-domain indices whose reflection is `v` (pad `pad` on both sides of an axis of n): up to three
__device__ __forceinline__ int reflect_sources(int v, int n, int pad, int* q) {
  int k = 0;
  q[k++] = v + pad;
  if (v >= 1 && v <= pad) q[k++] = pad - v;
  if (v <= n - 2 && v >= n - 1 - pad) q[k++] = 2 * (n - 1) - v + pad;
  return k;
}

// fold the reflect-pad band of the padded-domain input gradient back into the interior: dx[y][x] = sum of dxp over the
// padded positions that reflect onto (y, x)
__global__ void fold_reflect_kernel(const float* __restrict__ dxp, float* __restrict__ dx, int B, int H, int W, int C, int pad) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int C4 = C >> 2;
  if (i >= (size_t)B * H * W * C4) return;
  const int c4 = (int)(i % C4);
  size_t p = i / C4;
  const int x = (int)(p % W);
  p /= W;
  const int y = (int)(p % H), b = (int)(p / H);
  const int Hp = H + 2 * pad, Wp = W + 2 * pad;
  int qy[3], qx[3];
  const int ny = reflect_sources(y, H, pad, qy), nx = reflect_sources(x, W, pad, qx);
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
  for (int a = 0; a < ny; ++a)
    for (int e = 0; e < nx; ++e) {
      const float4 v = __ldg(reinterpret_cast<const float4*>(dxp + (((size_t)b * Hp + qy[a]) * Wp + qx[e]) * C) + c4);
      acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
    }
  reinterpret_cast<float4*>(dx)[i] = acc;
}

// BlurPool taps that read input row v (pad 1 before, 2 after, stride 2, 4 taps): (output row, tap) pairs, up to six
__device__ __forceinline__ int blur_sources(int v, int n, int no, int* o, int* t) {
  int q[3], nq = 0;
  q[nq++] = v;
  if (v == 1) q[nq++] = -1;
  if (v <= n - 2 && 2 * (n - 1) - v <= 2 * no) q[nq++] = 2 * (n - 1) - v;
  int k = 0;
  for (int a = 0; a < nq; ++a)
    for (int oo = (q[a] - 2) / 2 - 1; oo <= (q[a] + 1) / 2 + 1; ++oo) {
      const int tap = q[a] + 1 - 2 * oo;
      if (oo >= 0 && oo < no && tap >= 0 && tap < 4) { o[k] = oo; t[k++] = tap; }
    }
  return k;
}

// dz_prev = relu'(BN(y_prev)) * BlurPool^T(dx): the adjoint of the blur (reflect fold included) and the ReLU mask
__global__ void blur_adjoint_relu_kernel(const float* __restrict__ dx, const float* __restrict__ y, const double* __restrict__ mean,
                                         const double* __restrict__ invstd, const float* __restrict__ gamma,
                                         const float* __restrict__ beta, float* __restrict__ dz, int B, int H, int W, int C,
                                         int Ho, int Wo) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * H * W * C) return;
  const int c = (int)(i % C);
  size_t p = i / C;
  const int x = (int)(p % W);
  p /= W;
  const int yy = (int)(p % H), b = (int)(p / H);
  if (!(bn_affine(y[i], mean[c], invstd[c], gamma[c], beta[c]) > 0.f)) { dz[i] = 0.f; return; }
  const float f[4] = {1.f / 8.f, 3.f / 8.f, 3.f / 8.f, 1.f / 8.f};
  int oy[6], ty[6], ox[6], tx[6];
  const int ny = blur_sources(yy, H, Ho, oy, ty), nx = blur_sources(x, W, Wo, ox, tx);
  float acc = 0.f;
  for (int a = 0; a < ny; ++a)
    for (int e = 0; e < nx; ++e)
      acc = fmaf(dx[(((size_t)b * Ho + oy[a]) * Wo + ox[e]) * C + c], f[ty[a]] * f[tx[e]], acc);
  dz[i] = acc;
}

// acc[i] (+)= sum_s part[s][i] in float64, s in order; the last chunk writes dW = acc
__global__ void wgrad_reduce_kernel(const float* __restrict__ part, int S, size_t n, double* __restrict__ acc, int first,
                                    float* __restrict__ dw) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double a = first ? 0.0 : acc[i];
  for (int s = 0; s < S; ++s) a += part[(size_t)s * n + i];
  if (dw) dw[i] = (float)a; else acc[i] = a;
}

// ---- GEMMs -----------------------------------------------------------------------------------------------------------
// out[(g * rows_per_group + row0 + r) * ld + col] (+)= acc * 2^-e, e = the operand scale of grad_exp(*amax)
struct EpiScaled {
  float* out; const unsigned* amax; size_t ld, row0; int rows_per_group, accumulate;
  struct State { float inv; };
  __device__ __forceinline__ void tile_begin(State& s) const { s.inv = ldexpf(1.f, -grad_exp(*amax)); }
  __device__ __forceinline__ void tile_end(State&, int, int, int) const {}
  __device__ __forceinline__ void operator()(State& s, int g, int r, int col0, const float (&f)[32], int ncols) const {
    float* o = out + ((size_t)g * rows_per_group + row0 + r) * ld + col0;
#pragma unroll
    for (int i = 0; i < 32; i += 4)
      if (i < ncols)   // N % 8 == 0 -> ncols % 4 == 0
      {
        float4 v = make_float4(f[i] * s.inv, f[i + 1] * s.inv, f[i + 2] * s.inv, f[i + 3] * s.inv);
        if (accumulate) {
          const float4 p = *reinterpret_cast<const float4*>(o + i);
          v.x += p.x; v.y += p.y; v.z += p.z; v.w += p.w;
        }
        *reinterpret_cast<float4*>(o + i) = v;
      }
  }
};

// pixel splits of a layer's weight-gradient GEMM: S groups (a fixed function of the shape) of Kc pixels per launch
static void wgrad_split(const TrainGeom& g, int l, size_t col_elems, int* S_out, int* Kc_out) {
  const int tiles = cdiv(g.cout[l], TC_BM) * cdiv(g.Kp[l], tc_bn(g.Kp[l]));
  int S = cdiv(WG_TARGET_TILES, tiles);
  S = S < 1 ? 1 : (S > WG_MAX_SPLITS ? WG_MAX_SPLITS : S);
  const size_t per = (size_t)S * (g.cout[l] + g.Kp[l]);
  size_t kc = (col_elems - 128) / per / 64 * 64;
  const size_t need = align_up((g.M(l) + S - 1) / S, 64);
  if (kc > need) kc = need;
  if (kc > GEMM_K_CHUNK) kc = GEMM_K_CHUNK;
  *S_out = S; *Kc_out = (int)kc;
}

static size_t wgrad_part_elems(const TrainGeom& g, size_t col_elems) {
  size_t best = 0;
  for (int l = 0; l < 4; ++l) {
    int S, Kc;
    wgrad_split(g, l, col_elems, &S, &Kc);
    const size_t n = (size_t)S * g.cout[l] * g.Kp[l];
    if (n > best) best = n;
  }
  return best;
}

// fp16 im2col scratch (elements per half): the forward's CONV_TC_ROWS rows of the widest K, and at least what one
// launch of each gradient GEMM needs -- TC_BM rows of an input-gradient im2col (K = 25 C_out) and 64 pixels of every
// weight-gradient split -- so the backward never runs out of scratch for any legal widths
static size_t col_elems_of(const int* channels) {
  size_t n = CONV_TC_ROWS * delta_conv_kmax(channels);
  for (int l = 0; l < 4; ++l) {
    const size_t cout = channels[l + 1], kp = align_up((size_t)25 * (l == 0 ? 4 : channels[l]), 8);
    const size_t wg = 128 + (size_t)64 * WG_MAX_SPLITS * (cout + kp);
    const size_t dg = l > 0 ? (size_t)TC_BM * 25 * cout : 0;
    n = wg > n ? wg : n;
    n = dg > n ? dg : n;
  }
  return n;
}

static size_t max_input_elems(const TrainGeom& g) {
  size_t best = 0;
  for (int l = 0; l < 4; ++l) { size_t n = g.M(l) * g.cin[l]; if (n > best) best = n; }
  return best;
}

static size_t max_output_elems(const TrainGeom& g) {
  size_t best = 0;
  for (int l = 0; l < 4; ++l) { size_t n = g.M(l) * g.cout[l]; if (n > best) best = n; }
  return best;
}

static size_t max_padded_elems(const TrainGeom& g) {
  size_t best = 0;
  for (int l = 1; l < 4; ++l) {
    size_t n = (size_t)g.B * (g.H[l] + 4 * g.dil[l]) * (g.W[l] + 4 * g.dil[l]) * g.cin[l];
    if (n > best) best = n;
  }
  return best;
}

// BN statistics of layer l (train: batch statistics + running update; eval: running statistics)
static int bn_stats(const float* y, size_t M, int C, int train, float* run_mean, float* run_var, double momentum, double eps,
                    double* mean, double* invstd, double2* part, cudaStream_t st) {
  ProfRange pr(PROF_DELTA_BN, st);
  const unsigned cb = (unsigned)cdiv(C, 128);
  if (!train) {
    bn_eval_stats_kernel<<<cb, 128, 0, st>>>(run_mean, run_var, C, eps, mean, invstd);
    DTK_LAUNCHED();
    return DINOTRK_OK;
  }
  const int nblk = bn_blocks(M);
  const size_t rpb = (M + nblk - 1) / nblk;
  const dim3 grid(nblk, cdiv(C, 32)), block(32, 8);
  bn_reduce_kernel<<<grid, block, 0, st>>>(y, nullptr, M, C, rpb, nullptr, nullptr, 0, part);
  DTK_LAUNCHED();
  bn_mean_kernel<<<cb, 128, 0, st>>>(part, nblk, C, M, mean);
  DTK_LAUNCHED();
  bn_reduce_kernel<<<grid, block, 0, st>>>(y, nullptr, M, C, rpb, mean, nullptr, 1, part);
  DTK_LAUNCHED();
  bn_var_kernel<<<cb, 128, 0, st>>>(part, nblk, C, M, mean, invstd, run_mean, run_var, momentum, eps);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// the input of conv l: frames (l = 0) or BlurPool(relu(BN(y_{l-1})))
static int layer_input(const float* frames, const TrainGeom& g, int l, const SavedView& sv, const float* const* gamma,
                       const float* const* beta, float* x, cudaStream_t st) {
  if (l == 0) return launch_rgb_to_nhwc4(frames, x, g.B, g.H[0] * g.W[0], st);
  const int p = l - 1;
  const size_t tot = g.M(l) * g.cin[l];
  bn_relu_blur_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(sv.y[p], sv.mean[p], sv.invstd[p], gamma[p], beta[p], x,
                                                                     g.B, g.H[p], g.W[p], g.cout[p], g.H[l], g.W[l]);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

static int check_train_args(const char* who, int B, int H, int W, const int* channels, const float* ixs, const float* iys,
                            int h, int w) {
  DTK_CHECK_ARG(channels && ixs && iys, "%s: null pointer", who);
  DTK_CHECK_ARG(B >= 0 && h > 0 && w > 0, "%s: bad sizes", who);
  DTK_CHECK_ARG(channels[0] == 3, "%s: input must be RGB", who);
  for (int l = 1; l <= 4; ++l) DTK_CHECK_ARG(channels[l] > 0 && channels[l] % 8 == 0, "%s: channel counts must be multiples of 8", who);
  // reflect padding needs pad < size (torch rejects the same): conv pad 2d, BlurPool pad 2
  const TrainGeom g = train_geom(B, H, W, channels);
  for (int l = 0; l < 4; ++l)
    DTK_CHECK_ARG(g.H[l] > 2 * g.dil[l] && g.W[l] > 2 * g.dil[l] && (l == 3 || (g.H[l] > 2 && g.W[l] > 2)),
                  "%s: %d x %d frames are too small for the reflect padding of layer %d", who, H, W, l + 1);
  return DINOTRK_OK;
}

static int max_channels(const int* channels) {
  int c = 0;
  for (int l = 1; l <= 4; ++l) c = channels[l] > c ? channels[l] : c;
  return c;
}

struct FwdWs {
  float* x; __half* col_hi; __half* col_lo; int* plan; double2* part;
  FwdWs(Arena& ar, const TrainGeom& g, const int* channels) {
    x = ar.take<float>(max_input_elems(g));
    col_hi = ar.take<__half>(col_elems_of(channels));
    col_lo = ar.take<__half>(col_elems_of(channels));
    plan = ar.take<int>(16);
    part = ar.take<double2>((size_t)BN_MAX_BLOCKS * max_channels(channels));
  }
};

struct BwdWs {
  float* g; float* x; float* xp; __half* col_hi; __half* col_lo; float* wpart; double* wacc; int* plan; double2* part;
  double* m_dz; double* m_dzx; unsigned* amax;
  BwdWs(Arena& ar, const TrainGeom& tg, const int* channels) {
    const size_t ce = col_elems_of(channels);
    g = ar.take<float>(max_output_elems(tg));
    x = ar.take<float>(max_input_elems(tg));
    xp = ar.take<float>(max_padded_elems(tg));
    col_hi = ar.take<__half>(ce);
    col_lo = ar.take<__half>(ce);
    wpart = ar.take<float>(wgrad_part_elems(tg, ce));
    size_t wmax = 0;
    for (int l = 0; l < 4; ++l) wmax = (size_t)tg.cout[l] * tg.Kp[l] > wmax ? (size_t)tg.cout[l] * tg.Kp[l] : wmax;
    wacc = ar.take<double>(wmax);
    plan = ar.take<int>(4 * WG_MAX_SPLITS + 1);
    part = ar.take<double2>((size_t)BN_MAX_BLOCKS * max_channels(channels));
    m_dz = ar.take<double>(max_channels(channels));
    m_dzx = ar.take<double>(max_channels(channels));
    amax = ar.take<unsigned>(1);
  }
};

}  // namespace dtk

using namespace dtk;

extern "C" {

size_t dinotrk_delta_train_saved_bytes(int B, int H, int W, const int* channels) {
  if (!channels || B < 0) return 0;
  return layout_end<SavedView>(train_geom(B, H, W, channels));
}

size_t dinotrk_delta_train_forward_workspace_bytes(int B, int H, int W, const int* channels) {
  if (!channels || B < 0) return 0;
  return layout_end<FwdWs>(train_geom(B, H, W, channels), channels);
}

size_t dinotrk_delta_train_backward_workspace_bytes(int B, int H, int W, const int* channels) {
  if (!channels || B < 0) return 0;
  return layout_end<BwdWs>(train_geom(B, H, W, channels), channels);
}

static bool all_set(const void* const* a, int from = 0) {
  if (!a) return false;
  for (int l = from; l < 4; ++l) if (!a[l]) return false;
  return true;
}

int dinotrk_delta_train_forward(const float* frames, int B, int H, int W, const int* channels, const void* const* wgt_hi,
                                const void* const* wgt_lo, const float* const* conv_bias, const float* const* bn_weight,
                                const float* const* bn_bias, float* const* running_mean, float* const* running_var,
                                int training, float momentum, float eps, const float* ixs, const float* iys, int h, int w,
                                float* residual_tpc, void* saved, size_t saved_bytes, void* workspace, size_t workspace_bytes,
                                void* stream) {
  NvtxRange nvtx_range("dinotrk.delta_train_forward");
  if (int rc = check_train_args("delta_train_forward", B, H, W, channels, ixs, iys, h, w)) return rc;
  DTK_CHECK_ARG(frames && residual_tpc && saved && workspace && all_set((const void* const*)wgt_hi) &&
                all_set((const void* const*)wgt_lo) && all_set((const void* const*)conv_bias) &&
                all_set((const void* const*)bn_weight) && all_set((const void* const*)bn_bias),
                "delta_train_forward: null pointer");
  DTK_CHECK_ARG(all_set((const void* const*)running_mean) && all_set((const void* const*)running_var),
                "delta_train_forward: null running statistics");
  DTK_CHECK_ARG(momentum >= 0.f && momentum <= 1.f && eps > 0.f, "delta_train_forward: bad momentum / eps");
  DTK_CHECK_ARG(saved_bytes >= dinotrk_delta_train_saved_bytes(B, H, W, channels), "delta_train_forward: saved buffer too small");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_delta_train_forward_workspace_bytes(B, H, W, channels),
                "delta_train_forward: workspace too small");
  if (B == 0) return DINOTRK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const TrainGeom g = train_geom(B, H, W, channels);
  Arena saved_ar(saved), ar(workspace);
  const SavedView sv(saved_ar, g);
  const FwdWs ws(ar, g, channels);
  for (int l = 0; l < 4; ++l) {
    {
      ProfRange pr(PROF_DELTA_BN, st);
      if (int rc = layer_input(frames, g, l, sv, bn_weight, bn_bias, ws.x, st)) return rc;
    }
    ConvShape cs{B, g.H[l], g.W[l], g.cin[l], g.cout[l], g.dil[l], 0};
    if (int rc = launch_conv_tc(ws.x, (const __half*)wgt_hi[l], (const __half*)wgt_lo[l], conv_bias[l], sv.y[l], cs, g.Kp[l],
                                ws.col_hi, ws.col_lo, ws.plan, st, PROF_DELTA_TRAIN_CONV))
      return rc;
    if (int rc = bn_stats(sv.y[l], g.M(l), g.cout[l], training, running_mean[l], running_var[l], momentum, eps, sv.mean[l],
                          sv.invstd[l], ws.part, st))
      return rc;
  }
  ProfRange pr(PROF_ALIGN, st);
  bn_align_kernel<<<dim3(h * w, B), 128, 0, st>>>(sv.y[3], sv.mean[3], sv.invstd[3], bn_weight[3], bn_bias[3], ixs, iys,
                                                  g.Hc(), g.Wc(), g.cout[3], h, w, residual_tpc);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_delta_train_backward(const float* frames, int B, int H, int W, const int* channels, const void* const* wgtT_hi,
                                 const void* const* wgtT_lo, const float* const* bn_weight, const float* const* bn_bias,
                                 int training, const float* ixs, const float* iys, int h, int w, const float* grad_residual_tpc,
                                 const void* saved, size_t saved_bytes, float* const* grad_wgt, float* const* grad_bias,
                                 float* const* grad_bn_weight, float* const* grad_bn_bias, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  NvtxRange nvtx_range("dinotrk.delta_train_backward");
  if (int rc = check_train_args("delta_train_backward", B, H, W, channels, ixs, iys, h, w)) return rc;
  DTK_CHECK_ARG(frames && grad_residual_tpc && saved && workspace && all_set(wgtT_hi, 1) && all_set(wgtT_lo, 1) &&
                all_set((const void* const*)bn_weight) && all_set((const void* const*)bn_bias) &&
                all_set((const void* const*)grad_wgt) && all_set((const void* const*)grad_bias) &&
                all_set((const void* const*)grad_bn_weight) && all_set((const void* const*)grad_bn_bias),
                "delta_train_backward: null pointer");
  DTK_CHECK_ARG(saved_bytes >= dinotrk_delta_train_saved_bytes(B, H, W, channels), "delta_train_backward: saved buffer too small");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_delta_train_backward_workspace_bytes(B, H, W, channels),
                "delta_train_backward: workspace too small");
  if (B == 0) return DINOTRK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const TrainGeom g = train_geom(B, H, W, channels);
  Arena saved_ar(const_cast<void*>(saved)), ar(workspace);
  const SavedView sv(saved_ar, g);
  const BwdWs ws(ar, g, channels);
  const size_t ce = col_elems_of(channels);
  {
    ProfRange pr(PROF_ALIGN, st);
    const size_t sh = (size_t)(w + h) * 8;
    align_adjoint_kernel<<<dim3(g.Wc(), g.Hc(), B), 128, sh, st>>>(grad_residual_tpc, ixs, iys, g.Hc(), g.Wc(), g.cout[3], h, w,
                                                                    ws.g);
    DTK_LAUNCHED();
  }
  for (int l = 3; l >= 0; --l) {
    const size_t M = g.M(l);
    const int C = g.cout[l];
    const unsigned cb = (unsigned)cdiv(C, 128);
    const int nblk = bn_blocks(M);
    const size_t rpb = (M + nblk - 1) / nblk;
    const dim3 rgrid(nblk, cdiv(C, 32)), rblock(32, 8);
    {   // ws.g: d loss / d BN output (ReLU mask applied) -> d loss / d conv output; d gamma, d beta, d bias
      ProfRange pr(PROF_DELTA_BN, st);
      bn_reduce_kernel<<<rgrid, rblock, 0, st>>>(sv.y[l], ws.g, M, C, rpb, sv.mean[l], sv.invstd[l], 2, ws.part);
      DTK_LAUNCHED();
      bn_grad_kernel<<<cb, 128, 0, st>>>(ws.part, nblk, C, M, ws.m_dz, ws.m_dzx, grad_bn_weight[l], grad_bn_bias[l]);
      DTK_LAUNCHED();
      bn_backward_kernel<<<(unsigned)((M * C + 255) / 256), 256, 0, st>>>(sv.y[l], ws.g, M * C, C, sv.mean[l], sv.invstd[l],
                                                                          bn_weight[l], ws.m_dz, ws.m_dzx, training);
      DTK_LAUNCHED();
      bn_reduce_kernel<<<rgrid, rblock, 0, st>>>(ws.g, nullptr, M, C, rpb, nullptr, nullptr, 0, ws.part);
      DTK_LAUNCHED();
      chan_sum_kernel<<<cb, 128, 0, st>>>(ws.part, nblk, C, grad_bias[l]);
      DTK_LAUNCHED();
      DTK_CUDA(cudaMemsetAsync(ws.amax, 0, sizeof(unsigned), st));
      if (int rc = launch_amax(ws.g, M * C, ws.amax, 1024, st)) return rc;
      if (int rc = layer_input(frames, g, l, sv, bn_weight, bn_bias, ws.x, st)) return rc;
    }
    {   // weight gradient: pixel chunks of S x Kc, S groups per launch, partials summed in order
      int S, Kc;
      wgrad_split(g, l, ce, &S, &Kc);
      const int Kp = g.Kp[l];
      __half* a_hi = ws.col_hi; __half* a_lo = ws.col_lo;
      const size_t b_off = align_up((size_t)S * C * Kc, 64);
      __half* b_hi = ws.col_hi + b_off; __half* b_lo = ws.col_lo + b_off;
      const size_t chunk = (size_t)S * Kc;
      for (size_t p0 = 0; p0 < M; p0 += chunk) {
        {
          ProfRange pr(PROF_DELTA_WGRAD, st);
          dyT_split_kernel<<<dim3(cdiv(Kc, 32), cdiv(C, 32), S), dim3(32, 8), 0, st>>>(ws.g, ws.amax, a_hi, a_lo, M, C, p0, Kc);
          DTK_LAUNCHED();
          colT_split_kernel<<<dim3(cdiv(Kc, 128), cdiv(Kp, COLT_K), S), 128, 0, st>>>(ws.x, b_hi, b_lo, g.H[l], g.W[l], g.cin[l],
                                                                                      g.dil[l], Kp, M, p0, Kc);
          DTK_LAUNCHED();
        }
        {   // S groups: group s = the C rows of dY^T chunk s against the im2col^T chunk s
          ProfRange pr(PROF_DELTA_WGRAD, st);
          const TcPlan pl{ws.plan, ws.plan + S, ws.plan + 2 * S, ws.plan + 3 * S};
          if (int rc = launch_tc_plan(pl, S, C, C, 0, 0, TC_BM, st)) return rc;
          EpiScaled epi{ws.wpart, ws.amax, (size_t)Kp, 0, C, 0};
          if (int rc = tc_launch_bn<TcMode::F16X3>({a_hi, a_lo, (uint64_t)S * C, (uint64_t)Kc, b_hi, b_lo, (uint64_t)S, (uint64_t)Kc},
                                                   pl.problem(S, Kp, Kc), S * cdiv(C, TC_BM), epi, st))
            return rc;
        }
        ProfRange pr(PROF_DELTA_WGRAD, st);
        const size_t n = (size_t)C * Kp;
        wgrad_reduce_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws.wpart, S, n, ws.wacc, p0 == 0,
                                                                         p0 + chunk >= M ? grad_wgt[l] : nullptr);
        DTK_LAUNCHED();
      }
    }
    if (l == 0) break;
    {   // input gradient on the padded domain, row chunks, then the reflect band folded back
      const int d = g.dil[l], Hp = g.H[l] + 4 * d, Wp = g.W[l] + 4 * d, Kd = 25 * C, N = g.cin[l];
      const size_t Mp = (size_t)B * Hp * Wp;
      const size_t rows_max = ce / Kd / TC_BM * TC_BM;   // >= TC_BM by col_elems_of
      for (size_t m0 = 0; m0 < Mp; m0 += rows_max) {
        const size_t rows = Mp - m0 < rows_max ? Mp - m0 : rows_max;
        {
          ProfRange pr(PROF_DELTA_DGRAD, st);
          col_dgrad_split_kernel<<<(unsigned)rows, 128, 0, st>>>(ws.g, ws.amax, ws.col_hi, ws.col_lo, g.H[l], g.W[l], C, d, Hp,
                                                                 Wp, m0, rows);
          DTK_LAUNCHED();
        }
        for (int k0 = 0; k0 < Kd; k0 += GEMM_K_CHUNK) {   // K slices summed into the output in order
          const int kc = Kd - k0 < GEMM_K_CHUNK ? Kd - k0 : GEMM_K_CHUNK;
          ProfRange pr(PROF_DELTA_DGRAD, st);
          const TcPlan pl{ws.plan, ws.plan + 1, ws.plan + 2, ws.plan + 3};
          if (int rc = launch_tc_plan(pl, 1, (int)rows, 0, 0, 0, TC_BM, st)) return rc;
          EpiScaled epi{ws.xp, ws.amax, (size_t)N, m0, 0, k0 > 0};
          if (int rc = tc_launch_bn<TcMode::F16X3>({ws.col_hi + k0, ws.col_lo + k0, rows, (uint64_t)Kd, (const __half*)wgtT_hi[l] + k0,
                                                    (const __half*)wgtT_lo[l] + k0, 1, (uint64_t)Kd},
                                                   pl.problem(1, N, kc), cdiv((int)rows, TC_BM), epi, st))
            return rc;
        }
      }
      ProfRange pr(PROF_DELTA_DGRAD, st);
      const size_t n4 = g.M(l) * N / 4;
      fold_reflect_kernel<<<(unsigned)((n4 + 255) / 256), 256, 0, st>>>(ws.xp, ws.x, B, g.H[l], g.W[l], N, 2 * d);
      DTK_LAUNCHED();
    }
    {   // BlurPool adjoint + ReLU mask of layer l - 1: ws.g = d loss / d BN output of layer l - 1
      ProfRange pr(PROF_DELTA_BN, st);
      const int p = l - 1;
      const size_t n = g.M(p) * g.cout[p];
      blur_adjoint_relu_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws.x, sv.y[p], sv.mean[p], sv.invstd[p], bn_weight[p],
                                                                            bn_bias[p], ws.g, B, g.H[p], g.W[p], g.cout[p],
                                                                            g.H[l], g.W[l]);
      DTK_LAUNCHED();
    }
  }
  return DINOTRK_OK;
}

}  // extern "C"

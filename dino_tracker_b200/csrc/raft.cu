// RAFT-large optical flow (torchvision models/optical_flow/raft.py, eval mode) on the split-precision wgmma GEMM.
//
// Activations are NHWC fp32.  Every convolution is an explicit im2col (zero padding, stride; the fp16 hi / lo split on
// the fly) in chunks of RAFT_ROWS output pixels, feeding the grouped F16X3 GEMM (tcgemm.cuh) with K-major weights
// [Np][Kp] (k = (ky * kw + kx) * C_in + ci, the input channels in torchvision's concatenation order).  Epilogues fuse
// the weights' power-of-two scale, the bias, ReLU, tanh / ReLU of the context split, the GRU gates and the flow update.
//
//   encode:  per frame, the feature encoder (InstanceNorm) and the context encoder (BatchNorm folded into the weights on
//            the host).  A normalised convolution output is kept raw with its per-channel (mean, rstd); the
//            normalise + ReLU is applied by its consumer (the next im2col, or the residual kernel).
//   flow:    for a batch of pairs (i, j): level 0 of the correlation pyramid = fmap_i fmap_jᵀ / 16 (F16X3, or the exact
//            fp32 GEMM when the caller gives no hi / lo split), three 2 x 2 average pools, then the update loop on
//            M = pairs * h * w rows; the mask predictor and the convex upsampling run after the last update only.
#include <cuda_fp16.h>

#include "common.cuh"
#include "tcgemm.cuh"

namespace dtk {

constexpr size_t RAFT_ROWS = 32768;    // im2col rows per GEMM pass (bounds the fp16 scratch)
constexpr int RAFT_NCH = 64;           // pixel chunks of the InstanceNorm partial sums
constexpr int RAFT_KMAX_ENC = 1152;    // widest encoder K (3 x 3 x 128)
constexpr int RAFT_KMAX_UPD = 2304;    // widest update-block K (3 x 3 x 256)
constexpr int RAFT_HX = 384;           // hx row: h (128) | context (128) | motion (126) | flow (2)
constexpr int RAFT_CORR_K = 328;       // 4 levels x 81 taps, padded to a multiple of 8

struct RaftConv { int kh, kw, stride, cin, cout; };

// torchvision's parameter order (include/dinotrk.h: DINOTRK_RAFT_*); the GRU's convz and convr are one [z; r] matrix
static const RaftConv kConv[DINOTRK_RAFT_NCONV] = {
#define ENC {7, 7, 2, 3, 64}, {3, 3, 1, 64, 64}, {3, 3, 1, 64, 64}, {3, 3, 1, 64, 64}, {3, 3, 1, 64, 64},               \
            {3, 3, 2, 64, 96}, {3, 3, 1, 96, 96}, {1, 1, 2, 64, 96}, {3, 3, 1, 96, 96}, {3, 3, 1, 96, 96},               \
            {3, 3, 2, 96, 128}, {3, 3, 1, 128, 128}, {1, 1, 2, 96, 128}, {3, 3, 1, 128, 128}, {3, 3, 1, 128, 128},       \
            {1, 1, 1, 128, 256}
    ENC, ENC,
#undef ENC
    {1, 1, 1, 324, 256}, {3, 3, 1, 256, 192}, {7, 7, 1, 2, 128}, {3, 3, 1, 128, 64}, {3, 3, 1, 256, 126},
    {1, 5, 1, 384, 256}, {1, 5, 1, 384, 128}, {5, 1, 1, 384, 256}, {5, 1, 1, 384, 128},
    {3, 3, 1, 128, 256}, {3, 3, 1, 256, 2},
    {3, 3, 1, 128, 256}, {1, 1, 1, 256, 576}};

static inline int conv_kp(const RaftConv& c) { return (int)align_up((size_t)c.kh * c.kw * c.cin, 8); }
// weight rows padded so that the GEMM's N tile never exceeds N
static inline int conv_np(int cout) { return cout <= 64 ? 64 : cout <= 128 ? 128 : (int)align_up(cout, 256); }

// ---- im2col ----------------------------------------------------------------------------------------------------------
// One input of a (possibly concatenated) im2col: pixel (img, y, x) channel c at p[((img * H + y) * W + x) * pitch + c].
// aff (optional): per (img, channel) (mean, rstd) of a normalisation; the value is then relu((v - mean) * rstd).
struct ColSrc { const float* p; int C, pitch; const float2* aff; };
struct ColGeom { int Hin, Win, Hout, Wout, kh, kw, stride, ph, pw, Kp; };

// Power of two that puts the row's max |v| in [2^13, 2^14) (1 for a zero row), reduced over the block (blockDim 128):
// every operand row is split after this scale, so its fp16 lo halves stay normal numbers, and the GEMM's row is
// multiplied back by the inverse (exact).  Per row, so a row's bits do not depend on the other rows of a batch.
__device__ __forceinline__ float raft_row_scale(float local_max, float* inv) {
  __shared__ float red[4];
  local_max = warp_max(local_max);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = local_max;
  __syncthreads();
  const float m = fmaxf(fmaxf(red[0], red[1]), fmaxf(red[2], red[3]));
  const int e = grad_exp(__float_as_uint(m));
  *inv = ldexpf(1.f, -e);
  return ldexpf(1.f, e);
}

// Row r of the chunk: the operand row scaled by a power of two (raft_row_scale), whose inverse goes to rs[r]
__global__ void __launch_bounds__(128) raft_im2col_kernel(ColSrc s0, ColSrc s1, ColGeom g, __half* __restrict__ hi,
                                                          __half* __restrict__ lo, float* __restrict__ rs, size_t m0) {
  const size_t m = m0 + blockIdx.x;
  const int HWo = g.Hout * g.Wout;
  const int img = (int)(m / HWo), rem = (int)(m - (size_t)img * HWo);
  const int oy = rem / g.Wout, ox = rem - oy * g.Wout;
  const int cin = s0.C + s1.C, K = g.kh * g.kw * cin;
  __half* oh = hi + (size_t)blockIdx.x * g.Kp;
  __half* ol = lo + (size_t)blockIdx.x * g.Kp;
  auto val = [&](int k) {
    float v = 0.f;
    if (k < K) {
      const int tap = k / cin, ci = k - tap * cin;
      const int ky = tap / g.kw, kx = tap - ky * g.kw;
      const int iy = oy * g.stride - g.ph + ky, ix = ox * g.stride - g.pw + kx;
      if (iy >= 0 && iy < g.Hin && ix >= 0 && ix < g.Win) {
        const size_t pix = ((size_t)img * g.Hin + iy) * g.Win + ix;
        if (ci < s0.C) {
          v = __ldg(s0.p + pix * s0.pitch + ci);
          if (s0.aff) { const float2 a = s0.aff[img * s0.C + ci]; v = fmaxf(__fmul_rn(__fsub_rn(v, a.x), a.y), 0.f); }
        } else {
          v = __ldg(s1.p + pix * s1.pitch + (ci - s0.C));
        }
      }
    }
    return v;
  };
  float mx = 0.f;
  for (int k = threadIdx.x; k < K; k += blockDim.x) mx = fmaxf(mx, fabsf(val(k)));
  float inv;
  const float sc = raft_row_scale(mx, &inv);
  if (threadIdx.x == 0) rs[blockIdx.x] = inv;
  for (int k = threadIdx.x; k < g.Kp; k += blockDim.x) split16(val(k) * sc, oh[k], ol[k]);
}

// ---- epilogues -------------------------------------------------------------------------------------------------------
enum RaftAct { ACT_NONE = 0, ACT_RELU, ACT_CTX, ACT_ZR, ACT_Q, ACT_FLOW };

__device__ __forceinline__ float sigmoidf_(float v) { return 1.f / (1.f + expf(-v)); }

// row r of the chunk is output pixel m0 + r; column col < cout:  v = wscale * rs[r] * acc + bias[col] (the weights' and
// the operand row's power-of-two scales undone), then
//   NONE: out = scale * v   RELU: relu(v)   CTX: tanh(v) for col < 128, relu(v) after (hidden | context)
//   ZR:   col < 128: out = z = sigmoid(v);  col >= 128: aux[row][col - 128] = sigmoid(v) * h[row][col - 128]
//   Q:    h[row][col] = (1 - z) h + z tanh(v)  with z = aux[row][col]  (in place)
//   FLOW: out[row][col] += v  (coords1 += delta)
struct EpiRaft {
  float* out; int ldo; int cout; int act; float scale; const float* bias; size_t m0; float wscale; const float* rs;
  float* part; int pmode;   // K chunks: 1 = part = acc, 2 = part += acc, 3 = acc += part, then the epilogue (0: one pass)
  float* aux; float* h; int ldh;
  struct State {};
  __device__ __forceinline__ void tile_begin(State&) const {}
  __device__ __forceinline__ void tile_end(State&, int, int, int) const {}
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    const size_t row = m0 + r;
    const float unscale = wscale * rs[r];   // powers of two: exact
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      const int col = col0 + i;
      if (i >= ncols || col >= cout) continue;
      float a = f[i];
      if (pmode) {
        float* pp = part + (size_t)r * cout + col;
        if (pmode == 1) { *pp = a; continue; }
        a = __fadd_rn(*pp, a);
        if (pmode == 2) { *pp = a; continue; }
      }
      const float v = a * unscale + __ldg(bias + col);
      switch (act) {
        case ACT_NONE: out[row * ldo + col] = scale * v; break;
        case ACT_RELU: out[row * ldo + col] = fmaxf(v, 0.f); break;
        case ACT_CTX: out[row * ldo + col] = col < 128 ? tanhf(v) : fmaxf(v, 0.f); break;
        case ACT_ZR:
          if (col < 128) out[row * ldo + col] = sigmoidf_(v);
          else aux[row * 128 + col - 128] = __fmul_rn(sigmoidf_(v), h[row * ldh + col - 128]);
          break;
        case ACT_Q: {
          const float z = aux[row * 128 + col], hv = h[row * ldh + col];
          h[row * ldh + col] = __fadd_rn(__fmul_rn(1.f - z, hv), __fmul_rn(z, tanhf(v)));
          break;
        }
        default: out[row * ldo + col] += v; break;
      }
    }
  }
};

// corr[g][r][col] = acc / 16 (exact) for pair g's row r, level 0 of its pyramid
struct EpiCorr {
  float* pyr; size_t pair_stride; int hw;
  struct State {};
  __device__ __forceinline__ void tile_begin(State&) const {}
  __device__ __forceinline__ void tile_end(State&, int, int, int) const {}
  __device__ __forceinline__ void operator()(State&, int g, int r, int col0, const float (&f)[32], int ncols) const {
    float* o = pyr + g * pair_stride + (size_t)r * hw + col0;
#pragma unroll
    for (int i = 0; i < 32; ++i)
      if (i < ncols) o[i] = f[i] * 0.0625f;
  }
};

// ---- small kernels ---------------------------------------------------------------------------------------------------
// frame t [3][H][W] in [0, 1] -> [Hp][Wp][3]: replicate pad (top / left first), then (x - 0.5) / 0.5 (the weights' transforms)
__global__ void raft_prep_kernel(const float* __restrict__ frame, int H, int W, int Hp, int Wp, int pt, int pl,
                                 float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= Hp * Wp) return;
  const int y = i / Wp, x = i - y * Wp;
  const int sy = min(max(y - pt, 0), H - 1), sx = min(max(x - pl, 0), W - 1);
#pragma unroll
  for (int c = 0; c < 3; ++c) out[(size_t)i * 3 + c] = (frame[((size_t)c * H + sy) * W + sx] - 0.5f) / 0.5f;
}

// InstanceNorm statistics of one image x [HW][C]: float64 partial sums over RAFT_NCH fixed pixel ranges, then
// (mean, 1 / sqrt(var + 1e-5)) of the biased variance
__global__ void raft_inorm_partial_kernel(const float* __restrict__ x, int HW, int C, double* __restrict__ part) {
  const int c = threadIdx.x, ch = blockIdx.x;
  if (c >= C) return;
  const int p0 = (int)((long long)HW * ch / RAFT_NCH), p1 = (int)((long long)HW * (ch + 1) / RAFT_NCH);
  double s = 0.0, ss = 0.0;
  for (int p = p0; p < p1; ++p) { const double v = x[(size_t)p * C + c]; s += v; ss += v * v; }
  part[((size_t)ch * C + c) * 2] = s;
  part[((size_t)ch * C + c) * 2 + 1] = ss;
}

__global__ void raft_inorm_final_kernel(const double* __restrict__ part, int HW, int C, float2* __restrict__ aff) {
  const int c = threadIdx.x;
  if (c >= C) return;
  double s = 0.0, ss = 0.0;
  for (int ch = 0; ch < RAFT_NCH; ++ch) { s += part[((size_t)ch * C + c) * 2]; ss += part[((size_t)ch * C + c) * 2 + 1]; }
  const double mean = s / HW, var = fmax(ss / HW - mean * mean, 0.0), rstd = 1.0 / sqrt(var + 1e-5);
  aff[c] = make_float2((float)mean, (float)rstd);
}

__global__ void raft_identity_kernel(float2* aff, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) aff[i] = make_float2(0.f, 1.f);
}

__global__ void raft_norm_relu_kernel(float* __restrict__ x, const float2* __restrict__ a, size_t n, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) { const float2 ac = a[i % C]; x[i] = fmaxf(__fmul_rn(__fsub_rn(x[i], ac.x), ac.y), 0.f); }
}

// ResidualBlock's relu(x + y): y = relu(a2(y2)), x = ad(xd) (the normalised 1 x 1 projection) or xd itself
__global__ void raft_residual_kernel(const float* __restrict__ y2, const float2* __restrict__ a2, const float* __restrict__ xd,
                                     const float2* __restrict__ ad, float* __restrict__ out, size_t n, int C) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int c = (int)(i % C);
  const float y = fmaxf(__fmul_rn(__fsub_rn(y2[i], a2[c].x), a2[c].y), 0.f);
  const float x = ad ? __fmul_rn(__fsub_rn(xd[i], ad[c].x), ad[c].y) : xd[i];
  out[i] = fmaxf(x + y, 0.f);
}

// hx[m][0:256] = ctx[i][p] (tanh(hidden) | relu(context)) of the pair's first frame; coords1 = coords0 = (x, y)
__global__ void raft_init_kernel(const float* __restrict__ ctx, const int* __restrict__ pairs, int hw, int w8,
                                 float* __restrict__ hx, float* __restrict__ coords) {
  const int m = blockIdx.x, b = m / hw, p = m - b * hw;
  const float* src = ctx + ((size_t)pairs[2 * b] * hw + p) * 256;
  for (int c = threadIdx.x; c < 256; c += blockDim.x) hx[(size_t)m * RAFT_HX + c] = src[c];
  if (threadIdx.x == 0) { coords[2 * m] = (float)(p % w8); coords[2 * m + 1] = (float)(p / w8); }
}

// GEMM groups of the correlation volume: pair g = A rows of frame i against B item j
__global__ void raft_corr_plan_kernel(const int* __restrict__ pairs, int n, int hw, int* batch, int* row0, int* m,
                                      int* tile_start) {
  if (threadIdx.x || blockIdx.x) return;
  const int tiles = (hw + TC_BM - 1) / TC_BM;
  for (int g = 0; g < n; ++g) { batch[g] = pairs[2 * g + 1]; row0[g] = pairs[2 * g] * hw; m[g] = hw; tile_start[g] = g * tiles; }
  tile_start[n] = n * tiles;
}

// exact-fp32 level 0 (fmaps outside the fp16 split's faithful range): 64 x 64 tiles, sequential fmaf over k
__global__ void __launch_bounds__(256) raft_corr_f32_kernel(const float* __restrict__ fmap, const int* __restrict__ pairs,
                                                            int hw, float* __restrict__ pyr, size_t pair_stride) {
  __shared__ float sa[16][65], sb[16][65];
  const int g = blockIdx.z, r0 = blockIdx.y * 64, c0 = blockIdx.x * 64;
  const float* A = fmap + (size_t)pairs[2 * g] * hw * 256;
  const float* B = fmap + (size_t)pairs[2 * g + 1] * hw * 256;
  const int tx = threadIdx.x & 15, ty = threadIdx.x >> 4;
  float acc[4][4] = {};
  for (int k0 = 0; k0 < 256; k0 += 16) {
    for (int i = threadIdx.x; i < 64 * 16; i += 256) {
      const int rr = i >> 4, kk = i & 15;
      sa[kk][rr] = r0 + rr < hw ? A[(size_t)(r0 + rr) * 256 + k0 + kk] : 0.f;
      sb[kk][rr] = c0 + rr < hw ? B[(size_t)(c0 + rr) * 256 + k0 + kk] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int kk = 0; kk < 16; ++kk)
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = __fmaf_rn(sa[kk][ty + 16 * i], sb[kk][tx + 16 * j], acc[i][j]);
    __syncthreads();
  }
  float* o = pyr + g * pair_stride;
#pragma unroll
  for (int i = 0; i < 4; ++i)
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const int r = r0 + ty + 16 * i, c = c0 + tx + 16 * j;
      if (r < hw && c < hw) o[(size_t)r * hw + c] = acc[i][j] * 0.0625f;
    }
}

// F.avg_pool2d(kernel 2, stride 2) over the last two axes: [P * hw][hs][ws] -> [P * hw][hs / 2][ws / 2]
__global__ void raft_pool_kernel(const float* __restrict__ src, float* __restrict__ dst, int P, int hw, int hs, int ws,
                                 size_t pair_stride) {
  const int hd = hs / 2, wd = ws / 2;
  const size_t n = (size_t)P * hw * hd * wd;
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int x = (int)(i % wd);
  size_t q = i / wd;
  const int y = (int)(q % hd);
  q /= hd;
  const int r = (int)(q % hw), g = (int)(q / hw);
  const float* s = src + g * pair_stride + (size_t)r * hs * ws + (size_t)(2 * y) * ws + 2 * x;
  float a = 0.f;
  a += s[0]; a += s[1]; a += s[ws]; a += s[ws + 1];
  dst[g * pair_stride + (size_t)r * hd * wd + (size_t)y * wd + x] = a / 4.f;
}

// Pyramid lookup of row m (pair g, pixel p): channel l * 81 + i * 9 + j = grid_sample(level l, align_corners, zeros) at
// (x, y) = (cx / 2^l + i - 4, cy / 2^l + j - 4) in torchvision's normalise / unnormalise arithmetic; written as the hi / lo
// operand of convcorr1, scaled per row like the im2col rows (the inverse scale to rs[m]: correlations of any size stay
// inside the fp16 split's range).  Also hx's flow columns = coords1 - coords0.
struct Pyr { int h[4], w[4]; size_t off[4]; size_t pair_stride; };
__global__ void __launch_bounds__(128) raft_lookup_kernel(const float* __restrict__ pyr, Pyr py, int hw, int w8,
                                                          const float* __restrict__ coords, __half* __restrict__ hi,
                                                          __half* __restrict__ lo, float* __restrict__ rs,
                                                          float* __restrict__ hx) {
  constexpr int PER = (RAFT_CORR_K + 127) / 128;
  const int m = blockIdx.x, g = m / hw, p = m - g * hw;
  const float cx = coords[2 * m], cy = coords[2 * m + 1];
  if (threadIdx.x == 0) {
    hx[(size_t)m * RAFT_HX + 382] = cx - (float)(p % w8);
    hx[(size_t)m * RAFT_HX + 383] = cy - (float)(p / w8);
  }
  float vals[PER];
  float mx = 0.f;
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int c = threadIdx.x + q * 128;
    float v = 0.f;
    if (c < 324) {
      const int l = c / 81, t = c - l * 81, i = t / 9, j = t - i * 9;
      float ccx = cx, ccy = cy;
      for (int k = 0; k < l; ++k) { ccx = ccx / 2.f; ccy = ccy / 2.f; }
      const int H = py.h[l], W = py.w[l];
      const float sx = ccx + (float)(i - 4), sy = ccy + (float)(j - 4);
      const float gx = 2.f * sx / (float)(W - 1) - 1.f, gy = 2.f * sy / (float)(H - 1) - 1.f;
      const float ix = ((gx + 1.f) / 2.f) * (float)(W - 1), iy = ((gy + 1.f) / 2.f) * (float)(H - 1);
      const float fx = floorf(ix), fy = floorf(iy);
      const int x0 = (int)fx, y0 = (int)fy;
      const float nw = (fx + 1.f - ix) * (fy + 1.f - iy), ne = (ix - fx) * (fy + 1.f - iy);
      const float sw = (fx + 1.f - ix) * (iy - fy), se = (ix - fx) * (iy - fy);
      const float* map = pyr + g * py.pair_stride + py.off[l] + (size_t)p * H * W;
      auto at = [&](int y, int x) { return (x >= 0 && x < W && y >= 0 && y < H) ? map[(size_t)y * W + x] : 0.f; };
      v = __fadd_rn(v, __fmul_rn(at(y0, x0), nw));           // ATen's order: nw, ne, sw, se
      v = __fadd_rn(v, __fmul_rn(at(y0, x0 + 1), ne));
      v = __fadd_rn(v, __fmul_rn(at(y0 + 1, x0), sw));
      v = __fadd_rn(v, __fmul_rn(at(y0 + 1, x0 + 1), se));
    }
    vals[q] = v;
    mx = fmaxf(mx, fabsf(v));
  }
  float inv;
  const float sc = raft_row_scale(mx, &inv);
  if (threadIdx.x == 0) rs[m] = inv;
#pragma unroll
  for (int q = 0; q < PER; ++q) {
    const int c = threadIdx.x + q * 128;
    if (c < RAFT_CORR_K) split16(vals[q] * sc, hi[(size_t)m * RAFT_CORR_K + c], lo[(size_t)m * RAFT_CORR_K + c]);
  }
}

// upsample_flow with the convex mask, cropped to the frame: out[g][c][Y][X] for padded pixel (Y + pt, X + pl) =
// sum_k softmax_k(mask[k * 64 + dy * 8 + dx]) * 8 flow_c(y + k / 3 - 1, x + k % 3 - 1)  (zero outside the grid)
__global__ void raft_upsample_kernel(const float* __restrict__ mask, const float* __restrict__ coords, int P, int h8, int w8,
                                     int H, int W, int pt, int pl, float* __restrict__ out) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)P * H * W) return;
  const int X = (int)(i % W);
  const size_t q = i / W;
  const int Y = (int)(q % H), g = (int)(q / H);
  const int Yp = Y + pt, Xp = X + pl, y = Yp >> 3, x = Xp >> 3, dy = Yp & 7, dx = Xp & 7;
  const float* mk = mask + ((size_t)g * h8 * w8 + (size_t)y * w8 + x) * 576 + dy * 8 + dx;
  float mx = -INFINITY;
  float e[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) { e[k] = mk[k * 64]; mx = fmaxf(mx, e[k]); }
  float s = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) { e[k] = expf(e[k] - mx); s += e[k]; }
  float f0 = 0.f, f1 = 0.f;
#pragma unroll
  for (int k = 0; k < 9; ++k) {
    const int yy = y + k / 3 - 1, xx = x + k % 3 - 1;
    float u0 = 0.f, u1 = 0.f;
    if (yy >= 0 && yy < h8 && xx >= 0 && xx < w8) {
      const size_t m = (size_t)g * h8 * w8 + (size_t)yy * w8 + xx;
      u0 = 8.f * (coords[2 * m] - (float)xx);
      u1 = 8.f * (coords[2 * m + 1] - (float)yy);
    }
    const float wk = e[k] / s;
    f0 += wk * u0;
    f1 += wk * u1;
  }
  out[(((size_t)g * 2) * H + Y) * W + X] = f0;
  out[(((size_t)g * 2 + 1) * H + Y) * W + X] = f1;
}

// ---- host helpers ----------------------------------------------------------------------------------------------------
struct RaftScratch { __half* hi; __half* lo; float* rs; float* part; int* plan; };

// The GEMM of one row chunk in K chunks of RAFT_KC: the tensor cores' fp32 accumulation does not round to nearest, and
// its error grows with the number of accumulation steps; partial sums of RAFT_KC are added in fp32 (round to nearest)
// in the epilogue, through part [rows][cout].
constexpr int RAFT_KC = 256;
static int raft_gemm(const __half* a_hi, const __half* a_lo, size_t rows, const void* w_hi, const void* w_lo, int Np, int Kp,
                     EpiRaft epi, float* part, const TcPlan& pl, cudaStream_t st) {
  const int nk = Kp <= 2 * RAFT_KC ? 1 : cdiv(Kp, RAFT_KC);
  for (int c = 0; c < nk; ++c) {
    const int k0 = nk == 1 ? 0 : c * RAFT_KC, kc = nk == 1 ? Kp : (Kp - k0 < RAFT_KC ? Kp - k0 : RAFT_KC);
    EpiRaft e = epi;
    e.part = part;
    e.pmode = nk == 1 ? 0 : c == 0 ? 1 : c == nk - 1 ? 3 : 2;
    if (int rc = tc_launch_bn<TcMode::F16X3>({a_hi + k0, a_lo + k0, rows, (uint64_t)Kp, (const __half*)w_hi + k0,
                                              (const __half*)w_lo + k0, 1, (uint64_t)Kp},
                                             pl.problem(1, Np, kc), cdiv((int)rows, TC_BM), e, st))
      return rc;
  }
  return DINOTRK_OK;
}

// one convolution: rows of nimg images at (Hout, Wout); epi.m0 is set per chunk
static int raft_conv(const dinotrk_raft_weights* w, int idx, ColSrc s0, ColSrc s1, int nimg, int Hin, int Win, EpiRaft epi,
                     const RaftScratch& sc, cudaStream_t st) {
  const RaftConv& c = kConv[idx];
  const int ph = c.kh / 2, pw = c.kw / 2;
  const int Hout = (Hin + 2 * ph - c.kh) / c.stride + 1, Wout = (Win + 2 * pw - c.kw) / c.stride + 1;
  const ColGeom geo{Hin, Win, Hout, Wout, c.kh, c.kw, c.stride, ph, pw, conv_kp(c)};
  const size_t M = (size_t)nimg * Hout * Wout;
  const TcPlan pl{sc.plan, sc.plan + 4, sc.plan + 8, sc.plan + 12};
  epi.cout = c.cout;
  epi.bias = w->bias[idx];
  epi.wscale = w->scale[idx];
  epi.rs = sc.rs;
  for (size_t m0 = 0; m0 < M; m0 += RAFT_ROWS) {
    const size_t rows = M - m0 < RAFT_ROWS ? M - m0 : RAFT_ROWS;
    raft_im2col_kernel<<<(unsigned)rows, 128, 0, st>>>(s0, s1, geo, sc.hi, sc.lo, sc.rs, m0);
    DTK_LAUNCHED();
    if (int rc = launch_tc_plan(pl, 1, (int)rows, 0, 0, 0, TC_BM, st)) return rc;
    epi.m0 = m0;
    if (int rc = raft_gemm(sc.hi, sc.lo, rows, w->w_hi[idx], w->w_lo[idx], conv_np(c.cout), geo.Kp, epi, sc.part, pl, st))
      return rc;
  }
  return DINOTRK_OK;
}

static EpiRaft epi_out(float* out, int ldo, int act, float scale = 1.f) {
  EpiRaft e{};
  e.out = out; e.ldo = ldo; e.act = act; e.scale = scale;
  return e;
}

static int raft_inorm(const float* x, int HW, int C, float2* aff, double* part, cudaStream_t st) {
  raft_inorm_partial_kernel<<<RAFT_NCH, 128, 0, st>>>(x, HW, C, part);
  DTK_LAUNCHED();
  raft_inorm_final_kernel<<<1, 128, 0, st>>>(part, HW, C, aff);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

static bool raft_shape_ok(int H, int W) {   // the padded frame's 1/8 grid must survive three 2 x 2 pools (>= 2 x 2)
  return H > 0 && W > 0 && (H + 7) / 8 >= 16 && (W + 7) / 8 >= 16 && (size_t)H * W < (1u << 28);
}

struct RaftEncWs {
  float *xin, *b[5]; float2 *aff, *ident; double* part; RaftScratch sc;
  RaftEncWs(Arena& ar, int Hp, int Wp) {
    xin = ar.take<float>((size_t)Hp * Wp * 3);
    for (auto& p : b) p = ar.take<float>((size_t)(Hp / 2) * (Wp / 2) * 64);
    aff = ar.take<float2>(3 * 256);
    ident = ar.take<float2>(256);
    part = ar.take<double>((size_t)RAFT_NCH * 128 * 2);
    const size_t rows = (size_t)(Hp / 2) * (Wp / 2) < RAFT_ROWS ? (size_t)(Hp / 2) * (Wp / 2) : RAFT_ROWS;
    sc.hi = ar.take<__half>(rows * RAFT_KMAX_ENC);
    sc.lo = ar.take<__half>(rows * RAFT_KMAX_ENC);
    sc.rs = ar.take<float>(rows);
    sc.part = ar.take<float>(rows * 576);
    sc.plan = ar.take<int>(16);
  }
};

// one encoder (first conv index e0: 0 = feature encoder with InstanceNorm, 16 = context encoder, BatchNorm folded) of
// one frame already in ws.xin; the final 1 x 1 conv writes out [h8 * w8][256] with `act`
static int raft_encoder(const dinotrk_raft_weights* w, int e0, bool inorm, int Hp, int Wp, float* out, int act, RaftEncWs& ws,
                        cudaStream_t st) {
  const ColSrc none{nullptr, 0, 0, nullptr};
  float2* a1 = ws.aff; float2* a2 = ws.aff + 256; float2* ad = ws.aff + 512;
  // normalisation of a raw conv output x [HW][C] into the table `a` (identity for the folded BatchNorm)
  auto norm = [&](const float* x, int HW, int C, float2*& a, float2* slot) -> int {
    if (!inorm) { a = ws.ident; return DINOTRK_OK; }
    a = slot;
    return raft_inorm(x, HW, C, slot, ws.part, st);
  };
  int H = Hp / 2, W = Wp / 2, C = 64;
  float2* a = nullptr;
  if (int rc = raft_conv(w, e0, {ws.xin, 3, 3, nullptr}, none, 1, Hp, Wp, epi_out(ws.b[0], 64, ACT_NONE), ws.sc, st)) return rc;
  if (int rc = norm(ws.b[0], H * W, 64, a, a1)) return rc;
  {   // the stem's output is also the first block's identity branch: activate it in place
    const size_t nn = (size_t)H * W * 64;
    raft_norm_relu_kernel<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>(ws.b[0], a, nn, 64);
    DTK_LAUNCHED();
  }
  const float* x = ws.b[0];
  int idx = e0 + 1;
  const int widths[3] = {64, 96, 128}, strides[3] = {1, 2, 2};
  int cur = 0;   // buffer holding x (activated)
  for (int L = 0; L < 3; ++L)
    for (int blk = 0; blk < 2; ++blk) {
      const int s = blk ? 1 : strides[L], Cout = widths[L];
      const int Ho = (H - 1) / s + 1, Wo = (W - 1) / s + 1;
      int fr[4], n = 0;
      for (int k = 0; k < 5 && n < 4; ++k) if (k != cur) fr[n++] = k;
      float *t1 = ws.b[fr[0]], *t2 = ws.b[fr[1]], *d = ws.b[fr[2]], *o = ws.b[fr[3]];
      const ColSrc xin{x, C, C, nullptr};
      float2 *n1, *n2, *nd = nullptr;
      if (int rc = raft_conv(w, idx, xin, none, 1, H, W, epi_out(t1, Cout, ACT_NONE), ws.sc, st)) return rc;
      if (int rc = norm(t1, Ho * Wo, Cout, n1, a1)) return rc;
      if (int rc = raft_conv(w, idx + 1, {t1, Cout, Cout, n1}, none, 1, Ho, Wo, epi_out(t2, Cout, ACT_NONE), ws.sc, st)) return rc;
      if (int rc = norm(t2, Ho * Wo, Cout, n2, a2)) return rc;
      const float* xr = x;
      if (s != 1) {
        if (int rc = raft_conv(w, idx + 2, xin, none, 1, H, W, epi_out(d, Cout, ACT_NONE), ws.sc, st)) return rc;
        if (int rc = norm(d, Ho * Wo, Cout, nd, ad)) return rc;
        xr = d;
      }
      const size_t nn = (size_t)Ho * Wo * Cout;
      raft_residual_kernel<<<(unsigned)((nn + 255) / 256), 256, 0, st>>>(t2, n2, xr, nd, o, nn, Cout);
      DTK_LAUNCHED();
      idx += s != 1 ? 3 : 2;
      x = o; cur = fr[3];
      H = Ho; W = Wo; C = Cout;
    }
  return raft_conv(w, e0 + 15, {x, C, C, nullptr}, none, 1, H, W, epi_out(out, 256, act), ws.sc, st);
}

struct RaftFlowWs {
  float *pyr, *coords, *hx, *zb, *rh, *cc1, *cf, *f1, *mask, *crs; __half *chi, *clo; int* pairs; int* cplan; RaftScratch sc;
  Pyr py;
  RaftFlowWs(Arena& ar, int h8, int w8, int P) {
    const int hw = h8 * w8;
    size_t off = 0;
    for (int l = 0; l < 4; ++l) {
      py.h[l] = l ? py.h[l - 1] / 2 : h8;
      py.w[l] = l ? py.w[l - 1] / 2 : w8;
      py.off[l] = off;
      off += (size_t)hw * py.h[l] * py.w[l];
    }
    py.pair_stride = off;
    const size_t M = (size_t)P * hw;
    pyr = ar.take<float>(off * P);
    coords = ar.take<float>(M * 2);
    hx = ar.take<float>(M * RAFT_HX);
    zb = ar.take<float>(M * 128);
    rh = ar.take<float>(M * 128);
    cc1 = ar.take<float>(M * 256);
    cf = ar.take<float>(M * 256);
    f1 = ar.take<float>(M * 128);
    mask = ar.take<float>(M * 576);
    chi = ar.take<__half>(M * RAFT_CORR_K);
    clo = ar.take<__half>(M * RAFT_CORR_K);
    crs = ar.take<float>(M);
    pairs = ar.take<int>((size_t)2 * P);
    cplan = ar.take<int>((size_t)4 * P + 4);
    const size_t rows = M < RAFT_ROWS ? M : RAFT_ROWS;
    sc.hi = ar.take<__half>(rows * RAFT_KMAX_UPD);
    sc.lo = ar.take<__half>(rows * RAFT_KMAX_UPD);
    sc.rs = ar.take<float>(rows);
    sc.part = ar.take<float>(rows * 576);
    sc.plan = ar.take<int>(16);
  }
};

static int raft_weights_ok(const dinotrk_raft_weights* w, int first, int last) {
  for (int i = first; i < last; ++i)
    if (!w->w_hi[i] || !w->w_lo[i] || !w->bias[i] || !(w->scale[i] > 0.f)) return 0;
  return 1;
}

}  // namespace dtk

using namespace dtk;

extern "C" {

size_t dinotrk_raft_encode_workspace_bytes(int H, int W) {
  if (!raft_shape_ok(H, W)) return 0;
  return layout_end<RaftEncWs>((H + 7) / 8 * 8, (W + 7) / 8 * 8) + 256;
}

int dinotrk_raft_encode(const float* frames, int T, int T_ctx, int H, int W, const dinotrk_raft_weights* w, float* fmap,
                        float* ctx, void* workspace, size_t workspace_bytes, void* stream) {
  NvtxRange nvtx_range("dinotrk.raft_encode");
  DTK_CHECK_ARG(frames && w && fmap && T > 0 && T_ctx >= 0 && T_ctx <= T && (ctx || T_ctx == 0), "raft_encode: bad arguments");
  DTK_CHECK_ARG(raft_shape_ok(H, W), "raft_encode: frames must be at least 128 x 128 (after padding to a multiple of 8)");
  DTK_CHECK_ARG(raft_weights_ok(w, 0, 32), "raft_encode: missing encoder weights");
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_raft_encode_workspace_bytes(H, W), "raft_encode: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int Hp = (H + 7) / 8 * 8, Wp = (W + 7) / 8 * 8, pt = (Hp - H) / 2, pl = (Wp - W) / 2;
  const size_t hw = (size_t)(Hp / 8) * (Wp / 8);
  Arena ar(workspace);
  RaftEncWs ws(ar, Hp, Wp);
  raft_identity_kernel<<<1, 256, 0, st>>>(ws.ident, 256);
  DTK_LAUNCHED();
  for (int t = 0; t < T; ++t) {
    raft_prep_kernel<<<cdiv(Hp * Wp, 256), 256, 0, st>>>(frames + (size_t)t * 3 * H * W, H, W, Hp, Wp, pt, pl, ws.xin);
    DTK_LAUNCHED();
    if (int rc = raft_encoder(w, 0, true, Hp, Wp, fmap + t * hw * 256, ACT_NONE, ws, st)) return rc;
    if (t < T_ctx)
      if (int rc = raft_encoder(w, 16, false, Hp, Wp, ctx + t * hw * 256, ACT_CTX, ws, st)) return rc;
  }
  return DINOTRK_OK;
}

size_t dinotrk_raft_flow_workspace_bytes(int H, int W, int n_pairs) {
  if (!raft_shape_ok(H, W) || n_pairs <= 0) return 0;
  return layout_end<RaftFlowWs>((H + 7) / 8, (W + 7) / 8, n_pairs) + 256;
}

int dinotrk_raft_flow(const float* fmap, const void* fmap_hi, const void* fmap_lo, const float* ctx, int T, int T_ctx, int H,
                      int W, const int* pairs, int n_pairs, int num_flow_updates, const dinotrk_raft_weights* w, float* flows,
                      void* workspace, size_t workspace_bytes, void* stream) {
  NvtxRange nvtx_range("dinotrk.raft_flow");
  DTK_CHECK_ARG(fmap && ctx && pairs && w && flows && T > 0 && T_ctx > 0 && T_ctx <= T && n_pairs > 0 && num_flow_updates > 0,
                "raft_flow: bad arguments");
  DTK_CHECK_ARG(!fmap_hi == !fmap_lo, "raft_flow: give both halves of the fmap split or neither");
  DTK_CHECK_ARG(raft_shape_ok(H, W), "raft_flow: frames must be at least 128 x 128 (after padding to a multiple of 8)");
  DTK_CHECK_ARG(raft_weights_ok(w, 32, DINOTRK_RAFT_NCONV), "raft_flow: missing update-block weights");
  for (int g = 0; g < 2 * n_pairs; ++g) DTK_CHECK_ARG(pairs[g] >= 0 && pairs[g] < T, "raft_flow: frame index out of range");
  for (int g = 0; g < n_pairs; ++g)
    DTK_CHECK_ARG(pairs[2 * g] < T_ctx, "raft_flow: a flow starts from a frame encoded without its context (i >= T_ctx)");
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_raft_flow_workspace_bytes(H, W, n_pairs), "raft_flow: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int Hp = (H + 7) / 8 * 8, Wp = (W + 7) / 8 * 8, h8 = Hp / 8, w8 = Wp / 8, hw = h8 * w8;
  const int pt = (Hp - H) / 2, pl = (Wp - W) / 2;
  const int P = n_pairs;
  const size_t M = (size_t)P * hw;
  DTK_CHECK_ARG(M < (1u << 31) / RAFT_HX, "raft_flow: too many pairs for one call");
  Arena ar(workspace);
  RaftFlowWs ws(ar, h8, w8, P);
  DTK_CUDA(cudaMemcpyAsync(ws.pairs, pairs, sizeof(int) * 2 * P, cudaMemcpyHostToDevice, st));

  // correlation pyramid
  if (fmap_hi) {
    const TcPlan pl_{ws.cplan, ws.cplan + P, ws.cplan + 2 * P, ws.cplan + 3 * P};
    raft_corr_plan_kernel<<<1, 32, 0, st>>>(ws.pairs, P, hw, pl_.batch, pl_.row0, pl_.m, pl_.tile_start);
    DTK_LAUNCHED();
    EpiCorr epi{ws.pyr, ws.py.pair_stride, hw};
    if (int rc = tc_launch_bn<TcMode::F16X3>({fmap_hi, fmap_lo, (uint64_t)T * hw, 0, fmap_hi, fmap_lo, (uint64_t)T, 0},
                                             pl_.problem(P, hw, 256), P * cdiv(hw, TC_BM), epi, st))
      return rc;
  } else {
    raft_corr_f32_kernel<<<dim3(cdiv(hw, 64), cdiv(hw, 64), P), 256, 0, st>>>(fmap, ws.pairs, hw, ws.pyr, ws.py.pair_stride);
    DTK_LAUNCHED();
  }
  for (int l = 0; l < 3; ++l) {
    const size_t n = M * ws.py.h[l + 1] * ws.py.w[l + 1];
    raft_pool_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(ws.pyr + ws.py.off[l], ws.pyr + ws.py.off[l + 1], P, hw,
                                                                  ws.py.h[l], ws.py.w[l], ws.py.pair_stride);
    DTK_LAUNCHED();
  }

  raft_init_kernel<<<(unsigned)M, 128, 0, st>>>(ctx, ws.pairs, hw, w8, ws.hx, ws.coords);
  DTK_LAUNCHED();
  const ColSrc none{nullptr, 0, 0, nullptr};
  const int n = P;   // images of the update block's convolutions: one per pair, h8 x w8 each
  for (int it = 0; it < num_flow_updates; ++it) {
    raft_lookup_kernel<<<(unsigned)M, 128, 0, st>>>(ws.pyr, ws.py, hw, w8, ws.coords, ws.chi, ws.clo, ws.crs, ws.hx);
    DTK_LAUNCHED();
    {   // convcorr1: the lookup wrote its operand
      const TcPlan pl_{ws.sc.plan, ws.sc.plan + 4, ws.sc.plan + 8, ws.sc.plan + 12};
      for (size_t m0 = 0; m0 < M; m0 += RAFT_ROWS) {
        const size_t rows = M - m0 < RAFT_ROWS ? M - m0 : RAFT_ROWS;
        if (int rc = launch_tc_plan(pl_, 1, (int)rows, 0, 0, 0, TC_BM, st)) return rc;
        EpiRaft e = epi_out(ws.cc1, 256, ACT_RELU);
        e.cout = 256; e.bias = w->bias[DINOTRK_RAFT_CONVCORR1]; e.m0 = m0; e.wscale = w->scale[DINOTRK_RAFT_CONVCORR1];
        e.rs = ws.crs + m0;
        if (int rc = raft_gemm(ws.chi + m0 * RAFT_CORR_K, ws.clo + m0 * RAFT_CORR_K, rows, w->w_hi[DINOTRK_RAFT_CONVCORR1],
                               w->w_lo[DINOTRK_RAFT_CONVCORR1], 256, RAFT_CORR_K, e, ws.sc.part, pl_, st))
          return rc;
      }
    }
    int rc;
    if ((rc = raft_conv(w, DINOTRK_RAFT_CONVCORR2, {ws.cc1, 256, 256, nullptr}, none, n, h8, w8, epi_out(ws.cf, 256, ACT_RELU), ws.sc, st))) return rc;
    if ((rc = raft_conv(w, DINOTRK_RAFT_CONVFLOW1, {ws.hx + 382, 2, RAFT_HX, nullptr}, none, n, h8, w8, epi_out(ws.f1, 128, ACT_RELU), ws.sc, st))) return rc;
    if ((rc = raft_conv(w, DINOTRK_RAFT_CONVFLOW2, {ws.f1, 128, 128, nullptr}, none, n, h8, w8, epi_out(ws.cf + 192, 256, ACT_RELU), ws.sc, st))) return rc;
    if ((rc = raft_conv(w, DINOTRK_RAFT_MOTION_CONV, {ws.cf, 256, 256, nullptr}, none, n, h8, w8, epi_out(ws.hx + 256, RAFT_HX, ACT_RELU), ws.sc, st))) return rc;
    for (int gru = 0; gru < 2; ++gru) {
      const int zr = gru ? DINOTRK_RAFT_GRU2_ZR : DINOTRK_RAFT_GRU1_ZR;
      EpiRaft e = epi_out(ws.zb, 128, ACT_ZR);
      e.aux = ws.rh; e.h = ws.hx; e.ldh = RAFT_HX;
      if ((rc = raft_conv(w, zr, {ws.hx, RAFT_HX, RAFT_HX, nullptr}, none, n, h8, w8, e, ws.sc, st))) return rc;
      EpiRaft q = epi_out(nullptr, 0, ACT_Q);
      q.aux = ws.zb; q.h = ws.hx; q.ldh = RAFT_HX;
      if ((rc = raft_conv(w, zr + 1, {ws.rh, 128, 128, nullptr}, {ws.hx + 128, 256, RAFT_HX, nullptr}, n, h8, w8, q, ws.sc, st))) return rc;
    }
    if ((rc = raft_conv(w, DINOTRK_RAFT_FLOW_HEAD1, {ws.hx, 128, RAFT_HX, nullptr}, none, n, h8, w8, epi_out(ws.cc1, 256, ACT_RELU), ws.sc, st))) return rc;
    if ((rc = raft_conv(w, DINOTRK_RAFT_FLOW_HEAD2, {ws.cc1, 256, 256, nullptr}, none, n, h8, w8, epi_out(ws.coords, 2, ACT_FLOW), ws.sc, st))) return rc;
  }
  int rc;
  if ((rc = raft_conv(w, DINOTRK_RAFT_MASK1, {ws.hx, 128, RAFT_HX, nullptr}, none, n, h8, w8, epi_out(ws.cc1, 256, ACT_RELU), ws.sc, st))) return rc;
  if ((rc = raft_conv(w, DINOTRK_RAFT_MASK2, {ws.cc1, 256, 256, nullptr}, none, n, h8, w8, epi_out(ws.mask, 576, ACT_NONE, 0.25f), ws.sc, st))) return rc;
  const size_t nout = (size_t)P * H * W;
  raft_upsample_kernel<<<(unsigned)((nout + 255) / 256), 256, 0, st>>>(ws.mask, ws.coords, P, h8, w8, H, W, pt, pl, flows);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // extern "C"

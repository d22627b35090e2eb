// DINOv2 ViT feature extractor (SURVEY.md 8a row a1): ImageNet normalisation, 14x14 / stride-7 patch embedding,
// cls + interpolated position embedding, pre-LN blocks (LayerNorm eps 1e-6, MHA scale 1/8, LayerScale -- none in DINO v1's
// 8 x 8-patch ViT-S/8 and ViT-B/8 --, MLP 4x with exact GELU, or ViT-g/14's SwiGLU MLP), tap = output of block `layer` before the final norm -- or that block's query /
// key / value facet, its qkv Linear output -- cls dropped, written straight into the
// token-major feature video [T][P][C]   (models/extractor.py:41-85,137-150,224-266; utils.py:32-72; the block arithmetic is
// facebookresearch/dinov2's -- parity unpinned, see DESIGN.md).
//
// Default path (gemm_f16 = 1, attn_materialized = 0): fp16 operands / fp32 accumulation everywhere.  The linear layers
// (patch embedding, qkv, proj, fc1, fc2) run on the wgmma GEMMs of tcgemm.cuh (two-CTA clusters when gemm_pair = 1)
// with bias / position embedding / GELU / LayerScale + residual / head scatter as coalesced epilogues on the accumulator;
// the residual stream stays fp32.  Attention is the fused kernel of flash.cuh (scores never leave the SM).
// Validation path (attn_materialized = 1): TF32 GEMMs, attention scores materialised per (frame, row chunk) in a workspace
// (tensor-core GEMM -> row softmax -> tensor-core GEMM).
//
// DINOv3 and DINOv2 with registers (dinotrk_vit_weights' appended fields): R register rows after cls, so every frame has
// pre = 1 + R prefix rows ahead of its patches (N1 = P + pre); DINOv3 has no position table but a rotary position
// embedding on q and k of the patch rows, applied in the qkv epilogue (EpiQKV16Rope / EpiQKVRope), and LayerNorm eps 1e-5.
// The new layouts run on epilogue types of their own, so the one-cls-row DINOv2 / DINO v1 launches keep their kernels.
#include "common.cuh"
#include "corr.cuh"
#include "tcgemm.cuh"
#include "flash.cuh"

namespace dtk {

constexpr int HD = 64;  // head dim of every DINOv2 ViT

// ---------------------------------------------------------------------------------------------- small kernels
// patches of ImageNet-normalised frames: out[(b*P + p)][c*196 + ky*14 + kx], row length Kp (zero padded)
template <typename T> __device__ __forceinline__ T cvt_out(float v);
template <> __device__ __forceinline__ float cvt_out<float>(float v) { return v; }
template <> __device__ __forceinline__ __half cvt_out<__half>(float v) { return __float2half_rn(v); }

template <typename OutT>
__global__ void vit_im2col_kernel(const float* __restrict__ frames, OutT* __restrict__ out, int B, int H, int W, int h,
                                  int w, int patch, int stride, int Kp) {
  const size_t row = blockIdx.x;  // b*P + p
  const int P = h * w;
  const int b = (int)(row / P), p = (int)(row - (size_t)b * P);
  const int py = (p / w) * stride, px = (p % w) * stride;
  const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
  const int K = 3 * patch * patch;
  for (int k = threadIdx.x; k < Kp; k += blockDim.x) {
    float v = 0.f;
    if (k < K) {
      int c = k / (patch * patch), r = k - c * patch * patch;
      int ky = r / patch, kx = r - ky * patch;
      float x = frames[(((size_t)b * 3 + c) * H + py + ky) * W + px + kx];
      v = __fdiv_rn(__fsub_rn(x, mean[c]), stdv[c]);  // torchvision Normalize: (x - mean) / std
    }
    out[row * Kp + k] = cvt_out<OutT>(v);
  }
}

// the pre = 1 + R prefix rows of frame b: x[b][0] = cls_pos, x[b][1 + i] = registers[i] (no position: DINOv2 adds pos[0]
// to cls only, DINOv3 has none)
__global__ void vit_cls_kernel(float* __restrict__ x, const float* __restrict__ cls_pos, const float* __restrict__ registers,
                               int pre, int N1, int D) {
  const int b = blockIdx.x;
  for (int i = threadIdx.x; i < pre * D; i += blockDim.x) x[(size_t)b * N1 * D + i] = i < D ? cls_pos[i] : registers[i - D];
}

// warp per row, D <= 2048
template <typename OutT>
__global__ void vit_layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gw, const float* __restrict__ gb,
                                     OutT* __restrict__ y, size_t rows, int D, float eps) {
  const size_t row = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (row >= rows) return;
  const int lane = threadIdx.x & 31;
  const float4* xr = reinterpret_cast<const float4*>(x + row * D);
  float4 v[16];
  const int n4 = D >> 2;
  float s = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    int idx = lane + 32 * i;
    if (idx < n4) { v[i] = xr[idx]; s += (v[i].x + v[i].y) + (v[i].z + v[i].w); }
  }
  const float mu = warp_sum(s) / (float)D;
  float q = 0.f;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    int idx = lane + 32 * i;
    if (idx < n4) {
      float a = v[i].x - mu, b = v[i].y - mu, c = v[i].z - mu, d = v[i].w - mu;
      q += (a * a + b * b) + (c * c + d * d);
    }
  }
  const float rstd = rsqrtf(warp_sum(q) / (float)D + eps);
  OutT* yr = y + row * D;
#pragma unroll
  for (int i = 0; i < 16; ++i) {
    int idx = lane + 32 * i;
    if (idx < n4) {
      float4 w4 = __ldg(reinterpret_cast<const float4*>(gw) + idx), b4 = __ldg(reinterpret_cast<const float4*>(gb) + idx);
      float4 o;
      o.x = (v[i].x - mu) * rstd * w4.x + b4.x; o.y = (v[i].y - mu) * rstd * w4.y + b4.y;
      o.z = (v[i].z - mu) * rstd * w4.z + b4.z; o.w = (v[i].w - mu) * rstd * w4.w + b4.w;
      if constexpr (sizeof(OutT) == 4) {
        reinterpret_cast<float4*>(yr)[idx] = o;
      } else {
        __half2 a = __floats2half2_rn(o.x, o.y), b = __floats2half2_rn(o.z, o.w);
        reinterpret_cast<uint2*>(yr)[idx] = make_uint2(*reinterpret_cast<uint32_t*>(&a), *reinterpret_cast<uint32_t*>(&b));
      }
    }
  }
}

// in-place row softmax over n columns (row stride ld); block per row
__global__ void vit_softmax_kernel(float* __restrict__ s, int n, int ld, size_t group_stride) {
  extern __shared__ float row[];
  __shared__ float red[32];
  float* p = s + (size_t)blockIdx.y * group_stride + (size_t)blockIdx.x * ld;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = blockDim.x >> 5;
  float m = -INFINITY;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { float v = p[i]; row[i] = v; m = fmaxf(m, v); }
  m = warp_max(m);
  if (lane == 0) red[warp] = m;
  __syncthreads();
  m = red[0];
  for (int k = 1; k < nw; ++k) m = fmaxf(m, red[k]);
  __syncthreads();
  float sum = 0.f;
  for (int i = threadIdx.x; i < n; i += blockDim.x) { float e = expf(row[i] - m); row[i] = e; sum += e; }
  sum = warp_sum(sum);
  if (lane == 0) red[warp] = sum;
  __syncthreads();
  sum = 0.f;
  for (int k = 0; k < nw; ++k) sum += red[k];
  const float inv = 1.f / sum;
  for (int i = threadIdx.x; i < n; i += blockDim.x) p[i] = row[i] * inv;
}

// x[b][pre + p][:] -> tpc[b][p][:]
__global__ void vit_tap_kernel(const float* __restrict__ x, float* __restrict__ tpc, int B, int P, int pre, int D) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // float4 index
  const int n4 = D >> 2;
  size_t total = (size_t)B * P * n4;
  if (i >= total) return;
  size_t row = i / n4;
  int c = (int)(i - row * n4);
  size_t b = row / P, p = row - b * P;
  reinterpret_cast<float4*>(tpc)[i] = reinterpret_cast<const float4*>(x)[((b * (P + pre) + pre + p)) * n4 + c];
}

// ---------------------------------------------------------------------------------------------- epilogues
struct EpiBase {
  struct State {};
  __device__ __forceinline__ void tile_begin(State&) const {}
  __device__ __forceinline__ void tile_end(State&, int, int, int) const {}
  __device__ __forceinline__ bool direct(int) const { return false; }
};
// r / d for 0 <= r < 2^24 without the ~40-instruction integer division (the epilogues do it per 4 output values)
__device__ __forceinline__ int fast_div(int r, int d) {
  int q = __float2int_rd(__int2float_rn(r) * __frcp_rn(__int2float_rn(d)));
  q += ((q + 1) * d <= r) ? 1 : 0;
  q -= (q * d > r) ? 1 : 0;
  return q;
}
__device__ __forceinline__ uint2 pack_half4(float a, float b, float c, float d) {
  __half2 x = __floats2half2_rn(a, b), y = __floats2half2_rn(c, d);
  return make_uint2(*reinterpret_cast<uint32_t*>(&x), *reinterpret_cast<uint32_t*>(&y));
}

// tokens: x[b][1 + p][col] = acc + bias[col] + pos[p][col]   (row r = b*P + p)
struct EpiPatch : EpiBase {
  static constexpr bool kCoalesced = true;
  float* x; const float* bias; const float* pos; int P, D;
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v) const {
    const int b = fast_div(r, P), p = r - b * P;
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col)), pp = __ldg(reinterpret_cast<const float4*>(pos + (size_t)p * D + col));
    *reinterpret_cast<float4*>(x + ((size_t)b * (P + 1) + 1 + p) * D + col) =
        make_float4(v.x + bb.x + pp.x, v.y + bb.y + pp.y, v.z + bb.z + pp.z, v.w + bb.w + pp.w);
  }
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    const int b = r / P, p = r - b * P;
    float* o = x + ((size_t)b * (P + 1) + 1 + p) * D + col0;
    const float* ps = pos + (size_t)p * D + col0;
#pragma unroll
    for (int i = 0; i < 32; i += 4)
      if (i < ncols) {   // ncols is a multiple of 4 (D % 64 == 0)
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col0 + i)), pp = __ldg(reinterpret_cast<const float4*>(ps + i));
        *reinterpret_cast<float4*>(o + i) = make_float4(f[i] + bb.x + pp.x, f[i + 1] + bb.y + pp.y, f[i + 2] + bb.z + pp.z, f[i + 3] + bb.w + pp.w);
      }
  }
};

// tokens after pre = 1 + R prefix rows: x[b][pre + p][col] = acc + bias[col] (+ pos[p][col] unless pos is null: DINOv3)
struct EpiPatchPrefix : EpiPatch {
  int pre;
  __device__ __forceinline__ float4 pos4(int p, int col) const {
    return pos ? __ldg(reinterpret_cast<const float4*>(pos + (size_t)p * D + col)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v) const {
    const int b = fast_div(r, P), p = r - b * P;
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col)), pp = pos4(p, col);
    *reinterpret_cast<float4*>(x + ((size_t)b * (P + pre) + pre + p) * D + col) =
        make_float4(v.x + bb.x + pp.x, v.y + bb.y + pp.y, v.z + bb.z + pp.z, v.w + bb.w + pp.w);
  }
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    const int b = r / P, p = r - b * P;
    float* o = x + ((size_t)b * (P + pre) + pre + p) * D + col0;
#pragma unroll
    for (int i = 0; i < 32; i += 4)
      if (i < ncols) {
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col0 + i)), pp = pos4(p, col0 + i);
        *reinterpret_cast<float4*>(o + i) = make_float4(f[i] + bb.x + pp.x, f[i + 1] + bb.y + pp.y, f[i + 2] + bb.z + pp.z, f[i + 3] + bb.w + pp.w);
      }
  }
};

// DINOv3's rotary position embedding of one (j, j + 32) pair of a head, which the host's row permutation of the q / k
// weights (and q bias) puts in adjacent columns (2j, 2j + 1); (c, s) = (cos, sin) of the pair's angle for this token.
// q . k is unchanged by the same permutation of both, so attention needs nothing else.
__device__ __forceinline__ void rope_pair(float& a, float& b, float2 cs) {
  const float a0 = a;
  a = __fmaf_rn(a0, cs.x, -__fmul_rn(b, cs.y));
  b = __fmaf_rn(b, cs.x, __fmul_rn(a0, cs.y));
}

// qkv: scatter to q [b][hd][n][64] (scaled 1/8), k [b][hd][n][64], vT [b][hd][64][n]
struct EpiQKV : EpiBase {
  float* q; float* k; float* vT; const float* bias; int N1, D, heads, N1p;
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    const int b = r / N1, n = r - b * N1;
    const int which = col0 / D, c = col0 - which * D, hd = c / HD, e0 = c - hd * HD;
    const size_t bh = (size_t)b * heads + hd;
    if (which < 2) {
      float* o = (which == 0 ? q : k) + (bh * N1 + n) * HD + e0;
      const float sc = which == 0 ? 0.125f : 1.f;
#pragma unroll
      for (int i = 0; i < 32; ++i) if (i < ncols) o[i] = (f[i] + __ldg(bias + col0 + i)) * sc;
    } else {
      float* o = vT + (bh * HD + e0) * N1p + n;
#pragma unroll
      for (int i = 0; i < 32; ++i) if (i < ncols) o[(size_t)i * N1p] = f[i] + __ldg(bias + col0 + i);
    }
  }
};

// qkv for the fused attention: fp16 q [b][hd][n][64] (scaled 1/8), k [b][hd][n][64], vT [b][hd][64][n] (pitch N1p)
struct EpiQKV16 : EpiBase {
  static constexpr bool kCoalesced = true;
  __half* q; __half* k; __half* vT; const float* bias; int N1, D, heads, N1p; float qscale;
  int direct_from = 1 << 30;   // columns >= direct_from take the thread-per-row call (host: 2 * D, or 0 = every column)
  // v goes out transposed ([d][n]): thread-per-row already writes consecutive n per lane -> keep the direct call there
  __device__ __forceinline__ bool direct(int col0) const { return col0 >= direct_from; }
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v) const {
    const int b = fast_div(r, N1), n = r - b * N1;
    const int which = (col >= D) + (col >= 2 * D), c = col - which * D, hd = c / HD, e0 = c - hd * HD;
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col));
    const float sc = which == 0 ? qscale : 1.f;
    __half* o = (which == 0 ? q : k) + (((size_t)b * heads + hd) * N1 + n) * HD + e0;
    *reinterpret_cast<uint2*>(o) = pack_half4((v.x + bb.x) * sc, (v.y + bb.y) * sc, (v.z + bb.z) * sc, (v.w + bb.w) * sc);
  }
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    const int b = r / N1, n = r - b * N1;
    const int which = col0 / D, c = col0 - which * D, hd = c / HD, e0 = c - hd * HD;
    const size_t bh = (size_t)b * heads + hd;
    if (which < 2) {
      __half* o = (which == 0 ? q : k) + (bh * N1 + n) * HD + e0;
      const float sc = which == 0 ? qscale : 1.f;
#pragma unroll
      for (int i = 0; i < 32; i += 8)
        if (i < ncols) {
          const float4 b0 = __ldg(reinterpret_cast<const float4*>(bias + col0 + i)), b1 = __ldg(reinterpret_cast<const float4*>(bias + col0 + i + 4));
          __half2 h0 = __floats2half2_rn((f[i] + b0.x) * sc, (f[i + 1] + b0.y) * sc), h1 = __floats2half2_rn((f[i + 2] + b0.z) * sc, (f[i + 3] + b0.w) * sc);
          __half2 h2 = __floats2half2_rn((f[i + 4] + b1.x) * sc, (f[i + 5] + b1.y) * sc), h3 = __floats2half2_rn((f[i + 6] + b1.z) * sc, (f[i + 7] + b1.w) * sc);
          *reinterpret_cast<uint4*>(o + i) = make_uint4(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1),
                                                        *reinterpret_cast<uint32_t*>(&h2), *reinterpret_cast<uint32_t*>(&h3));
        }
    } else {
      __half* o = vT + (bh * HD + e0) * N1p + n;
#pragma unroll
      for (int i = 0; i < 32; ++i) if (i < ncols) o[(size_t)i * N1p] = __float2half_rn(f[i] + __ldg(bias + col0 + i));
    }
  }
};

// EpiQKV with the rotary embedding on q and k of the patch rows n >= pre; rope [P][32] (cos, sin) per token and pair,
// applied to acc + bias before the q scale
struct EpiQKVRope : EpiQKV {
  const float2* rope; int pre;
  __device__ __forceinline__ void operator()(State& st, int g, int r, int col0, const float (&f)[32], int ncols) const {
    if (col0 >= 2 * D) { EpiQKV::operator()(st, g, r, col0, f, ncols); return; }
    const int b = r / N1, n = r - b * N1;
    const int which = col0 / D, c = col0 - which * D, hd = c / HD, e0 = c - hd * HD;
    float* o = (which == 0 ? q : k) + (((size_t)b * heads + hd) * N1 + n) * HD + e0;
    const float sc = which == 0 ? 0.125f : 1.f;
    const float2* cs = rope + (size_t)(n - pre) * 32 + (e0 >> 1);
#pragma unroll
    for (int i = 0; i < 32; i += 2)
      if (i < ncols) {
        float a = f[i] + __ldg(bias + col0 + i), bv = f[i + 1] + __ldg(bias + col0 + i + 1);
        if (n >= pre) rope_pair(a, bv, __ldg(cs + i / 2));
        o[i] = a * sc;
        o[i + 1] = bv * sc;
      }
  }
};

// EpiQKV16 with the rotary embedding on q and k of the patch rows n >= pre (as EpiQKVRope, before the q scale and the
// fp16 rounding)
struct EpiQKV16Rope : EpiQKV16 {
  const float2* rope; int pre;
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v) const {
    const int b = fast_div(r, N1), n = r - b * N1;
    const int which = (col >= D) + (col >= 2 * D), c = col - which * D, hd = c / HD, e0 = c - hd * HD;
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col));
    const float sc = which == 0 ? qscale : 1.f;
    float a0 = v.x + bb.x, b0 = v.y + bb.y, a1 = v.z + bb.z, b1 = v.w + bb.w;
    if (n >= pre) {   // pairs e0 / 2 and e0 / 2 + 1: one 16-byte load (e0 % 4 == 0)
      const float4 cs = __ldg(reinterpret_cast<const float4*>(rope + (size_t)(n - pre) * 32 + (e0 >> 1)));
      rope_pair(a0, b0, make_float2(cs.x, cs.y));
      rope_pair(a1, b1, make_float2(cs.z, cs.w));
    }
    __half* o = (which == 0 ? q : k) + (((size_t)b * heads + hd) * N1 + n) * HD + e0;
    *reinterpret_cast<uint2*>(o) = pack_half4(a0 * sc, b0 * sc, a1 * sc, b1 * sc);
  }
  __device__ __forceinline__ void operator()(State& st, int g, int r, int col0, const float (&f)[32], int ncols) const {
    if (col0 >= 2 * D) { EpiQKV16::operator()(st, g, r, col0, f, ncols); return; }
    const int b = r / N1, n = r - b * N1;
    const int which = col0 / D, c = col0 - which * D, hd = c / HD, e0 = c - hd * HD;
    __half* o = (which == 0 ? q : k) + (((size_t)b * heads + hd) * N1 + n) * HD + e0;
    const float sc = which == 0 ? qscale : 1.f;
    const float2* cs = rope + (size_t)(n - pre) * 32 + (e0 >> 1);
#pragma unroll
    for (int i = 0; i < 32; i += 2)
      if (i < ncols) {
        float a = f[i] + __ldg(bias + col0 + i), bv = f[i + 1] + __ldg(bias + col0 + i + 1);
        if (n >= pre) rope_pair(a, bv, __ldg(cs + i / 2));
        *reinterpret_cast<__half2*>(o + i) = __floats2half2_rn(a * sc, bv * sc);
      }
  }
};

// plain store: out[(g * rows_per_group + r)][col] (attention scores)
struct EpiStore : EpiBase {
  float* out; int ld, rows_per_group;
  __device__ __forceinline__ void operator()(State&, int g, int r, int col0, const float (&f)[32], int ncols) const {
    float* o = out + ((size_t)g * rows_per_group + r) * ld + col0;
    if (ncols == 32) {
#pragma unroll
      for (int i = 0; i < 32; i += 4) *reinterpret_cast<float4*>(o + i) = make_float4(f[i], f[i + 1], f[i + 2], f[i + 3]);
    } else {
#pragma unroll
      for (int i = 0; i < 32; ++i) if (i < ncols) o[i] = f[i];
    }
  }
};

// p.v: group g = head; out[(frame_row0 + r)][g*64 + col]
struct EpiPV : EpiBase {
  float* out; size_t frame_row0; int D;
  __device__ __forceinline__ void operator()(State&, int g, int r, int col0, const float (&f)[32], int ncols) const {
    float* o = out + (frame_row0 + r) * D + g * HD + col0;
#pragma unroll
    for (int i = 0; i < 32; i += 4)
      if (i < ncols) *reinterpret_cast<float4*>(o + i) = make_float4(f[i], f[i + 1], f[i + 2], f[i + 3]);
  }
};

// x[r][col] += ls[col] * (acc + bias[col])
struct EpiResidual : EpiBase {
  static constexpr bool kCoalesced = true;
  static constexpr bool kPrefetch = true;
  float* x; const float* bias; const float* ls; int D;
  __device__ __forceinline__ float4 fetch(int, int r, int col) const { return *reinterpret_cast<const float4*>(x + (size_t)r * D + col); }
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v, float4 xv) const {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col)), ll = __ldg(reinterpret_cast<const float4*>(ls + col));
    xv.x += (v.x + bb.x) * ll.x; xv.y += (v.y + bb.y) * ll.y; xv.z += (v.z + bb.z) * ll.z; xv.w += (v.w + bb.w) * ll.w;
    *reinterpret_cast<float4*>(x + (size_t)r * D + col) = xv;
  }
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v) const {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col)), ll = __ldg(reinterpret_cast<const float4*>(ls + col));
    float4* o = reinterpret_cast<float4*>(x + (size_t)r * D + col);
    float4 xv = *o;
    xv.x += (v.x + bb.x) * ll.x; xv.y += (v.y + bb.y) * ll.y; xv.z += (v.z + bb.z) * ll.z; xv.w += (v.w + bb.w) * ll.w;
    *o = xv;
  }
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    float* o = x + (size_t)r * D + col0;
#pragma unroll
    for (int i = 0; i < 32; i += 4)
      if (i < ncols) {
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col0 + i)), ll = __ldg(reinterpret_cast<const float4*>(ls + col0 + i));
        float4 xv = *reinterpret_cast<const float4*>(o + i);
        xv.x += (f[i] + bb.x) * ll.x; xv.y += (f[i + 1] + bb.y) * ll.y; xv.z += (f[i + 2] + bb.z) * ll.z; xv.w += (f[i + 3] + bb.w) * ll.w;
        *reinterpret_cast<float4*>(o + i) = xv;
      }
  }
};

// x[r][col] += acc + bias[col]: the residual of a block without LayerScale (DINO v1; the host passes ls = nullptr).  A
// type of its own, so that the LayerScale launches keep their kernels; the sums are those of EpiResidual with ls = 1.
struct EpiResidualNoLS : EpiBase {
  static constexpr bool kCoalesced = true;
  static constexpr bool kPrefetch = true;
  float* x; const float* bias; int D;
  __device__ __forceinline__ float4 fetch(int, int r, int col) const { return *reinterpret_cast<const float4*>(x + (size_t)r * D + col); }
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v, float4 xv) const {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col));
    xv.x += v.x + bb.x; xv.y += v.y + bb.y; xv.z += v.z + bb.z; xv.w += v.w + bb.w;
    *reinterpret_cast<float4*>(x + (size_t)r * D + col) = xv;
  }
  __device__ __forceinline__ void vec4(int g, int r, int col, float4 v) const { vec4(g, r, col, v, fetch(g, r, col)); }
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    float* o = x + (size_t)r * D + col0;
#pragma unroll
    for (int i = 0; i < 32; i += 4)
      if (i < ncols) {
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col0 + i));
        float4 xv = *reinterpret_cast<const float4*>(o + i);
        xv.x += f[i] + bb.x; xv.y += f[i + 1] + bb.y; xv.z += f[i + 2] + bb.z; xv.w += f[i + 3] + bb.w;
        *reinterpret_cast<float4*>(o + i) = xv;
      }
  }
};

// 0.5 x (1 + erf(x / sqrt 2)) with erf by Abramowitz-Stegun 7.1.26 (|error| <= 1.5e-7, two MUFU + 9 FMA-pipe
// instructions, branch-free): libdevice's erff is ~3x the instructions and made the fc1 epilogue, not its MMAs, pace that
// GEMM.  The result is rounded to fp16 (relative 4.9e-4) right after.
__device__ __forceinline__ float gelu_exact(float v) {
  const float z = fabsf(v) * 0.70710678118654752f;
  float t;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(t) : "f"(fmaf(0.3275911f, z, 1.f)));      // one MUFU (1 ulp: below the 1.5e-7 of the fit)
  float p = fmaf(1.061405429f, t, -1.453152027f);
  p = fmaf(p, t, 1.421413741f);
  p = fmaf(p, t, -0.284496736f);
  p = fmaf(p, t, 0.254829592f);
  const float e = fast_exp2(-1.4426950408889634f * z * z);
  const float erf_abs = fmaf(-p * t, e, 1.f);          // erf(|v| / sqrt 2)
  // 0.5 v (1 + sign(v) erf(|v| / sqrt 2)); the explicit fmaf keeps the coalesced (vec4) and the thread-per-row
  // (CTA-pair default) epilogues bit-identical whatever contraction the compiler would pick at each call site
  return fmaf(v, 0.5f, __fmul_rn(0.5f * fabsf(v), erf_abs));
}

// h[r][col] = gelu(acc + bias[col])   (exact: 0.5 x (1 + erf(x / sqrt 2)))
template <typename OutT>
struct EpiGelu : EpiBase {
  static constexpr bool kCoalesced = true;
  OutT* h; const float* bias; int ld;
  int all_direct = 0;
  __device__ __forceinline__ bool direct(int) const { return all_direct != 0; }
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v) const {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col));
    float t[4] = {v.x + bb.x, v.y + bb.y, v.z + bb.z, v.w + bb.w};
#pragma unroll
    for (int j = 0; j < 4; ++j) t[j] = sizeof(OutT) == 4 ? 0.5f * t[j] * (1.f + erff(t[j] * 0.70710678118654752f)) : gelu_exact(t[j]);
    if constexpr (sizeof(OutT) == 4) *reinterpret_cast<float4*>(h + (size_t)r * ld + col) = make_float4(t[0], t[1], t[2], t[3]);
    else *reinterpret_cast<uint2*>(h + (size_t)r * ld + col) = pack_half4(t[0], t[1], t[2], t[3]);
  }
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    OutT* o = h + (size_t)r * ld + col0;
    float gl[32];
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col0 + (i < ncols ? i : 0)));
      const float bv[4] = {bb.x, bb.y, bb.z, bb.w};
#pragma unroll
      for (int j = 0; j < 4; ++j) {
        const float v = f[i + j] + bv[j];
        gl[i + j] = sizeof(OutT) == 4 ? 0.5f * v * (1.f + erff(v * 0.70710678118654752f)) : gelu_exact(v);
      }
    }
    if constexpr (sizeof(OutT) == 4) {
#pragma unroll
      for (int i = 0; i < 32; i += 4)
        if (i < ncols) *reinterpret_cast<float4*>(o + i) = make_float4(gl[i], gl[i + 1], gl[i + 2], gl[i + 3]);
    } else {
#pragma unroll
      for (int i = 0; i < 32; i += 8)
        if (i < ncols) {
          __half2 h0 = __floats2half2_rn(gl[i], gl[i + 1]), h1 = __floats2half2_rn(gl[i + 2], gl[i + 3]);
          __half2 h2 = __floats2half2_rn(gl[i + 4], gl[i + 5]), h3 = __floats2half2_rn(gl[i + 6], gl[i + 7]);
          *reinterpret_cast<uint4*>(o + i) = make_uint4(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1),
                                                        *reinterpret_cast<uint32_t*>(&h2), *reinterpret_cast<uint32_t*>(&h3));
        }
    }
  }
};

// silu(a) b.  fp16 path: a / (1 + 2^(-a log2 e)) with one ex2.approx and one rcp.approx (MUFU; relative error
// ~2^-21 + |a| 2^-24 from the rounded exponent argument, below the fp16 rounding of h right after); a -> -inf gives
// 2^+inf = inf and a * 0 = -0.  Explicit roundings keep the coalesced and thread-per-row calls bit-identical.
template <typename OutT>
__device__ __forceinline__ float swiglu_gate(float a, float b) {
  if constexpr (sizeof(OutT) == 4) return __fmul_rn(__fdiv_rn(a, __fadd_rn(1.f, expf(-a))), b);
  const float e = fast_exp2(__fmul_rn(-1.4426950408889634f, a));
  float r;
  asm("rcp.approx.ftz.f32 %0, %1;" : "=f"(r) : "f"(__fadd_rn(1.f, e)));
  return __fmul_rn(__fmul_rn(a, r), b);
}

// SwiGLU MLP: h[r][j] = silu(x1_j + b1_j) * (x2_j + b2_j) from the w12 GEMM of width 2 Hd, whose rows (and bias) the
// host interleaves per pair of hidden units: GEMM columns 4q .. 4q+3 = x1 of units 2q, 2q+1, then x2 of the same two.
// So every 4-column group (vec4) and every 32-column block (thread-per-row) holds whole (x1, x2) pairs, and output
// column = GEMM column / 2.  The 2 Hd-wide product never leaves the SM.  Hd % 8 == 0, so N = 2 Hd and every column
// count the GEMM passes are multiples of 16: a block's 8 or 16 outputs are one or two 16-byte fp16 stores.
template <typename OutT>
struct EpiSwiGLU : EpiBase {
  static constexpr bool kCoalesced = true;
  OutT* h; const float* bias; int ld;   // ld = Hd
  int all_direct = 0;
  __device__ __forceinline__ bool direct(int) const { return all_direct != 0; }
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v) const {
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col));
    const float g0 = swiglu_gate<OutT>(__fadd_rn(v.x, bb.x), __fadd_rn(v.z, bb.z));
    const float g1 = swiglu_gate<OutT>(__fadd_rn(v.y, bb.y), __fadd_rn(v.w, bb.w));
    OutT* o = h + (size_t)r * ld + (col >> 1);
    if constexpr (sizeof(OutT) == 4) *reinterpret_cast<float2*>(o) = make_float2(g0, g1);
    else *reinterpret_cast<__half2*>(o) = __floats2half2_rn(g0, g1);
  }
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    OutT* o = h + (size_t)r * ld + (col0 >> 1);
    float gl[16];
#pragma unroll
    for (int i = 0; i < 32; i += 4) {
      const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col0 + (i < ncols ? i : 0)));
      gl[i / 2] = swiglu_gate<OutT>(__fadd_rn(f[i], bb.x), __fadd_rn(f[i + 2], bb.z));
      gl[i / 2 + 1] = swiglu_gate<OutT>(__fadd_rn(f[i + 1], bb.y), __fadd_rn(f[i + 3], bb.w));
    }
    if constexpr (sizeof(OutT) == 4) {
#pragma unroll
      for (int i = 0; i < 16; i += 4)
        if (2 * i + 8 <= ncols) *reinterpret_cast<float4*>(o + i) = make_float4(gl[i], gl[i + 1], gl[i + 2], gl[i + 3]);
    } else {
#pragma unroll
      for (int i = 0; i < 16; i += 8)
        if (2 * i + 16 <= ncols) {
          __half2 h0 = __floats2half2_rn(gl[i], gl[i + 1]), h1 = __floats2half2_rn(gl[i + 2], gl[i + 3]);
          __half2 h2 = __floats2half2_rn(gl[i + 4], gl[i + 5]), h3 = __floats2half2_rn(gl[i + 6], gl[i + 7]);
          *reinterpret_cast<uint4*>(o + i) = make_uint4(*reinterpret_cast<uint32_t*>(&h0), *reinterpret_cast<uint32_t*>(&h1),
                                                        *reinterpret_cast<uint32_t*>(&h2), *reinterpret_cast<uint32_t*>(&h3));
        }
    }
  }
};

// query / key / value facet of the tap block: out[b][n - 1][col] = acc + bias[col] for token n >= 1 of frame b
// (row r = b N1 + n), fp32, token-major; the cls row (n = 0) is dropped
struct EpiFacet : EpiBase {
  static constexpr bool kCoalesced = true;
  float* out; const float* bias; int N1, D;
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v) const {
    const int b = fast_div(r, N1), n = r - b * N1;
    if (n == 0) return;
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col));
    *reinterpret_cast<float4*>(out + ((size_t)b * (N1 - 1) + n - 1) * D + col) =
        make_float4(v.x + bb.x, v.y + bb.y, v.z + bb.z, v.w + bb.w);
  }
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    const int b = r / N1, n = r - b * N1;
    if (n == 0) return;
    float* o = out + ((size_t)b * (N1 - 1) + n - 1) * D + col0;
#pragma unroll
    for (int i = 0; i < 32; i += 4)
      if (i < ncols) {   // ncols is a multiple of 4 (D % 64 == 0)
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col0 + i));
        *reinterpret_cast<float4*>(o + i) = make_float4(f[i] + bb.x, f[i + 1] + bb.y, f[i + 2] + bb.z, f[i + 3] + bb.w);
      }
  }
};

// EpiFacet after pre = 1 + R prefix rows: out[b][n - pre][col] for n >= pre
struct EpiFacetPrefix : EpiFacet {
  int pre;
  __device__ __forceinline__ void vec4(int, int r, int col, float4 v) const {
    const int b = fast_div(r, N1), n = r - b * N1;
    if (n < pre) return;
    const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col));
    *reinterpret_cast<float4*>(out + ((size_t)b * (N1 - pre) + n - pre) * D + col) =
        make_float4(v.x + bb.x, v.y + bb.y, v.z + bb.z, v.w + bb.w);
  }
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    const int b = r / N1, n = r - b * N1;
    if (n < pre) return;
    float* o = out + ((size_t)b * (N1 - pre) + n - pre) * D + col0;
#pragma unroll
    for (int i = 0; i < 32; i += 4)
      if (i < ncols) {
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col0 + i));
        *reinterpret_cast<float4*>(o + i) = make_float4(f[i] + bb.x, f[i + 1] + bb.y, f[i + 2] + bb.z, f[i + 3] + bb.w);
      }
  }
};

// group tables for the GEMMs: one group of `rows` rows, or `heads` groups (attention)
static int plan(const TcPlan& pl, int n_groups, int rows, int row_stride, int row_base, int batch_base, cudaStream_t st,
                int tile_rows = TC_BM) {
  ProfRange pr(PROF_VIT_MISC, st);
  return launch_tc_plan(pl, n_groups, rows, row_stride, row_base, batch_base, tile_rows, st);
}

// The linear layers run on the CTA-pair kernel (a cluster of two CTAs sharing the B tile by multicast, 256 x 256 tiles,
// single-pass fp16; the plan must be in 256-row tiles), or on the one-CTA kernel in fp16 or TF32.  a [rows][K] . w^T
static TcOperands linear_operands(const void* a, uint64_t rows, const void* w) { return {a, nullptr, rows, 0, w, nullptr, 1, 0}; }

constexpr int VIT_ROW_CHUNK = 1024;  // query rows per attention-score chunk

// fused attention over fp16 q [B*heads][N1][64] (pre-scaled by 64^-1/2 * log2 e), k [B*heads][N1][64] and
// v^T [B*heads][64][N1p] (row pitch N1p, a multiple of 8): out[b*N1 + n][h*64 + e], row pitch D, fp32 or fp16
static int launch_flash(const __half* q16, const __half* k16, const __half* v16, int B, int heads, int N1, int N1p, int D,
                        void* out, bool out_f16, cudaStream_t st) {
  CUtensorMap tmQ, tmK, tmV;
  int rc;
  if ((rc = make_tmap_2d(&tmQ, q16, (uint64_t)B * heads * N1, HD, FA_BQ, HD, TMAP_F16))) return rc;
  if ((rc = make_tmap_3d(&tmK, k16, (uint64_t)B * heads, N1, HD, FA_BKV, HD, TMAP_F16))) return rc;
  if ((rc = make_tmap_3d(&tmV, v16, (uint64_t)B * heads, HD, N1, HD, 64, TMAP_F16, (uint64_t)N1p))) return rc;
  static PerDev<bool> attr_dev;
  bool& attr = attr_dev.get();
  if (!attr) {
    DTK_CUDA(cudaFuncSetAttribute(flash_attn_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, FA_SMEM));
    attr = true;
  }
  FlashParams fpar{N1, D, heads, out, out_f16 ? 1 : 0};
  ProfRange pr(PROF_VIT_ATTN, st);
  const dim3 fgrid(cdiv(N1, FA_BQ), B * heads);
  flash_attn_kernel<<<fgrid, FA_THREADS, FA_SMEM, st>>>(tmQ, tmK, tmV, fpar);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// ---------------------------------------------------------------------------------------------- block stages
// One stage of dinotrk_vit_forward each, shared with dinotrk_vit_stage.  The linear stages after the patch embedding
// run on the tile plan of vit_row_plan (one group of all B * N1 rows); the forward makes it once per block half.
struct VitShape {
  int B, P, N1, D, heads, Kp;
  int pre;            // prefix rows per frame: cls + R registers (N1 = P + pre)
  size_t rows;        // B * N1
  bool f16, pairs;    // fp16 operands (else fp32 / TF32); linear layers on CTA pairs (fp16 only)
  float eps;          // LayerNorm eps
  const float2* rope; // [P][32] (cos, sin) of the rotary embedding, or null (no rotation)
};

// what dinotrk_vit_weights' appended fields say about the token layout; wt = null: one cls row, eps 1e-6, no RoPE
static int vit_prefix(const dinotrk_vit_weights* wt) { return 1 + (wt ? wt->n_registers : 0); }
static float vit_eps(const dinotrk_vit_weights* wt) { return wt && wt->ln_eps > 0.f ? wt->ln_eps : 1e-6f; }

// row length of the im2col matrix / patch weight: 16-byte multiple of the operand type
static int vit_kp(const dinotrk_vit_config* c) {
  const bool f16 = c->gemm_f16 != 0 && c->attn_materialized == 0;
  return (int)align_up((size_t)3 * c->patch * c->patch, f16 ? 8 : 4);
}

static VitShape vit_shape(const dinotrk_vit_config* c, const dinotrk_vit_weights* wt, const dinotrk_geom* g, int B) {
  VitShape s;
  s.B = B; s.P = g->h * g->w; s.pre = vit_prefix(wt); s.N1 = s.P + s.pre; s.D = c->dim; s.heads = c->heads; s.Kp = vit_kp(c);
  s.eps = vit_eps(wt);
  s.rope = wt ? reinterpret_cast<const float2*>(wt->rope) : nullptr;
  s.rows = (size_t)B * s.N1;
  s.f16 = c->gemm_f16 != 0 && c->attn_materialized == 0;
  s.pairs = s.f16 && c->gemm_pair != 0;
  return s;
}

static int vit_row_plan(const VitShape& s, const TcPlan& pl, cudaStream_t st) {
  return plan(pl, 1, (int)s.rows, 0, 0, 0, st, s.pairs ? TC2_BM : TC_BM);
}

// y = LayerNorm(x) (eps s.eps), x [rows][D] fp32 -> y [rows][D] (fp16 in fp16 operand mode)
static int vit_layernorm(const VitShape& s, const float* x, const float* gw, const float* gb, void* y, cudaStream_t st) {
  ProfRange pr(PROF_VIT_MISC, st);
  const unsigned grid = (unsigned)((s.rows + 7) / 8);
  if (s.f16) vit_layernorm_kernel<__half><<<grid, 256, 0, st>>>(x, gw, gb, reinterpret_cast<__half*>(y), s.rows, s.D, s.eps);
  else vit_layernorm_kernel<float><<<grid, 256, 0, st>>>(x, gw, gb, reinterpret_cast<float*>(y), s.rows, s.D, s.eps);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// x[b][pre + p] = cols[b P + p] . patch_w + bias (+ pos[p] when pos); cols [B P][Kp] (makes its own 128-row tile plan)
template <class Epi>
static int vit_patch_launch(const VitShape& s, const TcPlan& pl, const void* cols, const void* w, const Epi& ep, cudaStream_t st) {
  int rc;
  if ((rc = plan(pl, 1, s.B * s.P, 0, 0, 0, st))) return rc;
  const TcOperands op = linear_operands(cols, (uint64_t)s.B * s.P, w);
  const int tiles = cdiv(s.B * s.P, TC_BM);
  return s.f16 ? tc_launch<TcMode::F16, Epi>(op, pl.problem(1, s.D, s.Kp), tiles, ep, st, PROF_VIT_GEMM)
               : tc_launch<TcMode::TF32, Epi>(op, pl.problem(1, s.D, s.Kp), tiles, ep, st, PROF_VIT_GEMM);
}
static int vit_patch_embed(const VitShape& s, const TcPlan& pl, const void* cols, const void* w, const float* bias,
                           const float* pos, float* x, cudaStream_t st) {
  if (s.pre == 1 && pos) return vit_patch_launch(s, pl, cols, w, EpiPatch{{}, x, bias, pos, s.P, s.D}, st);
  return vit_patch_launch(s, pl, cols, w, EpiPatchPrefix{{{}, x, bias, pos, s.P, s.D}, s.pre}, st);
}

// qkv for the fused attention: y [rows][D] . qkv_w^T + bias -> fp16 q (scaled by 64^-1/2 log2 e), k, v^T (pitch align8(N1));
// with s.rope, q and k of the patch rows rotated first
template <class Epi>
static int vit_qkv_launch(const VitShape& s, const TcPlan& pl, const void* y, const void* w, const Epi& eq, cudaStream_t st) {
  const TcOperands op = linear_operands(y, s.rows, w);
  const TcProblem pb = pl.problem(1, 3 * s.D, s.D);
  const int tiles = cdiv((int)s.rows, TC_BM);
  return s.pairs ? tc_launch<TcMode::F16, Epi, TC_BN, true>(op, pb, cdiv((int)s.rows, TC2_BM), eq, st, PROF_VIT_GEMM)
       : s.f16 ? tc_launch<TcMode::F16, Epi>(op, pb, tiles, eq, st, PROF_VIT_GEMM)
               : tc_launch<TcMode::TF32, Epi>(op, pb, tiles, eq, st, PROF_VIT_GEMM);
}
static int vit_qkv_fused(const VitShape& s, const TcPlan& pl, const void* y, const void* w, const float* bias, __half* q16,
                         __half* k16, __half* v16, cudaStream_t st) {
  const int D = s.D, N1p8 = (int)align_up((size_t)s.N1, 8);
  EpiQKV16 eq{{}, q16, k16, v16, bias, s.N1, D, s.heads, N1p8, 0.125f * 1.4426950408889634f};  // 1/sqrt(64) * log2(e)
  eq.direct_from = 2 * D;   // v^T rows thread-per-row; q / k that way too measured slower
  if (!s.rope) return vit_qkv_launch(s, pl, y, w, eq, st);
  return vit_qkv_launch(s, pl, y, w, EpiQKV16Rope{eq, s.rope, s.pre}, st);
}

// x[r] += ls * (a[r] . w^T + bias), a [rows][K]: proj (K = D) and fc2 (K = 4 D); ls = nullptr: no LayerScale
template <class Epi>
static int vit_residual_launch(const VitShape& s, const TcPlan& pl, const void* a, const void* w, int K, const Epi& er,
                               cudaStream_t st) {
  const TcOperands op = linear_operands(a, s.rows, w);
  const TcProblem pb = pl.problem(1, s.D, K);
  const int tiles = cdiv((int)s.rows, TC_BM);
  return s.pairs ? tc_launch<TcMode::F16, Epi, TC_BN, true>(op, pb, cdiv((int)s.rows, TC2_BM), er, st, PROF_VIT_GEMM)
       : s.f16 ? tc_launch<TcMode::F16, Epi>(op, pb, tiles, er, st, PROF_VIT_GEMM)
               : tc_launch<TcMode::TF32, Epi>(op, pb, tiles, er, st, PROF_VIT_GEMM);
}
static int vit_residual(const VitShape& s, const TcPlan& pl, const void* a, const void* w, int K, const float* bias,
                        const float* ls, float* x, cudaStream_t st) {
  if (!ls) return vit_residual_launch(s, pl, a, w, K, EpiResidualNoLS{{}, x, bias, s.D}, st);
  return vit_residual_launch(s, pl, a, w, K, EpiResidual{{}, x, bias, ls, s.D}, st);
}

// h = gelu(y . fc1_w^T + bias), y [rows][D] -> h [rows][4 D] (fp16 in fp16 operand mode)
static int vit_fc1(const VitShape& s, const TcPlan& pl, const void* y, const void* w, const float* bias, void* h, cudaStream_t st) {
  const int D = s.D;
  const TcOperands op = linear_operands(y, s.rows, w);
  const TcProblem pb = pl.problem(1, 4 * D, D);
  const int tiles = cdiv((int)s.rows, TC_BM);
  if (s.pairs) {
    EpiGelu<__half> eg{{}, reinterpret_cast<__half*>(h), bias, 4 * D};
    eg.all_direct = 1;   // fp16 GELU rows written thread-per-row (64 B per thread, whole sectors)
    return tc_launch<TcMode::F16, EpiGelu<__half>, TC_BN, true>(op, pb, cdiv((int)s.rows, TC2_BM), eg, st, PROF_VIT_GEMM);
  }
  if (s.f16)
    return tc_launch<TcMode::F16, EpiGelu<__half>>(op, pb, tiles, EpiGelu<__half>{{}, reinterpret_cast<__half*>(h), bias, 4 * D}, st,
                                                   PROF_VIT_GEMM);
  return tc_launch<TcMode::TF32, EpiGelu<float>>(op, pb, tiles, EpiGelu<float>{{}, reinterpret_cast<float*>(h), bias, 4 * D}, st,
                                                 PROF_VIT_GEMM);
}

// h = silu(x1) * x2, [x1 x2] = y . w12^T + bias (rows interleaved, see EpiSwiGLU), y [rows][D] -> h [rows][Hd]
static int vit_swiglu(const VitShape& s, const TcPlan& pl, const void* y, const void* w, const float* bias, int Hd, void* h,
                      cudaStream_t st) {
  const TcOperands op = linear_operands(y, s.rows, w);
  const TcProblem pb = pl.problem(1, 2 * Hd, s.D);
  const int tiles = cdiv((int)s.rows, TC_BM);
  if (s.pairs) {
    EpiSwiGLU<__half> eg{{}, reinterpret_cast<__half*>(h), bias, Hd};
    eg.all_direct = 1;   // as fc1 on CTA pairs: each thread writes its row's 16 outputs per 32 columns as whole sectors
    return tc_launch<TcMode::F16, EpiSwiGLU<__half>, TC_BN, true>(op, pb, cdiv((int)s.rows, TC2_BM), eg, st, PROF_VIT_GEMM);
  }
  if (s.f16)
    return tc_launch<TcMode::F16, EpiSwiGLU<__half>>(op, pb, tiles, EpiSwiGLU<__half>{{}, reinterpret_cast<__half*>(h), bias, Hd},
                                                     st, PROF_VIT_GEMM);
  return tc_launch<TcMode::TF32, EpiSwiGLU<float>>(op, pb, tiles, EpiSwiGLU<float>{{}, reinterpret_cast<float*>(h), bias, Hd},
                                                   st, PROF_VIT_GEMM);
}

// facet f of the tap block: out_tpc [B][P][D] = (y . qkv_w[(f-1) D : f D]^T + qkv_b[(f-1) D : f D]) without the cls rows.
// The weight slice starts (f-1) D^2 elements into qkv_w; the caller checks that it and the bias slice are 16-byte aligned
// (the TMA base and the epilogue's float4 bias reads).
template <class Epi>
static int vit_facet_launch(const VitShape& s, const TcPlan& pl, const void* y, const void* w_slice, const Epi& ef,
                            cudaStream_t st) {
  const TcOperands op = linear_operands(y, s.rows, w_slice);
  const TcProblem pb = pl.problem(1, s.D, s.D);
  const int tiles = cdiv((int)s.rows, TC_BM);
  return s.pairs ? tc_launch<TcMode::F16, Epi, TC_BN, true>(op, pb, cdiv((int)s.rows, TC2_BM), ef, st, PROF_VIT_GEMM)
       : s.f16 ? tc_launch<TcMode::F16, Epi>(op, pb, tiles, ef, st, PROF_VIT_GEMM)
               : tc_launch<TcMode::TF32, Epi>(op, pb, tiles, ef, st, PROF_VIT_GEMM);
}
static int vit_facet(const VitShape& s, const TcPlan& pl, const void* y, const void* w_slice, const float* bias_slice,
                     float* out_tpc, cudaStream_t st) {
  const EpiFacet ef{{}, out_tpc, bias_slice, s.N1, s.D};
  if (s.pre == 1) return vit_facet_launch(s, pl, y, w_slice, ef, st);
  return vit_facet_launch(s, pl, y, w_slice, EpiFacetPrefix{ef, s.pre}, st);
}

// the activations of a forward; the MLP hidden buffer is also the patch embedding's im2col
struct VitWs {
  float *x, *y, *q, *k, *vT, *hbuf, *S; TcPlan pl;
  VitWs(Arena& ar, const dinotrk_vit_config& c, const dinotrk_geom& g, int B, int pre) {
    const size_t P = (size_t)g.h * g.w, rows = (size_t)B * (P + pre), D = c.dim, N1p = align_up(P + pre, 4);
    x = ar.take<float>(rows * D);
    y = ar.take<float>(rows * D);
    q = ar.take<float>(rows * D);
    k = ar.take<float>(rows * D);
    vT = ar.take<float>((size_t)B * N1p * D);
    const size_t hid = rows * (c.swiglu_hidden > 0 ? (size_t)c.swiglu_hidden : 4 * D), col = (size_t)B * P * vit_kp(&c);
    hbuf = ar.take<float>(hid > col ? hid : col);
    S = ar.take<float>((size_t)c.heads * VIT_ROW_CHUNK * N1p);   // attention scores of one row chunk
    pl = TcPlan{ar.take<int>(c.heads + 2), ar.take<int>(c.heads + 2), ar.take<int>(c.heads + 2), ar.take<int>(c.heads + 2)};
  }
};

}  // namespace dtk

using namespace dtk;

extern "C" {

size_t dinotrk_vit_workspace_bytes_ext(const dinotrk_vit_config* c, const dinotrk_vit_weights* wt, const dinotrk_geom* g, int B) {
  if (!c || !g) return 0;
  return align_up(layout_end<VitWs>(*c, *g, B, vit_prefix(wt)), 256) + 4096;
}

size_t dinotrk_vit_workspace_bytes(const dinotrk_vit_config* c, const dinotrk_geom* g, int B) {
  return dinotrk_vit_workspace_bytes_ext(c, nullptr, g, B);
}

int dinotrk_vit_attention(const void* q16, const void* k16, const void* vT16, int B, int heads, int N1, int N1p,
                          float* out, void* stream) {
  DTK_CHECK_ARG(q16 && k16 && vT16 && out, "vit_attention: null pointer");
  DTK_CHECK_ARG(B > 0 && heads > 0 && N1 > 0 && N1p >= N1 && N1p % 8 == 0, "vit_attention: bad sizes");
  return launch_flash(reinterpret_cast<const __half*>(q16), reinterpret_cast<const __half*>(k16),
                      reinterpret_cast<const __half*>(vT16), B, heads, N1, N1p, heads * HD, out, false, (cudaStream_t)stream);
}

int dinotrk_vit_attention_f16(const void* q16, const void* k16, const void* vT16, int B, int heads, int N1, int N1p,
                              void* out16, void* stream) {
  DTK_CHECK_ARG(q16 && k16 && vT16 && out16, "vit_attention_f16: null pointer");
  DTK_CHECK_ARG(B > 0 && heads > 0 && N1 > 0 && N1p >= N1 && N1p % 8 == 0, "vit_attention_f16: bad sizes");
  return launch_flash(reinterpret_cast<const __half*>(q16), reinterpret_cast<const __half*>(k16),
                      reinterpret_cast<const __half*>(vT16), B, heads, N1, N1p, heads * HD, out16, true, (cudaStream_t)stream);
}

int dinotrk_vit_stage_ext(int stage, const dinotrk_vit_config* c, const dinotrk_vit_weights* wt, const dinotrk_geom* g, int B,
                          const void* in, const void* w, const float* p0, const float* p1, void* out0, void* out1, void* out2,
                          void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(c && g && in && p0 && out0, "vit_stage: null pointer");
  DTK_CHECK_ARG(!wt || wt->n_registers >= 0, "vit_stage: negative register count");
  const bool rope = wt && wt->rope;
  DTK_CHECK_ARG(stage >= DINOTRK_VIT_LAYERNORM && stage <= DINOTRK_VIT_SWIGLU, "vit_stage: unknown stage %d", stage);
  DTK_CHECK_ARG(c->gemm_f16 != 0 && c->attn_materialized == 0, "vit_stage: fp16 operand mode only");
  DTK_CHECK_ARG(B > 0 && c->dim == c->heads * HD && c->dim <= 2048, "vit_stage: dim must be heads x 64 (<= 2048)");
  DTK_CHECK_ARG(c->swiglu_hidden >= 0 && c->swiglu_hidden % 8 == 0, "vit_stage: swiglu_hidden must be a multiple of 8");
  DTK_CHECK_ARG(stage != DINOTRK_VIT_SWIGLU || c->swiglu_hidden > 0, "vit_stage: the SwiGLU stage needs swiglu_hidden > 0");
  DTK_CHECK_ARG(stage == DINOTRK_VIT_LAYERNORM || w, "vit_stage: null weight");
  DTK_CHECK_ARG(stage != DINOTRK_VIT_LAYERNORM || p1, "vit_stage: null LayerNorm bias");
  DTK_CHECK_ARG(stage != DINOTRK_VIT_PATCH || p1 || rope, "vit_stage: null position table (only a RoPE model has none)");
  DTK_CHECK_ARG(stage != DINOTRK_VIT_QKV || (out1 && out2), "vit_stage: qkv needs q, k and v^T");
  DTK_CHECK_ARG(workspace && workspace_bytes >= DINOTRK_VIT_STAGE_WORKSPACE_BYTES, "vit_stage: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const VitShape s = vit_shape(c, wt, g, B);
  Arena ar(workspace);
  TcPlan pl{ar.take<int>(2), ar.take<int>(2), ar.take<int>(2), ar.take<int>(2)};
  if (stage == DINOTRK_VIT_LAYERNORM) return vit_layernorm(s, reinterpret_cast<const float*>(in), p0, p1, out0, st);
  if (stage == DINOTRK_VIT_PATCH) return vit_patch_embed(s, pl, in, w, p0, p1, reinterpret_cast<float*>(out0), st);
  int rc;
  if ((rc = vit_row_plan(s, pl, st))) return rc;
  switch (stage) {
    case DINOTRK_VIT_QKV:
      return vit_qkv_fused(s, pl, in, w, p0, reinterpret_cast<__half*>(out0), reinterpret_cast<__half*>(out1),
                           reinterpret_cast<__half*>(out2), st);
    case DINOTRK_VIT_PROJ: return vit_residual(s, pl, in, w, s.D, p0, p1, reinterpret_cast<float*>(out0), st);
    case DINOTRK_VIT_FC1: return vit_fc1(s, pl, in, w, p0, out0, st);
    case DINOTRK_VIT_SWIGLU: return vit_swiglu(s, pl, in, w, p0, c->swiglu_hidden, out0, st);
    default:
      return vit_residual(s, pl, in, w, c->swiglu_hidden ? c->swiglu_hidden : 4 * s.D, p0, p1, reinterpret_cast<float*>(out0), st);
  }
}

int dinotrk_vit_stage(int stage, const dinotrk_vit_config* c, const dinotrk_geom* g, int B, const void* in, const void* w,
                      const float* p0, const float* p1, void* out0, void* out1, void* out2, void* workspace,
                      size_t workspace_bytes, void* stream) {
  return dinotrk_vit_stage_ext(stage, c, nullptr, g, B, in, w, p0, p1, out0, out1, out2, workspace, workspace_bytes, stream);
}

int dinotrk_vit_forward(const float* frames, int B, const dinotrk_geom* g, const dinotrk_vit_config* c,
                        const dinotrk_vit_weights* wt, float* out_tpc, void* workspace, size_t workspace_bytes,
                        void* stream) {
  NvtxRange nvtx_range("dinotrk.vit_forward");
  DTK_CHECK_ARG(frames && g && c && wt && out_tpc && wt->blocks && wt->cls_pos, "vit_forward: null pointer");
  DTK_CHECK_ARG(wt->n_registers >= 0 && (wt->n_registers == 0 || wt->registers), "vit_forward: register rows missing");
  DTK_CHECK_ARG(wt->pos || wt->rope, "vit_forward: a model without a position table needs the RoPE table");
  const int D = c->dim, heads = c->heads, P = g->h * g->w, pre = vit_prefix(wt), N1 = P + pre, Kp = vit_kp(c);
  DTK_CHECK_ARG(D == heads * HD && D % 64 == 0 && D <= 2048, "vit_forward: dim must be heads x 64 (<= 2048)");
  DTK_CHECK_ARG(c->tap_layer >= 0 && c->tap_layer < c->depth, "vit_forward: tap layer out of range");
  DTK_CHECK_ARG(c->swiglu_hidden >= 0 && c->swiglu_hidden % 8 == 0, "vit_forward: swiglu_hidden must be a multiple of 8");
  DTK_CHECK_ARG(c->facet >= 0 && c->facet <= 3, "vit_forward: facet must be 0 (tokens), 1 (queries), 2 (keys) or 3 (values)");
  const int Hd = c->swiglu_hidden, hid_k = Hd ? Hd : 4 * D;   // MLP hidden width: the K of fc2 / w3
  const int N1p = (int)align_up((size_t)N1, 4);   // row pitch of the score / v^T arrays (TMA strides are 16-byte multiples)
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_vit_workspace_bytes_ext(c, wt, g, B), "vit_forward: workspace too small");
  // fp16 operand mode (default): LayerNorm / GELU / attention write fp16 activations, weights are fp16 (11-bit
  // significand like TF32, twice the tensor rate, half the operand traffic).  The validation path
  // (attn_materialized) keeps every operand fp32 / TF32.
  const VitShape s = vit_shape(c, wt, g, B);
  const bool f16 = s.f16;
  // facet > 0: the features are the tap block's qkv Linear output (what the reference's qkv hook records), rows
  // [(f-1) D, f D) of qkv.w and qkv.b -- one N = D GEMM after that block's LayerNorm 1, written straight into out_tpc;
  // the block's attention and MLP do not run.  The slices are the GEMM's TMA base and its float4 bias reads.
  const void* facet_w = nullptr;
  const float* facet_b = nullptr;
  if (c->facet) {
    const float* const* wtap = wt->blocks + (size_t)c->tap_layer * 14;
    const size_t off = (size_t)(c->facet - 1) * D;
    facet_w = reinterpret_cast<const char*>(wtap[2]) + off * D * (f16 ? sizeof(__half) : sizeof(float));
    facet_b = wtap[3] + off;
    DTK_CHECK_ARG(wtap[2] && wtap[3] && ((uintptr_t)facet_w & 15) == 0 && ((uintptr_t)facet_b & 15) == 0,
                  "vit_forward: qkv weight / bias of the tap block not 16-byte aligned");
  }
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(workspace);
  const VitWs ws(ar, *c, *g, B, pre);
  const size_t rows = (size_t)B * N1;
  float *x = ws.x, *y = ws.y, *q = ws.q, *k = ws.k, *vT = ws.vT, *hbuf = ws.hbuf, *S = ws.S;
  const TcPlan pl = ws.pl;
  int rc;
  // y and hbuf hold fp16 activations in fp16 operand mode, fp32 ones otherwise
  __half* h16 = reinterpret_cast<__half*>(hbuf);

  // ---- patch embedding + cls + position embedding
  {
    ProfRange pr(PROF_VIT_MISC, st);
    if (f16) vit_im2col_kernel<__half><<<B * P, 128, 0, st>>>(frames, h16, B, g->H, g->W, g->h, g->w, c->patch, c->stride, Kp);
    else vit_im2col_kernel<float><<<B * P, 128, 0, st>>>(frames, hbuf, B, g->H, g->W, g->h, g->w, c->patch, c->stride, Kp);
    DTK_LAUNCHED();
  }
  if ((rc = vit_patch_embed(s, pl, hbuf, wt->patch_w, wt->patch_b, wt->rope ? nullptr : wt->pos, x, st))) return rc;
  {
    ProfRange pr(PROF_VIT_MISC, st);
    vit_cls_kernel<<<B, 256, 0, st>>>(x, wt->cls_pos, wt->registers, pre, N1, D);
    DTK_LAUNCHED();
  }

  const int all_tiles = cdiv((int)rows, TC_BM);
  for (int l = 0; l <= c->tap_layer; ++l) {
    const float* const* w = wt->blocks + (size_t)l * 14;
    // w: 0 norm1.w 1 norm1.b 2 qkv.w 3 qkv.b 4 proj.w 5 proj.b 6 ls1 7 norm2.w 8 norm2.b 9 fc1.w 10 fc1.b 11 fc2.w 12 fc2.b 13 ls2
    // (ls1 / ls2 null: no LayerScale, DINO v1)
    // (the four weight matrices are fp16 arrays in fp16 operand mode; SwiGLU: 9-12 are w12.w, w12.b, w3.w, w3.b)
    if ((rc = vit_layernorm(s, x, w[0], w[1], y, st))) return rc;
    if ((rc = vit_row_plan(s, pl, st))) return rc;
    if (facet_w && l == c->tap_layer) return vit_facet(s, pl, y, facet_w, facet_b, out_tpc, st);
    if (c->attn_materialized == 0) {
      // fused attention: fp16 q / k / v^T, scores stay in registers
      __half* q16 = reinterpret_cast<__half*>(q);
      __half* k16 = reinterpret_cast<__half*>(k);
      __half* v16 = reinterpret_cast<__half*>(vT);
      if ((rc = vit_qkv_fused(s, pl, y, w[2], w[3], q16, k16, v16, st))) return rc;
      if ((rc = launch_flash(q16, k16, v16, B, heads, N1, (int)align_up((size_t)N1, 8), D, y, f16, st))) return rc;
    } else {
      const EpiQKV eq{{}, q, k, vT, w[3], N1, D, heads, N1p};
      const TcOperands op = linear_operands(y, rows, w[2]);
      if ((rc = s.rope ? tc_launch<TcMode::TF32, EpiQKVRope>(op, pl.problem(1, 3 * D, D), all_tiles, EpiQKVRope{eq, s.rope, pre}, st,
                                                           PROF_VIT_GEMM)
                       : tc_launch<TcMode::TF32, EpiQKV>(op, pl.problem(1, 3 * D, D), all_tiles, eq, st, PROF_VIT_GEMM))) return rc;
      // attention, per frame and chunk of query rows: S = q k^T (all heads) -> softmax -> y = S v
      for (int b = 0; b < B; ++b) {
        for (int c0 = 0; c0 < N1; c0 += VIT_ROW_CHUNK) {
          const int rc_rows = N1 - c0 < VIT_ROW_CHUNK ? N1 - c0 : VIT_ROW_CHUNK;
          if ((rc = plan(pl, heads, rc_rows, N1, (b * heads) * N1 + c0, b * heads, st))) return rc;
          if ((rc = tc_launch<TcMode::TF32, EpiStore>({q, nullptr, rows * heads, 0, k, nullptr, (uint64_t)B * heads, 0},
                                                      pl.problem(heads, N1, HD), heads * cdiv(rc_rows, TC_BM),
                                                      EpiStore{{}, S, N1p, VIT_ROW_CHUNK}, st, PROF_VIT_ATTN))) return rc;
          {
            const size_t smem = (size_t)N1 * 4;   // one score row; above 48 KiB from 12,288 tokens (e.g. 714 x 1274 frames)
            static PerDev<size_t> attr_dev;
            if (smem > 48 * 1024 && smem > attr_dev.get()) {
              DTK_CHECK_ARG(smem <= 227 * 1024, "vit: %d tokens exceed the materialized attention's score row", N1);
              DTK_CUDA(cudaFuncSetAttribute(vit_softmax_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
              attr_dev.get() = smem;
            }
            ProfRange pr(PROF_VIT_ATTN, st);  // rows of S live at (head * VIT_ROW_CHUNK + r)
            vit_softmax_kernel<<<dim3(rc_rows, heads), 256, smem, st>>>(S, N1, N1p, (size_t)VIT_ROW_CHUNK * N1p);
            DTK_LAUNCHED();
          }
          if ((rc = plan(pl, heads, rc_rows, VIT_ROW_CHUNK, 0, b * heads, st))) return rc;
          if ((rc = tc_launch<TcMode::TF32, EpiPV, 64>({S, nullptr, (uint64_t)heads * VIT_ROW_CHUNK, (uint64_t)N1p, vT, nullptr,
                                                        (uint64_t)B * heads, (uint64_t)N1p},
                                                       pl.problem(heads, HD, N1), heads * cdiv(rc_rows, TC_BM),
                                                       EpiPV{{}, y, (size_t)b * N1 + c0, D}, st, PROF_VIT_ATTN))) return rc;
        }
      }
    }
    if ((rc = vit_row_plan(s, pl, st))) return rc;
    if ((rc = vit_residual(s, pl, y, w[4], D, w[5], w[6], x, st))) return rc;              // proj + LayerScale + residual
    if ((rc = vit_layernorm(s, x, w[7], w[8], y, st))) return rc;
    if (Hd) {
      if ((rc = vit_swiglu(s, pl, y, w[9], w[10], Hd, hbuf, st))) return rc;
    } else {
      if ((rc = vit_fc1(s, pl, y, w[9], w[10], hbuf, st))) return rc;
    }
    if ((rc = vit_residual(s, pl, hbuf, w[11], hid_k, w[12], w[13], x, st))) return rc;   // fc2 / w3 + LayerScale + residual
  }
  {
    ProfRange pr(PROF_VIT_MISC, st);
    size_t tot = (size_t)B * P * (D / 4);
    vit_tap_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(x, out_tpc, B, P, pre, D);
    DTK_LAUNCHED();
  }
  return DINOTRK_OK;
}

}  // extern "C"

// Delta-DINO: 4 x [conv5x5 (reflect pad, dilation d) + BatchNorm(eval) (+ ReLU + BlurPool)] and the
// resampling of its output onto the ViT token grid, fused with the residual add
// (models/networks/delta_dino.py:8-61, models/utils.py:7-45, models/tracker.py:113-129).
//
// Activations are NHWC fp32.  Each convolution is an implicit GEMM (M = output pixels, N = C_out,
// K = 25 taps x C_in, K-major weights with the BatchNorm folded in on the host) on the same
// 128 x 128 x 16 cp.async pipeline as the correlation GEMM; the im2col gather (reflection, dilation)
// happens in the cp.async address computation, nothing is materialised.
#include <cuda_fp16.h>

#include <utility>

#include "common.cuh"
#include "corr.cuh"
#include "delta.cuh"
#include "tcgemm.cuh"

namespace dtk {

constexpr int CBM = 128, CBN = 128, CBK = 16, CKPAD = 20, CSTAGES = 3;
constexpr int CONV_THREADS = 256;
constexpr int CONV_SMEM = CSTAGES * (CBM + CBN) * CKPAD * 4;

__device__ __forceinline__ void cp16(void* smem, const void* gmem, bool valid) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}

__global__ void __launch_bounds__(CONV_THREADS, 2)
conv5x5_kernel(const float* __restrict__ in, const float* __restrict__ wgt, const float* __restrict__ bias,
               float* __restrict__ out, ConvShape cs) {
  extern __shared__ __align__(16) float smem[];
  const int M = cs.B * cs.H * cs.W, K = 25 * cs.Cin;
  const int m0 = blockIdx.x * CBM, n0 = blockIdx.y * CBN;
  const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;

  // the two A rows (output pixels) this thread gathers, and the two B rows (output channels)
  int pb[2], py[2], px[2];
  bool pv[2];
#pragma unroll
  for (int it = 0; it < 2; ++it) {
    int r = (tid + it * CONV_THREADS) >> 2;
    int m = m0 + r;
    pv[it] = m < M;
    int mm = pv[it] ? m : 0;
    pb[it] = mm / (cs.H * cs.W);
    int rem = mm - pb[it] * cs.H * cs.W;
    py[it] = rem / cs.W;
    px[it] = rem - py[it] * cs.W;
  }
  const int c4 = (tid & 3) * 4;

  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  const int KT = (K + CBK - 1) / CBK;
  auto load_stage = [&](int kt, int s) {
    float* sa = smem + s * (CBM + CBN) * CKPAD;
    float* sb = sa + CBM * CKPAD;
    const int k = kt * CBK + c4;
    const bool kin = k < K;
    const int tap = kin ? k / cs.Cin : 0;
    const int ci = kin ? k - tap * cs.Cin : 0;
    const int ky = tap / 5, kx = tap - ky * 5;
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      int r = (tid + it * CONV_THREADS) >> 2;
      int sy = reflect(py[it] + (ky - 2) * cs.dil, cs.H), sx = reflect(px[it] + (kx - 2) * cs.dil, cs.W);
      const float* src = in + (((size_t)pb[it] * cs.H + sy) * cs.W + sx) * cs.Cin + ci;
      bool va = kin && pv[it];
      cp16(sa + r * CKPAD + c4, va ? src : in, va);
      int n = n0 + r;
      bool vb = kin && n < cs.Cout;
      cp16(sb + r * CKPAD + c4, vb ? wgt + (size_t)n * K + k : wgt, vb);
    }
  };

#pragma unroll
  for (int s = 0; s < CSTAGES - 1; ++s) {
    if (s < KT) load_stage(s, s);
    asm volatile("cp.async.commit_group;\n" ::);
  }
  for (int kt = 0; kt < KT; ++kt) {
    asm volatile("cp.async.wait_group %0;\n" ::"n"(CSTAGES - 2));
    __syncthreads();
    {
      int nk = kt + CSTAGES - 1;
      if (nk < KT) load_stage(nk, nk % CSTAGES);
      asm volatile("cp.async.commit_group;\n" ::);
    }
    const float* sa = smem + (kt % CSTAGES) * (CBM + CBN) * CKPAD;
    const float* sb = sa + CBM * CKPAD;
#pragma unroll
    for (int kk = 0; kk < CBK; kk += 4) {
      float4 a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = *reinterpret_cast<const float4*>(sa + (ty + 16 * i) * CKPAD + kk);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float4 b = *reinterpret_cast<const float4*>(sb + (tx + 16 * j) * CKPAD + kk);
#pragma unroll
        for (int i = 0; i < 8; ++i) {
          acc[i][j] = fmaf(a[i].x, b.x, acc[i][j]);
          acc[i][j] = fmaf(a[i].y, b.y, acc[i][j]);
          acc[i][j] = fmaf(a[i].z, b.z, acc[i][j]);
          acc[i][j] = fmaf(a[i].w, b.w, acc[i][j]);
        }
      }
    }
  }
  asm volatile("cp.async.wait_group 0;\n" ::);

  float bv[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) bv[j] = (n0 + tx + 16 * j) < cs.Cout ? bias[n0 + tx + 16 * j] : 0.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int m = m0 + ty + 16 * i;
    if (m >= M) continue;
    float* o = out + (size_t)m * cs.Cout + n0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int c = tx + 16 * j;
      if (n0 + c < cs.Cout) {
        float v = acc[i][j] + bv[j];
        o[c] = cs.relu ? fmaxf(v, 0.f) : v;
      }
    }
  }
}

// RGB frames [B][3][H][W] (reference layout) -> NHWC with a zero 4th channel
__global__ void rgb_to_nhwc4_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int HW) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)B * HW) return;
  size_t b = i / HW, p = i - b * HW;
  const float* s = in + b * 3 * HW + p;
  reinterpret_cast<float4*>(out)[i] = make_float4(s[0], s[HW], s[2 * HW], 0.f);
}

// antialiased_cnns.BlurPool(stride 2, filt 4): reflect pad (1,2,1,2), depthwise outer([1,3,3,1])/64.
__global__ void blurpool_kernel(const float* __restrict__ in, float* __restrict__ out, int B, int H, int W, int C,
                                int Ho, int Wo) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;  // over B*Ho*Wo*(C/4)
  const int C4 = C >> 2;
  size_t total = (size_t)B * Ho * Wo * C4;
  if (i >= total) return;
  int c4 = (int)(i % C4);
  size_t p = i / C4;
  int ox = (int)(p % Wo);
  size_t q = p / Wo;
  int oy = (int)(q % Ho);
  int b = (int)(q / Ho);
  const float f[4] = {1.f / 8.f, 3.f / 8.f, 3.f / 8.f, 1.f / 8.f};
  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
  for (int ky = 0; ky < 4; ++ky) {
    int sy = reflect(2 * oy + ky - 1, H);
#pragma unroll
    for (int kx = 0; kx < 4; ++kx) {
      int sx = reflect(2 * ox + kx - 1, W);
      float wv = f[ky] * f[kx];  // exact: (1|3)*(1|3)/64
      float4 v = __ldg(reinterpret_cast<const float4*>(in + (((size_t)b * H + sy) * W + sx) * C) + c4);
      acc.x = fmaf(v.x, wv, acc.x); acc.y = fmaf(v.y, wv, acc.y);
      acc.z = fmaf(v.z, wv, acc.z); acc.w = fmaf(v.w, wv, acc.w);
    }
  }
  reinterpret_cast<float4*>(out + (((size_t)b * Ho + oy) * Wo + ox) * C)[c4] = acc;
}

// refined[t][p][:] = dino[t][p][:] + bilinear(cnn[t], iy[r], ix[c])   (grid_sample border, align_corners=True)
// ix/iy: un-normalised, clipped source coordinates per token column / row (computed on the host with the
// reference's fp32 arithmetic, models/utils.py:31-43).
// When `peers` is set (frame-sharded multi-GPU run), every refined row is also stored into the same slot of each
// peer GPU's feature video through its NVLink-mapped pointer: the all-gather of the refined features is fused into
// this epilogue (stores to mapped peer memory; no separate collective, no staging copy).
struct PeerOut {
  float* base[8];       // peers' [T][P][C] buffers (device pointers mapped with cudaIpcOpenMemHandle)
  int n;                // number of peers (0: single GPU)
  size_t row_offset;    // row (t*P + p) of this call's first output row inside the peers' buffers
};

__global__ void align_add_kernel(const float* __restrict__ cnn, const float* __restrict__ dino,
                                 float* __restrict__ refined, const float* __restrict__ ixs,
                                 const float* __restrict__ iys, int Hc, int Wc, int C, int h, int w, PeerOut peers) {
  const int p = blockIdx.x, b = blockIdx.y;
  const int r = p / w, c = p - r * w;
  const float ix = ixs[c], iy = iys[r];
  const float x0f = floorf(ix), y0f = floorf(iy);
  const int x0 = (int)x0f, y0 = (int)y0f, x1 = x0 + 1, y1 = y0 + 1;
  // ATen grid_sampler_2d: nw = (ix_se - ix) * (iy_se - iy), ne = (ix - ix_sw) * (iy_sw - iy), ...
  const float wnw = (x0f + 1.f - ix) * (y0f + 1.f - iy), wne = (ix - x0f) * (y0f + 1.f - iy);
  const float wsw = (x0f + 1.f - ix) * (iy - y0f), wse = (ix - x0f) * (iy - y0f);
  const bool okx1 = x1 <= Wc - 1, oky1 = y1 <= Hc - 1;
  const float4* base = reinterpret_cast<const float4*>(cnn + (size_t)b * Hc * Wc * C);
  const int C4 = C >> 2;
  const float4* pnw = base + ((size_t)y0 * Wc + x0) * C4;
  const float4* pne = base + ((size_t)y0 * Wc + (okx1 ? x1 : x0)) * C4;
  const float4* psw = base + ((size_t)(oky1 ? y1 : y0) * Wc + x0) * C4;
  const float4* pse = base + ((size_t)(oky1 ? y1 : y0) * Wc + (okx1 ? x1 : x0)) * C4;
  const float4* d = reinterpret_cast<const float4*>(dino + ((size_t)b * h * w + p) * C);
  float4* o = reinterpret_cast<float4*>(refined + ((size_t)b * h * w + p) * C);
  for (int i = threadIdx.x; i < C4; i += blockDim.x) {
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 v = __ldg(pnw + i);
    acc.x = fmaf(v.x, wnw, acc.x); acc.y = fmaf(v.y, wnw, acc.y); acc.z = fmaf(v.z, wnw, acc.z); acc.w = fmaf(v.w, wnw, acc.w);
    if (okx1) { v = __ldg(pne + i); acc.x = fmaf(v.x, wne, acc.x); acc.y = fmaf(v.y, wne, acc.y); acc.z = fmaf(v.z, wne, acc.z); acc.w = fmaf(v.w, wne, acc.w); }
    if (oky1) { v = __ldg(psw + i); acc.x = fmaf(v.x, wsw, acc.x); acc.y = fmaf(v.y, wsw, acc.y); acc.z = fmaf(v.z, wsw, acc.z); acc.w = fmaf(v.w, wsw, acc.w); }
    if (okx1 && oky1) { v = __ldg(pse + i); acc.x = fmaf(v.x, wse, acc.x); acc.y = fmaf(v.y, wse, acc.y); acc.z = fmaf(v.z, wse, acc.z); acc.w = fmaf(v.w, wse, acc.w); }
    float4 dv = __ldg(d + i);
    const float4 val = make_float4(dv.x + acc.x, dv.y + acc.y, dv.z + acc.z, dv.w + acc.w);
    o[i] = val;
    for (int k = 0; k < peers.n; ++k)
      reinterpret_cast<float4*>(peers.base[k] + (peers.row_offset + (size_t)b * h * w + p) * C)[i] = val;
  }
}


// ---- tensor-core path: explicit im2col (fp16 hi/lo split on the fly) + wgmma split-precision GEMM --------------------
// A[m][k] = in[b][reflect(y + (ky-2) d)][reflect(x + (kx-2) d)][ci],  k = (ky*5 + kx)*Cin + ci, zero padded to Kp
__global__ void im2col_split_kernel(const float* __restrict__ in, __half* __restrict__ hi, __half* __restrict__ lo,
                                    int H, int W, int Cin, int dil, int Kp, size_t m0, size_t m_count) {
  const size_t m = m0 + blockIdx.x;          // pixel index within the batch (b*H*W + y*W + x)
  if (blockIdx.x >= m_count) return;
  const int HW = H * W;
  const int b = (int)(m / HW), rem = (int)(m - (size_t)b * HW);
  const int y = rem / W, x = rem - y * W;
  const int K = 25 * Cin;
  __half* oh = hi + (size_t)blockIdx.x * Kp;
  __half* ol = lo + (size_t)blockIdx.x * Kp;
  for (int k4 = threadIdx.x * 4; k4 < Kp; k4 += blockDim.x * 4) {
    float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
    if (k4 < K) {
      const int tap = k4 / Cin, ci = k4 - tap * Cin;   // Cin % 4 == 0: the 4 elements share the tap
      const int ky = tap / 5, kx = tap - ky * 5;
      const int sy = reflect(y + (ky - 2) * dil, H), sx = reflect(x + (kx - 2) * dil, W);
      v = __ldg(reinterpret_cast<const float4*>(in + (((size_t)b * H + sy) * W + sx) * Cin + ci));
    }
    __half h0 = __float2half_rn(v.x), h1 = __float2half_rn(v.y), h2 = __float2half_rn(v.z), h3 = __float2half_rn(v.w);
    __half l0 = __float2half_rn(v.x - __half2float(h0)), l1 = __float2half_rn(v.y - __half2float(h1));
    __half l2 = __float2half_rn(v.z - __half2float(h2)), l3 = __float2half_rn(v.w - __half2float(h3));
    __half2 a = __halves2half2(h0, h1), c = __halves2half2(h2, h3), d = __halves2half2(l0, l1), e = __halves2half2(l2, l3);
    *reinterpret_cast<uint2*>(oh + k4) = make_uint2(*reinterpret_cast<unsigned*>(&a), *reinterpret_cast<unsigned*>(&c));
    *reinterpret_cast<uint2*>(ol + k4) = make_uint2(*reinterpret_cast<unsigned*>(&d), *reinterpret_cast<unsigned*>(&e));
  }
}

// out[m0 + r][col] = relu?(acc + bias[col])   (NHWC fp32)
struct EpiConv {
  float* out; const float* bias; int Cout, relu; size_t m0;
  struct State {};
  __device__ __forceinline__ void tile_begin(State&) const {}
  __device__ __forceinline__ void tile_end(State&, int, int, int) const {}
  __device__ __forceinline__ void operator()(State&, int, int r, int col0, const float (&f)[32], int ncols) const {
    float* o = out + (m0 + r) * Cout + col0;
#pragma unroll
    for (int i = 0; i < 32; i += 4)
      if (i < ncols) {   // Cout % 8 == 0 -> ncols % 4 == 0
        const float4 bb = __ldg(reinterpret_cast<const float4*>(bias + col0 + i));
        float4 v = make_float4(f[i] + bb.x, f[i + 1] + bb.y, f[i + 2] + bb.z, f[i + 3] + bb.w);
        if (relu) { v.x = fmaxf(v.x, 0.f); v.y = fmaxf(v.y, 0.f); v.z = fmaxf(v.z, 0.f); v.w = fmaxf(v.w, 0.f); }
        *reinterpret_cast<float4*>(o + i) = v;
      }
  }
};

size_t delta_conv_kmax(const int* channels) {
  size_t kmax = 0;
  for (int l = 0; l < 4; ++l) { size_t k = align_up((size_t)25 * (l == 0 ? 4 : channels[l]), 8); if (k > kmax) kmax = k; }
  return kmax;
}

int launch_rgb_to_nhwc4(const float* frames, float* out, int B, int HW, cudaStream_t st) {
  const size_t n = (size_t)B * HW;
  rgb_to_nhwc4_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(frames, out, B, HW);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// one conv layer on tensor cores, row chunks of CONV_TC_ROWS output pixels
int launch_conv_tc(const float* in, const __half* w_hi, const __half* w_lo, const float* bias, float* out,
                   ConvShape cs, int Kp, __half* col_hi, __half* col_lo, int* plan, cudaStream_t st, int prof) {
  const size_t M = (size_t)cs.B * cs.H * cs.W;
  const TcPlan pl{plan, plan + 4, plan + 8, plan + 12};
  for (size_t m0 = 0; m0 < M; m0 += CONV_TC_ROWS) {
    const size_t rows = M - m0 < CONV_TC_ROWS ? M - m0 : CONV_TC_ROWS;
    int rc;
    {
      ProfRange pr(prof, st);
      im2col_split_kernel<<<(unsigned)rows, 128, 0, st>>>(in, col_hi, col_lo, cs.H, cs.W, cs.Cin, cs.dil, Kp, m0, rows);
      DTK_LAUNCHED();
      if ((rc = launch_tc_plan(pl, 1, (int)rows, 0, 0, 0, TC_BM, st))) return rc;
    }
    EpiConv epi{out, bias, cs.Cout, cs.relu, m0};
    if ((rc = tc_launch_bn<TcMode::F16X3>({col_hi, col_lo, rows, 0, w_hi, w_lo, 1, 0}, pl.problem(1, cs.Cout, Kp),
                                          cdiv((int)rows, TC_BM), epi, st, prof)))
      return rc;
  }
  return DINOTRK_OK;
}

static int launch_conv(const float* in, const float* wgt, const float* bias, float* out, ConvShape cs, cudaStream_t st) {
  static PerDev<bool> attr_dev;
  bool& attr = attr_dev.get();
  if (!attr) {
    DTK_CUDA(cudaFuncSetAttribute(conv5x5_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, CONV_SMEM));
    attr = true;
  }
  dim3 grid(cdiv(cs.B * cs.H * cs.W, CBM), cdiv(cs.Cout, CBN));
  ProfRange pr(PROF_CONV, st);
  conv5x5_kernel<<<grid, CONV_THREADS, CONV_SMEM, st>>>(in, wgt, bias, out, cs);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // namespace dtk

using namespace dtk;

extern "C" {

static size_t delta_max_activation(int B, int H, int W, const int* channels) {
  // largest NHWC activation over the stack (input padded to 4 channels, conv outputs, blur outputs)
  size_t best = (size_t)B * H * W * 4;
  int ch = H, cw = W;
  for (int l = 0; l < 4; ++l) {
    size_t a = (size_t)B * ch * cw * channels[l + 1];
    if (a > best) best = a;
    if (l < 3) { ch = (ch - 1) / 2 + 1; cw = (cw - 1) / 2 + 1; }
  }
  return best;
}

// two activation buffers; the tensor-core path adds its fp16 im2col scratch and tile plan
struct DeltaWs {
  float* buf0; float* buf1; __half* col_hi = nullptr; __half* col_lo = nullptr; int* cplan = nullptr;
  DeltaWs(Arena& ar, int B, int H, int W, const int* channels, bool tensor) {
    const size_t half = delta_max_activation(B, H, W, channels);
    buf0 = ar.take<float>(half);
    buf1 = ar.take<float>(half);
    if (tensor) {
      const size_t kmax = delta_conv_kmax(channels);
      col_hi = ar.take<__half>(CONV_TC_ROWS * kmax);
      col_lo = ar.take<__half>(CONV_TC_ROWS * kmax);
      cplan = ar.take<int>(16);
    }
  }
};

size_t dinotrk_delta_workspace_bytes(int B, int H, int W, const int* channels) {
  return align_up(layout_end<DeltaWs>(B, H, W, channels, true), 256) + 7936;
}

static int delta_refine_impl(const float* frames, int B, int H, int W, const int* channels, const float* const* wgt,
                             const float* const* bias, const float* dino_tpc, const float* ixs, const float* iys,
                             int h, int w, float* refined_tpc, float* norms, void* workspace, size_t workspace_bytes,
                             const PeerOut& peers, void* stream, const void* const* wgt_hi = nullptr,
                             const void* const* wgt_lo = nullptr) {
  DTK_CHECK_ARG(frames && channels && (wgt || (wgt_hi && wgt_lo)) && bias && dino_tpc && ixs && iys && refined_tpc,
                "delta_refine: null pointer");
  if (wgt_hi && wgt_lo)
    for (int l = 1; l <= 4; ++l) DTK_CHECK_ARG(channels[l] % 8 == 0, "delta_refine (tensor path): channel counts must be multiples of 8");
  DTK_CHECK_ARG(channels[0] == 3, "delta_refine: input must be RGB");
  for (int l = 1; l <= 4; ++l) DTK_CHECK_ARG(channels[l] % 4 == 0, "delta_refine: channel counts must be multiples of 4");
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_delta_workspace_bytes(B, H, W, channels),
                "delta_refine: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const bool tensor = wgt_hi != nullptr && wgt_lo != nullptr;
  Arena ar(workspace);
  const DeltaWs ws(ar, B, H, W, channels, tensor);

  {
    ProfRange pr(PROF_MISC, st);
    if (int rc = launch_rgb_to_nhwc4(frames, ws.buf0, B, H * W, st)) return rc;
  }
  int ch = H, cw = W, cin = 4;
  float* cur = ws.buf0;
  float* oth = ws.buf1;
  const int dil[4] = {1, 1, 1, 2};
  for (int l = 0; l < 4; ++l) {
    ConvShape cs{B, ch, cw, cin, channels[l + 1], dil[l], l < 3 ? 1 : 0};
    int rc = tensor ? launch_conv_tc(cur, (const __half*)wgt_hi[l], (const __half*)wgt_lo[l], bias[l], oth, cs,
                                     (int)align_up((size_t)25 * cin, 8), ws.col_hi, ws.col_lo, ws.cplan, st)
                    : launch_conv(cur, wgt[l], bias[l], oth, cs, st);
    if (rc) return rc;
    std::swap(cur, oth);
    cin = channels[l + 1];
    if (l < 3) {
      int ho = (ch - 1) / 2 + 1, wo = (cw - 1) / 2 + 1;
      size_t tot = (size_t)B * ho * wo * (cin / 4);
      {
        ProfRange pr(PROF_BLUR, st);
        blurpool_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(cur, oth, B, ch, cw, cin, ho, wo);
        DTK_LAUNCHED();
      }
      std::swap(cur, oth);
      ch = ho; cw = wo;
    }
  }
  {
    ProfRange pr(PROF_ALIGN, st);
    align_add_kernel<<<dim3(h * w, B), 128, 0, st>>>(cur, dino_tpc, refined_tpc, ixs, iys, ch, cw, cin, h, w, peers);
    DTK_LAUNCHED();
  }
  if (norms) return dinotrk_token_norms(refined_tpc, norms, B, cin, h * w, stream);
  return DINOTRK_OK;
}

int dinotrk_delta_refine(const float* frames, int B, int H, int W, const int* channels, const float* const* wgt,
                         const float* const* bias, const float* dino_tpc, const float* ixs, const float* iys,
                         int h, int w, float* refined_tpc, float* norms, void* workspace, size_t workspace_bytes,
                         void* stream) {
  NvtxRange nvtx_range("dinotrk.delta_refine");
  PeerOut none{};
  return delta_refine_impl(frames, B, H, W, channels, wgt, bias, dino_tpc, ixs, iys, h, w, refined_tpc, norms, workspace,
                           workspace_bytes, none, stream);
}

int dinotrk_delta_refine_tc(const float* frames, int B, int H, int W, const int* channels, const void* const* wgt_hi,
                            const void* const* wgt_lo, const float* const* bias, const float* dino_tpc, const float* ixs,
                            const float* iys, int h, int w, float* refined_tpc, float* norms, void* workspace,
                            size_t workspace_bytes, float* const* peer_bases, int n_peers, size_t first_frame,
                            void* stream) {
  NvtxRange nvtx_range("dinotrk.delta_refine");
  DTK_CHECK_ARG(n_peers >= 0 && n_peers <= 8 && (n_peers == 0 || peer_bases), "delta_refine_tc: bad peer list");
  PeerOut po{};
  po.n = n_peers;
  for (int k = 0; k < n_peers; ++k) po.base[k] = peer_bases[k];
  po.row_offset = first_frame * (size_t)h * w;
  return delta_refine_impl(frames, B, H, W, channels, nullptr, bias, dino_tpc, ixs, iys, h, w, refined_tpc, norms, workspace,
                           workspace_bytes, po, stream, wgt_hi, wgt_lo);
}

int dinotrk_delta_refine_allgather(const float* frames, int B, int H, int W, const int* channels, const float* const* wgt,
                                   const float* const* bias, const float* dino_tpc, const float* ixs, const float* iys,
                                   int h, int w, float* refined_tpc, float* norms, void* workspace,
                                   size_t workspace_bytes, float* const* peer_bases, int n_peers, size_t first_frame,
                                   void* stream) {
  NvtxRange nvtx_range("dinotrk.delta_refine");
  DTK_CHECK_ARG(n_peers >= 0 && n_peers <= 8 && (n_peers == 0 || peer_bases), "delta_refine_allgather: bad peer list");
  PeerOut po{};
  po.n = n_peers;
  for (int k = 0; k < n_peers; ++k) po.base[k] = peer_bases[k];
  po.row_offset = first_frame * (size_t)h * w;
  return delta_refine_impl(frames, B, H, W, channels, wgt, bias, dino_tpc, ixs, iys, h, w, refined_tpc, norms, workspace,
                           workspace_bytes, po, stream);
}

// ---- peer-mapped buffers (one process per GPU on one node): cudaMalloc + CUDA IPC --------------------------------
int dinotrk_peer_alloc(size_t bytes, void** ptr, unsigned char* handle64) {
  DTK_CHECK_ARG(ptr && handle64 && bytes > 0, "peer_alloc: bad args");
  DTK_CUDA(cudaMalloc(ptr, bytes));
  cudaIpcMemHandle_t hdl;
  DTK_CUDA(cudaIpcGetMemHandle(&hdl, *ptr));
  static_assert(sizeof(hdl) == 64, "cudaIpcMemHandle_t is 64 bytes");
  memcpy(handle64, &hdl, 64);
  return DINOTRK_OK;
}
int dinotrk_peer_open(const unsigned char* handle64, void** ptr) {
  DTK_CHECK_ARG(ptr && handle64, "peer_open: bad args");
  cudaIpcMemHandle_t hdl;
  memcpy(&hdl, handle64, 64);
  DTK_CUDA(cudaIpcOpenMemHandle(ptr, hdl, cudaIpcMemLazyEnablePeerAccess));
  return DINOTRK_OK;
}
int dinotrk_peer_close(void* ptr) { DTK_CUDA(cudaIpcCloseMemHandle(ptr)); return DINOTRK_OK; }
int dinotrk_peer_free(void* ptr) { DTK_CUDA(cudaFree(ptr)); return DINOTRK_OK; }

}  // extern "C"

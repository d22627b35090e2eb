// Training backward of the tracker forward (SURVEY.md 8f-4): the gradient of
//     coords = TrackerHead(relu(corr(sample(E, points), E[target])))          models/tracker.py:170-180, 303-325
// with respect to the frame embeddings E (the frame set's refined features, which carry delta-DINO's graph in
// dino_tracker.py:405-429) and to the refiner's (normalised) weights.  The forward of a training step is the inference
// forward with the maps kept (dinotrk_sample_descriptors + dinotrk_corr_maps + dinotrk_head with aux); this file is the
// reverse pass, three kernels:
//   1. track_head_bwd_kernel  one block per map, the whole map in shared memory (in a workspace slice in global memory on
//                             grids whose five map buffers do not fit, P > 11,560 tokens): refiner recomputed channel by channel,
//                             softmax / disc soft-argmax (tracker_head.py:68-105, both branches), then d/dlogits,
//                             conv2^T, ReLU', conv1^T -> d/dmap, and the weight gradients (block reductions + atomics).
//   2. track_corr_bwd_kernel  one block per map (token list in shared memory, or in the workspace beyond 19,366 tokens):
//                             cosine-correlation backward (tracker.py:158-169) on the tokens that
//                             carry gradient -> d/ddescriptor and atomic adds into d/dE[target frame].
//   3. track_sample_bwd_kernel one block per point: the trilinear sampling weights of the forward (utils.py:75-101,
//                             including the fp32 temporal leak) scatter d/ddescriptor into d/dE.
// arg-max and the disc mask are piecewise constant (no gradient), as in autograd.  For a map that did not take the
// stability branch the term  sum_k p_k dL/dp_k  of the softmax backward is exactly 0 (soft-argmax is a ratio of sums
// over the disc), so its d/dlogits vanishes outside the disc and everything upstream is local to a 15 x 15 window; autograd
// carries rounding noise ~1e-9 there instead.  Maps on the stability branch take the same kernels on the full map.
#include <math.h>

#include "common.cuh"
#include "head.cuh"
#include "sample.cuh"

namespace dtk {

constexpr int TB_THREADS = 512;
constexpr int TB_WARPS = TB_THREADS / 32;
constexpr int TB_NRED = 19;          // per hidden channel: dw2[9], dw1[9], db1

__device__ __forceinline__ float block_reduce(float v, float* red, bool is_max) {
  v = is_max ? warp_max(v) : warp_sum(v);
  __syncthreads();
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
  __syncthreads();
  float r = red[0];
  for (int k = 1; k < TB_WARPS; ++k) r = is_max ? fmaxf(r, red[k]) : r + red[k];
  return r;
}

// cross-correlation with zero padding: sum_k wk[k] * src[(r + ky - 1) * w + c + kx - 1]
__device__ __forceinline__ float conv3(const float* __restrict__ src, int r, int c, int h, int w, const float* wk) {
  float a = 0.f;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int rr = r + ky - 1;
    if (rr < 0 || rr >= h) continue;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int cc = c + kx - 1;
      if (cc >= 0 && cc < w) a = fmaf(wk[ky * 3 + kx], src[rr * w + cc], a);
    }
  }
  return a;
}
// its transpose: sum_k wk[k] * src[(r - ky + 1) * w + c - kx + 1]
__device__ __forceinline__ float conv3t(const float* __restrict__ src, int r, int c, int h, int w, const float* wk) {
  float a = 0.f;
#pragma unroll
  for (int ky = 0; ky < 3; ++ky) {
    const int rr = r - ky + 1;
    if (rr < 0 || rr >= h) continue;
#pragma unroll
    for (int kx = 0; kx < 3; ++kx) {
      const int cc = c - kx + 1;
      if (cc >= 0 && cc < w) a = fmaf(wk[ky * 3 + kx], src[rr * w + cc], a);
    }
  }
  return a;
}

// kGlobal: the five map buffers of block b are gbuf[b * 5 P ...] in global memory (grids whose 5 P floats exceed shared
// memory); shared memory then holds the reduction slots only.  Same arithmetic either way.
template <bool kGlobal>
__global__ void __launch_bounds__(TB_THREADS, 1)
track_head_bwd_kernel(const float* __restrict__ maps, const int* __restrict__ aux, const float* __restrict__ grad_out,
                      HeadParams hp, dinotrk_head_weights wts, float* __restrict__ dcorr, float* __restrict__ grad_w,
                      float* __restrict__ gbuf) {
  extern __shared__ __align__(16) float tb_smem[];
  const int P = hp.P, h = hp.h, w = hp.w;
  const int b = blockIdx.x, tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  float* m = kGlobal ? gbuf + (size_t)b * 5 * P : tb_smem;   // relu(corr)
  float* z = m + P;              // logits, then d/dlogits
  float* ho = z + P;             // hidden channel o
  float* dho = ho + P;           // its gradient
  float* dm = dho + P;           // d/dmap
  float* red = kGlobal ? tb_smem : dm + P;   // [TB_WARPS * TB_NRED]
  __shared__ float sc[8];        // px, py, s', count, dot
  const float* mp = maps + (size_t)b * hp.map_stride;
  const int amax = aux[2 * b], fb = aux[2 * b + 1];
  const int arow = amax / w, acol = amax - arow * w;

  for (int p = tid; p < P; p += TB_THREADS) { m[p] = mp[p]; z[p] = wts.b2; dm[p] = 0.f; dho[p] = 0.f; }
  __syncthreads();
  // ---- logits of the whole map (the softmax denominator needs them all) ----
  for (int o = 0; o < 16; ++o) {
    for (int p = tid; p < P; p += TB_THREADS) {
      const int r = p / w, c = p - r * w;
      ho[p] = fmaxf(wts.b1[o] + conv3(m, r, c, h, w, wts.w1[o]), 0.f);
    }
    __syncthreads();
    for (int p = tid; p < P; p += TB_THREADS) {
      const int r = p / w, c = p - r * w;
      z[p] += conv3(ho, r, c, h, w, wts.w2[o]);
    }
    __syncthreads();
  }
  float zmax = -INFINITY;
  for (int p = tid; p < P; p += TB_THREADS) zmax = fmaxf(zmax, z[p]);
  zmax = block_reduce(zmax, red, true);
  float se = 0.f;
  for (int p = tid; p < P; p += TB_THREADS) se += expf(z[p] - zmax);
  se = block_reduce(se, red, false);
  const float inv_se = 1.f / se;
  // ---- soft-argmax on the disc (warp 0; the disc lies inside the 11 x 11 box around the arg-max) ----
  if (wid == 0) {
    float cnt = 0.f, s = 0.f;
    for (int q = lane; q < WB * WB; q += 32) {
      const int r = arow - HEAD_BOX_R + q / WB, c = acol - HEAD_BOX_R + q % WB;
      if (r >= 0 && r < h && c >= 0 && c < w && in_disc(hp, r, c, arow, acol)) {
        cnt += 1.f;
        s += expf(z[r * w + c] - zmax) * inv_se;
      }
    }
    cnt = warp_sum(cnt); s = warp_sum(s);
    const float uni = fb ? 1.f / cnt : 0.f;
    float s2 = 0.f, sx = 0.f, sy = 0.f;
    for (int q = lane; q < WB * WB; q += 32) {
      const int r = arow - HEAD_BOX_R + q / WB, c = acol - HEAD_BOX_R + q % WB;
      if (r >= 0 && r < h && c >= 0 && c < w && in_disc(hp, r, c, arow, acol)) {
        const float qv = expf(z[r * w + c] - zmax) * inv_se + uni;
        s2 += qv;
        sx = fmaf(token_px(hp, c), qv, sx);
        sy = fmaf(token_px(hp, r), qv, sy);
      }
    }
    s2 = warp_sum(s2); sx = warp_sum(sx); sy = warp_sum(sy);
    const float px = sx / s2, py = sy / s2;
    // out = 2 * point / (W - 1, H - 1) - 1
    const float dpx = grad_out[2 * b] * 2.f / hp.normW, dpy = grad_out[2 * b + 1] * 2.f / hp.normH;
    float dot = 0.f;
    if (fb) {
      for (int q = lane; q < WB * WB; q += 32) {
        const int r = arow - HEAD_BOX_R + q / WB, c = acol - HEAD_BOX_R + q % WB;
        if (r >= 0 && r < h && c >= 0 && c < w && in_disc(hp, r, c, arow, acol)) {
          const float dq = ((token_px(hp, c) - px) * dpx + (token_px(hp, r) - py) * dpy) / s2;
          dot = fmaf(expf(z[r * w + c] - zmax) * inv_se, dq, dot);
        }
      }
      dot = warp_sum(dot);
    }
    if (lane == 0) { sc[0] = px; sc[1] = py; sc[2] = s2; sc[3] = dot; sc[4] = dpx; sc[5] = dpy; }
  }
  __syncthreads();
  {
    const float px = sc[0], py = sc[1], s2 = sc[2], dot = sc[3], dpx = sc[4], dpy = sc[5];
    float db2 = 0.f;
    for (int p = tid; p < P; p += TB_THREADS) {
      const int r = p / w, c = p - r * w;
      const bool in = in_disc(hp, r, c, arow, acol);
      float g = 0.f;
      if (in || fb) {
        const float pv = expf(z[p] - zmax) * inv_se;
        const float dq = in ? ((token_px(hp, c) - px) * dpx + (token_px(hp, r) - py) * dpy) / s2 : 0.f;
        g = pv * (dq - dot);
      }
      db2 += g;
      ho[p] = g;            // staged: z is still being read by other threads
    }
    __syncthreads();
    for (int p = tid; p < P; p += TB_THREADS) z[p] = ho[p];
    db2 = block_reduce(db2, red, false);
    if (tid == 0) atomicAdd(grad_w + 304, db2);
  }
  __syncthreads();
  // ---- conv2^T, ReLU', conv1^T and the weight gradients; rows that can carry gradient only ----
  const int r_lo = fb ? 0 : max(0, arow - 8), r_hi = fb ? h : min(h, arow + 9);
  const int p_lo = r_lo * w, p_hi = r_hi * w;
  for (int o = 0; o < 16; ++o) {
    float acc[TB_NRED];
#pragma unroll
    for (int k = 0; k < TB_NRED; ++k) acc[k] = 0.f;
    for (int p = p_lo + tid; p < p_hi; p += TB_THREADS) {
      const int r = p / w, c = p - r * w;
      ho[p] = fmaxf(wts.b1[o] + conv3(m, r, c, h, w, wts.w1[o]), 0.f);
    }
    __syncthreads();
    for (int p = p_lo + tid; p < p_hi; p += TB_THREADS) {
      const int r = p / w, c = p - r * w;
      dho[p] = ho[p] > 0.f ? conv3t(z, r, c, h, w, wts.w2[o]) : 0.f;
      const float g = z[p];
      if (g != 0.f) {
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const int rr = r + ky - 1, cc = c + kx - 1;
            if (rr >= r_lo && rr < r_hi && cc >= 0 && cc < w) acc[ky * 3 + kx] = fmaf(g, ho[rr * w + cc], acc[ky * 3 + kx]);
          }
      }
    }
    __syncthreads();
    for (int p = p_lo + tid; p < p_hi; p += TB_THREADS) {
      const int r = p / w, c = p - r * w;
      const float g = dho[p];
      if (g != 0.f) {
        acc[18] += g;
#pragma unroll
        for (int ky = 0; ky < 3; ++ky)
#pragma unroll
          for (int kx = 0; kx < 3; ++kx) {
            const int rr = r + ky - 1, cc = c + kx - 1;
            if (rr >= 0 && rr < h && cc >= 0 && cc < w) acc[9 + ky * 3 + kx] = fmaf(g, m[rr * w + cc], acc[9 + ky * 3 + kx]);
          }
      }
      dm[p] += conv3t(dho, r, c, h, w, wts.w1[o]);
    }
#pragma unroll
    for (int k = 0; k < TB_NRED; ++k) {
      const float v = warp_sum(acc[k]);
      if (lane == 0) red[wid * TB_NRED + k] = v;
    }
    __syncthreads();
    if (tid < TB_NRED) {
      float v = 0.f;
      for (int k = 0; k < TB_WARPS; ++k) v += red[k * TB_NRED + tid];
      // grad_w layout: w1[16][9] | b1[16] | w2[16][9] | b2
      float* dst = tid < 9 ? grad_w + 160 + o * 9 + tid : tid < 18 ? grad_w + o * 9 + (tid - 9) : grad_w + 144 + o;
      if (v != 0.f) atomicAdd(dst, v);
    }
    __syncthreads();
  }
  // ---- through the ReLU of the correlation map ----
  float* dc = dcorr + (size_t)b * hp.map_stride;
  for (int p = tid; p < P; p += TB_THREADS) dc[p] = m[p] > 0.f ? dm[p] : 0.f;
}

// corr = <s, F> / max(|s| |F|, 1e-8):  d/ds = g (F / D - corr s / |s|^2),  d/dF = g (s / D - corr F / |F|^2)  (the
// second terms only where the clamp is inactive).  The map holds relu(corr); where it is 0 the incoming gradient is 0 too.
// kGlobal: the token list of block b is gbuf[b * 3 P ...] in global memory (grids whose 3 P words exceed shared memory).
constexpr int TC_THREADS_BWD = 256;
template <bool kGlobal>
__global__ void __launch_bounds__(TC_THREADS_BWD)
track_corr_bwd_kernel(const float* __restrict__ tpc, const float* __restrict__ norms, int C, int P, int map_stride,
                      const float* __restrict__ maps, const float* __restrict__ dcorr, const float* __restrict__ desc,
                      const float* __restrict__ desc_norm, const int* __restrict__ tgt_frame, float* __restrict__ ddesc,
                      float* __restrict__ grad_tpc, float* __restrict__ gbuf) {
  extern __shared__ __align__(16) float tcb_smem[];
  const int b = blockIdx.x, tid = threadIdx.x;
  float* lbuf = kGlobal ? gbuf + (size_t)b * 3 * P : tcb_smem;
  int* l_tok = reinterpret_cast<int*>(lbuf);           // [P]
  float* l_a = lbuf + P;                                // g / D
  float* l_b = l_a + P;                                 // g corr / |F|^2 (0 under the clamp)
  __shared__ int n_list;
  __shared__ float red[TC_THREADS_BWD / 32];
  const int f = tgt_frame[b];
  const float sn = desc_norm[b];
  const float* fn = norms + (size_t)f * P;
  const float* mp = maps + (size_t)b * map_stride;
  const float* gp = dcorr + (size_t)b * map_stride;
  if (tid == 0) n_list = 0;
  __syncthreads();
  float sgc = 0.f;
  for (int p = tid; p < P; p += TC_THREADS_BWD) {
    const float g = gp[p];
    if (g != 0.f) {
      const float nf = fn[p], prod = sn * nf;
      const bool clamped = !(prod > 1e-8f);
      const float D = clamped ? 1e-8f : prod;
      const float corr = mp[p];
      const int i = atomicAdd(&n_list, 1);
      l_tok[i] = p;
      l_a[i] = g / D;
      l_b[i] = clamped ? 0.f : g * corr / (nf * nf);
      if (!clamped) sgc = fmaf(g, corr, sgc);
    }
  }
  sgc = warp_sum(sgc);
  if ((tid & 31) == 0) red[tid >> 5] = sgc;
  __syncthreads();
  sgc = 0.f;
  for (int k = 0; k < TC_THREADS_BWD / 32; ++k) sgc += red[k];
  const int n = n_list;
  const float self = sn > 0.f ? sgc / (sn * sn) : 0.f;
  const float* frow = tpc + (size_t)f * P * C;
  float* grow = grad_tpc ? grad_tpc + (size_t)f * P * C : nullptr;
  for (int c = tid; c < C; c += TC_THREADS_BWD) {
    const float sc_ = desc[(size_t)b * C + c];
    float acc = 0.f;
    for (int i = 0; i < n; ++i) {
      const size_t off = (size_t)l_tok[i] * C + c;
      const float F = __ldg(frow + off);
      acc = fmaf(l_a[i], F, acc);
      if (grow) atomicAdd(grow + off, l_a[i] * sc_ - l_b[i] * F);
    }
    ddesc[(size_t)b * C + c] = acc - self * sc_;
  }
}

__global__ void __launch_bounds__(SAMPLE_THREADS)
track_sample_bwd_kernel(int C, int P, int h, int w, PointAffine pa, const float* __restrict__ points,
                        const int* __restrict__ frames_set, int N, int normalized, const float* __restrict__ ddesc,
                        float* __restrict__ grad_tpc) {
  const int b = blockIdx.x;
  float x = points[b * 3 + 0], y = points[b * 3 + 1];
  if (!normalized) {
    x = __fadd_rn(__fmul_rn(pa.aw, x), pa.bw);
    y = __fadd_rn(__fmul_rn(pa.ah, y), pa.bh);
  }
  const TriCorners c = tri_setup(x, y, points[b * 3 + 2], N, h, w);
  const int fr[2] = {frames_set[c.z0], c.z1 >= 0 ? frames_set[c.z1] : -1};
#pragma unroll
  for (int zz = 0; zz < 2; ++zz)
#pragma unroll
    for (int k = 0; k < 4; ++k) {
      const float wt = c.wxy[k][zz];
      if (fr[zz] < 0 || c.tok[k] < 0 || wt == 0.f) continue;
      float* dst = grad_tpc + ((size_t)fr[zz] * P + c.tok[k]) * C;
      for (int i = threadIdx.x; i < C; i += SAMPLE_THREADS) atomicAdd(dst + i, wt * ddesc[(size_t)b * C + i]);
    }
}

}  // namespace dtk

using namespace dtk;

extern "C" {

// shared memory of the map buffers of the two per-map kernels; above the limit they live in the workspace instead
static size_t head_bwd_smem(int P) { return ((size_t)5 * P + TB_WARPS * TB_NRED) * sizeof(float); }
static size_t corr_bwd_smem(int P) { return (size_t)3 * P * sizeof(float); }
// The shared-memory variant runs when its dynamic buffers plus the kernel's static shared memory fit the per-block opt-in
// limit (227 KiB on sm_90: P <= 11,560 for the head kernel, P <= 19,366 for the correlation kernel).  A failed query
// counts as "does not fit": the workspace variant runs on every grid.
static bool bwd_smem_fits(const void* kernel, size_t dyn) {
  int dev = 0, optin = 0;
  cudaFuncAttributes fa{};
  if (cudaGetDevice(&dev) != cudaSuccess || cudaDeviceGetAttribute(&optin, cudaDevAttrMaxSharedMemoryPerBlockOptin, dev) != cudaSuccess ||
      cudaFuncGetAttributes(&fa, kernel) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return dyn + fa.sharedSizeBytes <= (size_t)optin;
}
static bool head_bwd_global(int P) { return !bwd_smem_fits((const void*)track_head_bwd_kernel<false>, head_bwd_smem(P)); }
static bool corr_bwd_global(int P) { return !bwd_smem_fits((const void*)track_corr_bwd_kernel<false>, corr_bwd_smem(P)); }

// the gradients of the maps and descriptors; the map buffers of a per-map kernel whose shared-memory variant does not fit
struct TrackBwdWs {
  float* dcorr; float* ddesc; bool g1, g2; float* gbuf1 = nullptr; float* gbuf2 = nullptr;
  TrackBwdWs(Arena& ar, int B, int C, const dinotrk_geom& g) {
    const int P = g.h * g.w;
    dcorr = ar.take<float>((size_t)B * dinotrk_map_stride(&g));
    ddesc = ar.take<float>((size_t)B * C);
    g1 = head_bwd_global(P);
    g2 = corr_bwd_global(P);
    if (g1) gbuf1 = ar.take<float>((size_t)B * 5 * P);
    if (g2) gbuf2 = ar.take<float>((size_t)B * 3 * P);
  }
};

size_t dinotrk_track_backward_workspace_bytes(int B, int C, const dinotrk_geom* g) {
  if (!g || B <= 0) return 0;
  return align_up(layout_end<TrackBwdWs>(B, C, *g), 256) + 1024;
}

int dinotrk_track_backward(const dinotrk_features* feat, const dinotrk_geom* g, const dinotrk_head_weights* hw,
                           const float* points, const int* frames_set, int N, const float* desc, const float* desc_norm,
                           const int* tgt_frame, const float* maps, const int* aux, const float* grad_out, int B,
                           float* grad_w, float* grad_tpc, void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(feat && feat->tpc && feat->norms && g && hw && points && frames_set && desc && desc_norm && tgt_frame && maps &&
                    aux && grad_out && grad_w && workspace,
                "track_backward: null pointer");
  DTK_CHECK_ARG(B >= 0 && N > 0 && feat->C > 0, "track_backward: bad sizes");
  DTK_CHECK_GRID(*g, "track_backward");
  DTK_CHECK_ARG(disc_fits_box(*g), "track_backward: disc radius %d exceeds 5 tokens", g->radius);
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_track_backward_workspace_bytes(B, feat->C, g), "track_backward: workspace too small");
  if (B == 0) return DINOTRK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int P = g->h * g->w, C = feat->C;
  Arena ar(workspace);
  const TrackBwdWs ws(ar, B, C, *g);
  float *dcorr = ws.dcorr, *ddesc = ws.ddesc, *gbuf1 = ws.gbuf1, *gbuf2 = ws.gbuf2;
  const HeadParams hp = make_head_params(*g, *hw, dinotrk_map_stride(g), 2, 1);
  const bool g1 = ws.g1, g2 = ws.g2;
  const size_t smem1 = g1 ? TB_WARPS * TB_NRED * sizeof(float) : head_bwd_smem(P);
  const size_t smem2 = g2 ? 0 : corr_bwd_smem(P);
  static PerDev<size_t> attr1_dev, attr2_dev;
  if (!g1 && attr1_dev.get() < smem1) {
    DTK_CUDA(cudaFuncSetAttribute(track_head_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem1));
    attr1_dev.get() = smem1;
  }
  if (!g2 && attr2_dev.get() < smem2) {
    DTK_CUDA(cudaFuncSetAttribute(track_corr_bwd_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem2));
    attr2_dev.get() = smem2;
  }
  NvtxRange nv("dinotrk_track_backward");
  ProfRange pr(PROF_TRAIN_BWD, st);
  (g1 ? track_head_bwd_kernel<true> : track_head_bwd_kernel<false>)<<<B, TB_THREADS, smem1, st>>>(maps, aux, grad_out, hp, *hw,
                                                                                              dcorr, grad_w, gbuf1);
  DTK_LAUNCHED();
  (g2 ? track_corr_bwd_kernel<true> : track_corr_bwd_kernel<false>)<<<B, TC_THREADS_BWD, smem2, st>>>(
      feat->tpc, feat->norms, C, P, hp.map_stride, maps, dcorr, desc, desc_norm, tgt_frame, ddesc, grad_tpc, gbuf2);
  DTK_LAUNCHED();
  if (grad_tpc) {
    track_sample_bwd_kernel<<<B, SAMPLE_THREADS, 0, st>>>(C, P, g->h, g->w, make_point_affine(*g), points, frames_set, N, 0, ddesc, grad_tpc);
    DTK_LAUNCHED();
  }
  return DINOTRK_OK;
}

int dinotrk_sample_backward(int T, int C, const dinotrk_geom* g, const float* points, int B, const int* frames_set, int N,
                            int points_normalized, const float* grad_desc, float* grad_tpc, void* stream) {
  DTK_CHECK_ARG(g && points && frames_set && grad_desc && grad_tpc, "sample_backward: null pointer");
  DTK_CHECK_ARG(T > 0 && C > 0 && N > 0 && B >= 0, "sample_backward: bad sizes");
  if (B == 0) return DINOTRK_OK;
  ProfRange pr(PROF_TRAIN_BWD, (cudaStream_t)stream);
  track_sample_bwd_kernel<<<B, SAMPLE_THREADS, 0, (cudaStream_t)stream>>>(C, g->h * g->w, g->h, g->w, make_point_affine(*g), points,
                                                                        frames_set, N, points_normalized, grad_desc, grad_tpc);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // extern "C"

// The embedding regularisers of the training step (dino_tracker.py:136-146, models/utils.py:79-84) as one node.
//
// For the frame set's refined embeddings E and raw DINO embeddings R, token-major [n][P][C], and per token p
// a = |E_p|, b = |R_p|, d = E_p . R_p:
//   norm_reg  = mean_p |a / b - 1|          angle_reg = mean_p |d / (a b) - 1|
// The forward reads E and R once (one warp per token, float4 over C), keeps (a, b, d) per token for the backward and
// reduces the two sums through fixed per-block partials and one fixed-order final sum, so two runs give the same bits.
// The backward reads E, R and (a, b, d) and writes dE once:
//   dE_p = g_n / (nP) s1 E_p / (a b) + g_a / (nP) s2 (R_p / (a b) - cos_p E_p / a^2),
// s1 = sgn(a / b - 1), s2 = sgn(cos_p - 1) with sgn(0) = 0 (torch's abs backward), the ratios evaluated as the forward
// evaluates them, so a token at |x - 1|'s kink in the forward gets no gradient from that term.
#include "common.cuh"

namespace dtk {

constexpr int EMB_REG_WARPS = 8;          // tokens per block
constexpr int EMB_REG_FINAL_THREADS = 256;

// the two ratios of one token, in the reference's fp32 op order
__device__ __forceinline__ float emb_norm_ratio(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ float emb_cos(float a, float b, float d) { return __fdiv_rn(d, __fmul_rn(a, b)); }
__device__ __forceinline__ float sgn0(float x) { return x > 0.f ? 1.f : (x < 0.f ? -1.f : 0.f); }

// One warp per token: aux[p] = (a, b, d); part[block] = (sum |a/b - 1|, sum |cos - 1|) over the block's tokens in warp
// order.
__global__ void __launch_bounds__(EMB_REG_WARPS * 32)
emb_reg_forward_kernel(const float4* __restrict__ E, const float4* __restrict__ R, int NP, int C4, float* __restrict__ aux,
                       float2* __restrict__ part) {
  __shared__ float2 s_term[EMB_REG_WARPS];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int p = blockIdx.x * EMB_REG_WARPS + warp;
  float2 term = make_float2(0.f, 0.f);
  if (p < NP) {
    const float4* e = E + (size_t)p * C4;
    const float4* r = R + (size_t)p * C4;
    float ee = 0.f, rr = 0.f, er = 0.f;
#pragma unroll 4
    for (int k = lane; k < C4; k += 32) {
      const float4 x = __ldcs(e + k), y = __ldcs(r + k);
      ee = fmaf(x.x, x.x, fmaf(x.y, x.y, fmaf(x.z, x.z, fmaf(x.w, x.w, ee))));
      rr = fmaf(y.x, y.x, fmaf(y.y, y.y, fmaf(y.z, y.z, fmaf(y.w, y.w, rr))));
      er = fmaf(x.x, y.x, fmaf(x.y, y.y, fmaf(x.z, y.z, fmaf(x.w, y.w, er))));
    }
    ee = warp_sum(ee);
    rr = warp_sum(rr);
    er = warp_sum(er);
    const float a = __fsqrt_rn(ee), b = __fsqrt_rn(rr);
    term = make_float2(fabsf(__fsub_rn(emb_norm_ratio(a, b), 1.f)), fabsf(__fsub_rn(emb_cos(a, b, er), 1.f)));
    if (lane == 0) {
      float* o = aux + (size_t)p * 3;
      o[0] = a; o[1] = b; o[2] = er;
    }
  }
  if (lane == 0) s_term[warp] = term;
  __syncthreads();
  if (threadIdx.x == 0) {
    float2 s = s_term[0];
#pragma unroll
    for (int k = 1; k < EMB_REG_WARPS; ++k) s = make_float2(s.x + s_term[k].x, s.y + s_term[k].y);
    part[blockIdx.x] = s;
  }
}

// out = (sum of part.x, sum of part.y) / NP: per thread a strided sum in block order, then a tree, all in double
__global__ void __launch_bounds__(EMB_REG_FINAL_THREADS)
emb_reg_final_kernel(const float2* __restrict__ part, int nb, double inv_np, float* __restrict__ out) {
  __shared__ double s_n[EMB_REG_FINAL_THREADS], s_a[EMB_REG_FINAL_THREADS];
  double n = 0.0, a = 0.0;
  for (int i = threadIdx.x; i < nb; i += EMB_REG_FINAL_THREADS) {
    n += (double)part[i].x;
    a += (double)part[i].y;
  }
  s_n[threadIdx.x] = n;
  s_a[threadIdx.x] = a;
  __syncthreads();
  for (int o = EMB_REG_FINAL_THREADS / 2; o > 0; o >>= 1) {
    if (threadIdx.x < o) {
      s_n[threadIdx.x] += s_n[threadIdx.x + o];
      s_a[threadIdx.x] += s_a[threadIdx.x + o];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    out[0] = (float)(s_n[0] * inv_np);
    out[1] = (float)(s_a[0] * inv_np);
  }
}

// One warp per token: dE_p = cE E_p + cR R_p
__global__ void __launch_bounds__(EMB_REG_WARPS * 32)
emb_reg_backward_kernel(const float4* __restrict__ E, const float4* __restrict__ R, int NP, int C4,
                        const float* __restrict__ aux, const float* __restrict__ g_norm, const float* __restrict__ g_angle,
                        float inv_np, float4* __restrict__ dE) {
  const int lane = threadIdx.x & 31;
  const int p = blockIdx.x * EMB_REG_WARPS + (threadIdx.x >> 5);
  if (p >= NP) return;
  const float a = aux[(size_t)p * 3], b = aux[(size_t)p * 3 + 1], d = aux[(size_t)p * 3 + 2];
  const float ab = __fmul_rn(a, b), cosv = emb_cos(a, b, d);
  const float gn = *g_norm * inv_np * sgn0(__fsub_rn(emb_norm_ratio(a, b), 1.f));
  const float ga = *g_angle * inv_np * sgn0(__fsub_rn(cosv, 1.f));
  const float cE = gn / ab - ga * cosv / (a * a), cR = ga / ab;
  const float4* e = E + (size_t)p * C4;
  const float4* r = R + (size_t)p * C4;
  float4* g = dE + (size_t)p * C4;
#pragma unroll 4
  for (int k = lane; k < C4; k += 32) {
    const float4 x = __ldcs(e + k), y = __ldcs(r + k);
    __stcs(g + k, make_float4(fmaf(cE, x.x, cR * y.x), fmaf(cE, x.y, cR * y.y), fmaf(cE, x.z, cR * y.z),
                              fmaf(cE, x.w, cR * y.w)));
  }
}

struct EmbRegWs {
  float2* part;   // [cdiv(nP, EMB_REG_WARPS)] per-block sums
  EmbRegWs(Arena& ar, int n, int P) { part = ar.take<float2>((size_t)cdiv(n * P, EMB_REG_WARPS)); }
};

static bool emb_reg_shape_ok(int n, int P, int C) {
  return n > 0 && P > 0 && C > 0 && (long long)n * P <= (long long)INT32_MAX - EMB_REG_WARPS;
}

}  // namespace dtk

using namespace dtk;

extern "C" {

size_t dinotrk_emb_reg_workspace_bytes(int n, int P) {
  if (!emb_reg_shape_ok(n, P, 4)) return 0;
  return align_up(layout_end<EmbRegWs>(n, P), 256);
}

int dinotrk_emb_reg_forward(const float* E, const float* R, int n, int P, int C, float* out, float* aux, void* workspace,
                            size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(E && R && out && aux && workspace && emb_reg_shape_ok(n, P, C),
                "emb_reg_forward: bad arguments (n = %d, P = %d, C = %d)", n, P, C);
  DTK_CHECK_ARG(C % 4 == 0, "emb_reg_forward: C = %d is not a multiple of 4", C);
  DTK_CHECK_ARG(((uintptr_t)E & 15) == 0 && ((uintptr_t)R & 15) == 0, "emb_reg_forward: E and R must be 16-byte aligned");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_emb_reg_workspace_bytes(n, P), "emb_reg_forward: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int NP = n * P, nb = cdiv(NP, EMB_REG_WARPS);
  Arena ar(workspace);
  const EmbRegWs ws(ar, n, P);
  ProfRange pr(PROF_EMB_REG, st);
  emb_reg_forward_kernel<<<nb, EMB_REG_WARPS * 32, 0, st>>>((const float4*)E, (const float4*)R, NP, C / 4, aux, ws.part);
  DTK_LAUNCHED();
  emb_reg_final_kernel<<<1, EMB_REG_FINAL_THREADS, 0, st>>>(ws.part, nb, 1.0 / (double)NP, out);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_emb_reg_backward(const float* E, const float* R, int n, int P, int C, const float* aux, const float* g_norm,
                             const float* g_angle, float* dE, void* stream) {
  DTK_CHECK_ARG(E && R && aux && g_norm && g_angle && dE && emb_reg_shape_ok(n, P, C),
                "emb_reg_backward: bad arguments (n = %d, P = %d, C = %d)", n, P, C);
  DTK_CHECK_ARG(C % 4 == 0, "emb_reg_backward: C = %d is not a multiple of 4", C);
  DTK_CHECK_ARG(((uintptr_t)E & 15) == 0 && ((uintptr_t)R & 15) == 0 && ((uintptr_t)dE & 15) == 0,
                "emb_reg_backward: E, R and dE must be 16-byte aligned");
  cudaStream_t st = (cudaStream_t)stream;
  const int NP = n * P;
  ProfRange pr(PROF_EMB_REG, st);
  emb_reg_backward_kernel<<<cdiv(NP, EMB_REG_WARPS), EMB_REG_WARPS * 32, 0, st>>>(
      (const float4*)E, (const float4*)R, NP, C / 4, aux, g_norm, g_angle, (float)(1.0 / (double)NP), (float4*)dE);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // extern "C"

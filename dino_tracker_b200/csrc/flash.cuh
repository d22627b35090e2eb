// Fused attention for the ViT (sm_90a, wgmma):  O = softmax(Q K^T) V  per (frame, head).  Q arrives pre-scaled by
// head_dim^-1/2 * log2(e), so the softmax is exp2(s - max).
//
// One CTA per (frame*head, 128-query tile); 384 threads:
//   warpgroup 0     : TMA producer (Q once; K_j [64 keys][64] and V^T_j [64][64 keys] through a 4-stage ring)
//   warpgroups 1, 2 : 64 query rows each.  Per key tile: S = Q K_j^T (m64n64k16 x 4, both operands from shared memory)
//                     into registers, online softmax on the accumulator fragment (a row lives in the 4 lanes of a quad),
//                     p = exp2(s - m) packed to fp16 pairs that ARE the A fragments of O += P V_j (m64n64k16 x 4, A from
//                     registers, V^T from shared memory).  O and the row sums stay in registers across all key tiles.
// The score matrix (N1 x N1 per head) never leaves the SM.
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"
#include "tc05.cuh"

namespace dtk {

constexpr int FA_BQ = 128, FA_BKV = 64, FA_D = 64, FA_THREADS = 384;
constexpr int FA_KV_STAGES = 4;
constexpr int FA_SQ = FA_BQ * 128;                 // Q tile bytes (128 rows x 64 fp16)
constexpr int FA_SK = FA_BKV * 128;                // K tile bytes
constexpr int FA_SV = FA_D * 128;                  // V^T tile bytes
constexpr int FA_STAGE = FA_SK + FA_SV;
constexpr int FA_SMEM = 1024 + FA_SQ + FA_KV_STAGES * FA_STAGE + 256;

__device__ __forceinline__ float fast_exp2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_half2(float a, float b) {
  __half2 h = __floats2half2_rn(a, b);
  return *reinterpret_cast<uint32_t*>(&h);
}

struct FlashParams {
  int N1;          // tokens per frame (keys = queries)
  int D;           // model dim (output row pitch)
  int heads;
  void* out;       // [B*N1][D] fp32 or fp16; head h writes columns [h*64, h*64+64)
  int out_f16;
};

__global__ void __launch_bounds__(FA_THREADS, 1)
flash_attn_kernel(const __grid_constant__ CUtensorMap tmQ, const __grid_constant__ CUtensorMap tmK,
                  const __grid_constant__ CUtensorMap tmV, FlashParams fp) {
  extern __shared__ uint8_t fa_smem_raw[];
  uint8_t* sQ = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(fa_smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t* sKV = sQ + FA_SQ;                 // stage s: K at sKV + s*FA_STAGE, V^T at + FA_SK
  uint64_t* bars = reinterpret_cast<uint64_t*>(sKV + FA_KV_STAGES * FA_STAGE);
  uint64_t* q_full = bars;                                    // 1
  uint64_t* kv_full = bars + 1;                               // [FA_KV_STAGES]
  uint64_t* kv_empty = kv_full + FA_KV_STAGES;                // [FA_KV_STAGES] (one arrival per consumer warpgroup)

  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, wg = threadIdx.x >> 7, t = threadIdx.x & 127;
  const int bh = blockIdx.y, q0 = blockIdx.x * FA_BQ;
  const int N1 = fp.N1;
  const int n_kv = (N1 + FA_BKV - 1) / FA_BKV;

  if (threadIdx.x == 0) {
    tc::prefetch_tmap(&tmQ); tc::prefetch_tmap(&tmK); tc::prefetch_tmap(&tmV);
    tc::mbar_init(q_full, 1);
    for (int s = 0; s < FA_KV_STAGES; ++s) { tc::mbar_init(&kv_full[s], 1); tc::mbar_init(&kv_empty[s], 2); }
    tc::mbar_fence_init();
  }
  __syncthreads();

  if (wg == 0) {
    if (warp == 0 && tc::elect_one()) {
      tc::mbar_expect_tx(q_full, FA_SQ);
      tc::tma_load_2d(&tmQ, q_full, sQ, 0, bh * N1 + q0);
      int s = 0, ph = 0;
      for (int j = 0; j < n_kv; ++j) {
        tc::mbar_wait(&kv_empty[s], ph ^ 1);
        tc::mbar_expect_tx(&kv_full[s], FA_STAGE);
        uint8_t* st = sKV + s * FA_STAGE;
        tc::tma_load_3d(&tmK, &kv_full[s], st, 0, j * FA_BKV, bh);
        tc::tma_load_3d(&tmV, &kv_full[s], st + FA_SK, j * FA_BKV, 0, bh);
        if (++s == FA_KV_STAGES) { s = 0; ph ^= 1; }
      }
    }
    return;
  }

  // ---------------- consumer warpgroup cw: query rows [64 cw, 64 cw + 64) of the tile ----------------
  const int cw = wg - 1;
  const int fr = (warp & 3) * 16 + (lane >> 2), fc = 2 * (lane & 3);   // fragment rows fr, fr + 8; columns 8 i + fc (+1)
  const uint32_t qa = tc::smem_u32(sQ) + cw * 64 * 128;
  float o[FA_D / 2];
#pragma unroll
  for (int i = 0; i < FA_D / 2; ++i) o[i] = 0.f;
  float m_run[2] = {-INFINITY, -INFINITY}, l_run[2] = {0.f, 0.f};   // per fragment row; l_run is this lane's partial sum
  tc::mbar_wait(q_full, 0);
  for (int j = 0; j < n_kv; ++j) {
    const int s = j % FA_KV_STAGES, kbase = j * FA_BKV;
    tc::mbar_wait(&kv_full[s], (j / FA_KV_STAGES) & 1);
    const uint32_t kb = tc::smem_u32(sKV + s * FA_STAGE), vb = kb + FA_SK;
    float sc[FA_BKV / 2];
#pragma unroll
    for (int i = 0; i < FA_BKV / 2; ++i) sc[i] = 0.f;
    tc::wgmma_fence();
#pragma unroll
    for (int ks = 0; ks < FA_D / 16; ++ks)
      tc::wgmma_ss<false, FA_BKV>(sc, tc::smem_desc_sw128(qa + ks * 32), tc::smem_desc_sw128(kb + ks * 32), 1u);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::reg_fence(sc);
    if (kbase + FA_BKV > N1) {                      // only the last key tile needs masking
#pragma unroll
      for (int i = 0; i < FA_BKV / 8; ++i)
#pragma unroll
        for (int e = 0; e < 4; ++e)
          if (kbase + 8 * i + fc + (e & 1) >= N1) sc[4 * i + e] = -INFINITY;   // ignored by the max, exp2 -> 0
    }
    uint32_t pa[FA_BKV / 16][4];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      float mx = -INFINITY;
#pragma unroll
      for (int i = 0; i < FA_BKV / 8; ++i) mx = fmaxf(mx, fmaxf(sc[4 * i + 2 * h], sc[4 * i + 2 * h + 1]));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
      mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
      const float m_new = fmaxf(m_run[h], mx);      // finite: every key tile holds at least one key
      const float alpha = fast_exp2(m_run[h] - m_new);
      m_run[h] = m_new;
      float sum = 0.f;
#pragma unroll
      for (int i = 0; i < FA_BKV / 8; ++i) {
        const float p0 = fast_exp2(sc[4 * i + 2 * h] - m_new), p1 = fast_exp2(sc[4 * i + 2 * h + 1] - m_new);
        sum += p0 + p1;
        // S columns 16 kk + {fc, fc + 1} (i = 2 kk) and 16 kk + 8 + {fc, fc + 1} (i = 2 kk + 1) of rows fr / fr + 8 are
        // registers {0, 2} / {1, 3} of the A fragment of K step kk
        pa[i >> 1][(i & 1) * 2 + h] = pack_half2(p0, p1);
      }
      l_run[h] = l_run[h] * alpha + sum;
#pragma unroll
      for (int i = 0; i < FA_D / 8; ++i) { o[4 * i + 2 * h] *= alpha; o[4 * i + 2 * h + 1] *= alpha; }
    }
    tc::wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < FA_BKV / 16; ++kk) tc::wgmma_rs_f16<FA_D>(o, pa[kk], tc::smem_desc_sw128(vb + kk * 32), 1u);
    tc::wgmma_commit();
    tc::wgmma_wait<0>();
    tc::reg_fence(o);
    if (t == 0) tc::mbar_arrive(&kv_empty[s]);
  }
  // normalise by the row sums and store
  const int b = bh / fp.heads, hd = bh - b * fp.heads;
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    float l = l_run[h];
    l += __shfl_xor_sync(0xffffffffu, l, 1);
    l += __shfl_xor_sync(0xffffffffu, l, 2);
    const float inv = 1.f / l;
    const int qrow = q0 + cw * 64 + fr + 8 * h;
    if (qrow >= N1) continue;
    const size_t off = ((size_t)b * N1 + qrow) * fp.D + hd * FA_D + fc;
#pragma unroll
    for (int i = 0; i < FA_D / 8; ++i) {
      const float v0 = o[4 * i + 2 * h] * inv, v1 = o[4 * i + 2 * h + 1] * inv;
      if (fp.out_f16) *reinterpret_cast<uint32_t*>(reinterpret_cast<__half*>(fp.out) + off + 8 * i) = pack_half2(v0, v1);
      else *reinterpret_cast<float2*>(reinterpret_cast<float*>(fp.out) + off + 8 * i) = make_float2(v0, v1);
    }
  }
}

}  // namespace dtk

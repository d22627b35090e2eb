// Cosine-correlation maps: descriptors x all tokens of a frame (models/tracker.py:158-169, :173).
//
//   corr[j][p] = relu( <d_j, F[frame][p]> / max(|d_j| * |F[frame][p]|, 1e-8) )
//
// Two exact-fp32 kernels over the token-major feature video [T][P][C]:
//   * corr_gemm_kernel   -- grouped SGEMM (128 x 128 x 16 tiles, cp.async 3-stage ring) for groups with
//                           many descriptors per frame (anchor phase, wide trajectory batches);
//   * corr_stream_kernel -- HBM-streaming mat-vec for thin groups (<= STREAM_MAX_M descriptors per frame):
//                           every token row is read once, descriptors live in shared memory.
// The reference instead runs einsum("bc,nchw->bnhw") over all B x N pairs and keeps the diagonal.
#include "common.cuh"
#include "corr.cuh"
#include "tcgemm.cuh"

namespace dtk {

constexpr int BM = 128, BN = 128, BK = 16, KPAD = 20, STAGES = 3;
constexpr int GEMM_THREADS = 256;
constexpr int GEMM_SMEM = STAGES * (BM + BN) * KPAD * 4;

__device__ __forceinline__ void cp_async16(void* smem, const void* gmem, bool valid) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  int sz = valid ? 16 : 0;
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;\n" ::"r"(s), "l"(gmem), "r"(sz));
}
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;\n" ::); }
template <int N>
__device__ __forceinline__ void cp_async_wait() { asm volatile("cp.async.wait_group %0;\n" ::"n"(N)); }

// prefix of 128-row tiles per group; thin groups (m <= stream_max) get 0 GEMM tiles.
__global__ void corr_plan_kernel(const int* __restrict__ grp_m, int n_groups, int stream_max, int tile_rows,
                                 int* __restrict__ tile_start, const int* __restrict__ grp_map0, unsigned long long* __restrict__ tkeys,
                                 int n_tiles, int* __restrict__ zero_word) {
  if (tkeys != nullptr) {   // maps of thin groups get no tile keys from the streaming kernel: mark them
    for (int k = 0; k < n_groups; ++k) {
      const int m = grp_m[k];
      if (m <= stream_max)
        for (int r = threadIdx.x; r < m; r += blockDim.x) tkeys[(size_t)(grp_map0[k] + r) * n_tiles] = ~0ull;
    }
  }
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    if (zero_word != nullptr) *zero_word = 0;
    int acc = 0;
    for (int k = 0; k < n_groups; ++k) {
      tile_start[k] = acc;
      int m = grp_m[k];
      if (m > stream_max) acc += (m + tile_rows - 1) / tile_rows;
    }
    tile_start[n_groups] = acc;
  }
}

__global__ void __launch_bounds__(GEMM_THREADS, 2)
corr_gemm_kernel(const float* __restrict__ tpc, const float* __restrict__ norms, int C, int P,
                 const float* __restrict__ desc, const float* __restrict__ desc_norm,
                 const int* __restrict__ grp_frame, const int* __restrict__ grp_row0,
                 const int* __restrict__ grp_m, const int* __restrict__ grp_map0,
                 const int* __restrict__ tile_start, int n_groups, float* __restrict__ maps, int map_stride) {
  extern __shared__ __align__(16) float smem[];
  const int mt = blockIdx.x;
  if (mt >= tile_start[n_groups]) return;
  // last group k with tile_start[k] <= mt and a non-empty tile range: groups with zero tiles share a start with their
  // successor; "last <=" skips them
  const int g = last_le(n_groups, mt, tile_start);
  const int m_grp = grp_m[g];
  const int m0 = (mt - tile_start[g]) * BM;
  const int n0 = blockIdx.y * BN;
  const float* A = desc + (size_t)(grp_row0[g] + m0) * C;
  const float* B = tpc + ((size_t)grp_frame[g] * P + n0) * C;
  const int m_valid = min(BM, m_grp - m0), n_valid = min(BN, P - n0);

  const int tid = threadIdx.x;
  const int tx = tid & 15, ty = tid >> 4;
  float acc[8][8];
#pragma unroll
  for (int i = 0; i < 8; ++i)
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;

  const int KT = (C + BK - 1) / BK;
  auto load_stage = [&](int kt, int s) {
    float* sa = smem + s * (BM + BN) * KPAD;
    float* sb = sa + BM * KPAD;
    const int k0 = kt * BK;
#pragma unroll
    for (int it = 0; it < 2; ++it) {
      int ch = tid + it * GEMM_THREADS;   // 0..511: row = ch / 4, chunk = ch % 4
      int r = ch >> 2, c4 = (ch & 3) * 4;
      bool kin = (k0 + c4) < C;
      bool va = kin && r < m_valid, vb = kin && r < n_valid;  // invalid chunks: zero-fill, in-bounds dummy src
      cp_async16(sa + r * KPAD + c4, va ? A + (size_t)r * C + k0 + c4 : A, va);
      cp_async16(sb + r * KPAD + c4, vb ? B + (size_t)r * C + k0 + c4 : B, vb);
    }
  };

#pragma unroll
  for (int s = 0; s < STAGES - 1; ++s) {
    if (s < KT) load_stage(s, s);
    cp_async_commit();
  }
  for (int kt = 0; kt < KT; ++kt) {
    cp_async_wait<STAGES - 2>();
    __syncthreads();
    {
      int nk = kt + STAGES - 1;
      if (nk < KT) load_stage(nk, nk % STAGES);
      cp_async_commit();
    }
    const float* sa = smem + (kt % STAGES) * (BM + BN) * KPAD;
    const float* sb = sa + BM * KPAD;
#pragma unroll
    for (int kk = 0; kk < BK; kk += 4) {
      float4 a[8];
#pragma unroll
      for (int i = 0; i < 8; ++i) a[i] = *reinterpret_cast<const float4*>(sa + (ty + 16 * i) * KPAD + kk);
#pragma unroll
      for (int j = 0; j < 8; ++j) {
        float4 b = *reinterpret_cast<const float4*>(sb + (tx + 16 * j) * KPAD + kk);
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
  cp_async_wait<0>();

  // epilogue: cosine-normalise (clamp 1e-8), ReLU, store
  const float* fn = norms + (size_t)grp_frame[g] * P + n0;
  const float* dn = desc_norm + grp_row0[g] + m0;
  float fnv[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) fnv[j] = (tx + 16 * j) < n_valid ? fn[tx + 16 * j] : 1.f;
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    int r = ty + 16 * i;
    if (r >= m_valid) continue;
    float dnv = dn[r];
    float* out = maps + (size_t)(grp_map0[g] + m0 + r) * map_stride + n0;
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      int c = tx + 16 * j;
      if (c < n_valid) {
        float v = corr_cos(acc[i][j], dnv, fnv[j]);
        out[c] = fmaxf(v, 0.f);
      }
    }
  }
}

// ---- thin groups: stream every token row once --------------------------------------------------
// HBM-bound: a warp owns 4 token rows at a time; per 16-byte column chunk it issues the 4 row loads
// back to back (x2 unrolled: 8 x LDG.128 in flight per lane, L1 bypassed), reads each descriptor chunk once from
// shared memory and reuses it for the 4 rows.  Grid = token tiles x groups.
constexpr int STREAM_THREADS = 256;
constexpr int STREAM_TOK = 64;   // tokens per CTA: 8 warps x (64 / (8 * RB)) passes x RB rows

__device__ __forceinline__ float4 ldg_stream(const float4* p) {
  float4 r;
  asm volatile("ld.global.nc.L1::no_allocate.v4.f32 {%0, %1, %2, %3}, [%4];"
               : "=f"(r.x), "=f"(r.y), "=f"(r.z), "=f"(r.w) : "l"(p));
  return r;
}

template <int MAXM, int STREAM_RB>
__global__ void __launch_bounds__(STREAM_THREADS)
corr_stream_kernel(const float* __restrict__ tpc, const float* __restrict__ norms, int C, int P,
                   const float* __restrict__ desc, const float* __restrict__ desc_norm,
                   const int* __restrict__ grp_frame, const int* __restrict__ grp_row0,
                   const int* __restrict__ grp_m, const int* __restrict__ grp_map0, int stream_max,
                   float* __restrict__ maps, int map_stride) {
  extern __shared__ __align__(16) float sdesc[];  // [MAXM][C]
  const int g = blockIdx.y;
  const int m = grp_m[g];
  if (m <= 0 || m > stream_max) return;
  const int frame = grp_frame[g], row0 = grp_row0[g], map0 = grp_map0[g];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int C4 = C >> 2;
  for (int mb = 0; mb < m; mb += MAXM) {
    const int mc = min(MAXM, m - mb);
    __syncthreads();
    for (int i = threadIdx.x; i < MAXM * C4; i += STREAM_THREADS)   // unused descriptor slots are zero: no predicates below
      reinterpret_cast<float4*>(sdesc)[i] = i < mc * C4
          ? __ldg(reinterpret_cast<const float4*>(desc + (size_t)(row0 + mb) * C) + i) : make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    for (int t0 = warp * STREAM_RB; t0 < STREAM_TOK; t0 += (STREAM_THREADS / 32) * STREAM_RB) {
      const int p0 = blockIdx.x * STREAM_TOK + t0;
      if (p0 >= P) break;
      const float4* rows[STREAM_RB];
#pragma unroll
      for (int r = 0; r < STREAM_RB; ++r)   // rows past the end re-read the last valid row (result discarded)
        rows[r] = reinterpret_cast<const float4*>(tpc + ((size_t)frame * P + min(p0 + r, P - 1)) * C);
      float acc[MAXM][STREAM_RB];
#pragma unroll
      for (int q = 0; q < MAXM; ++q)
#pragma unroll
        for (int r = 0; r < STREAM_RB; ++r) acc[q][r] = 0.f;
      for (int i = lane; i < C4; i += 64) {
        const int i2 = i + 32;
        const bool two = i2 < C4;
        float4 f0[STREAM_RB], f1[STREAM_RB];
#pragma unroll
        for (int r = 0; r < STREAM_RB; ++r) f0[r] = ldg_stream(rows[r] + i);
#pragma unroll
        for (int r = 0; r < STREAM_RB; ++r) f1[r] = two ? ldg_stream(rows[r] + i2) : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
        for (int q = 0; q < MAXM; ++q) {
          const float4 d0 = reinterpret_cast<const float4*>(sdesc + q * C)[i];
          const float4 d1 = two ? reinterpret_cast<const float4*>(sdesc + q * C)[i2] : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int r = 0; r < STREAM_RB; ++r) {
            float a = acc[q][r];
            a = fmaf(f0[r].x, d0.x, a); a = fmaf(f0[r].y, d0.y, a); a = fmaf(f0[r].z, d0.z, a); a = fmaf(f0[r].w, d0.w, a);
            a = fmaf(f1[r].x, d1.x, a); a = fmaf(f1[r].y, d1.y, a); a = fmaf(f1[r].z, d1.z, a); a = fmaf(f1[r].w, d1.w, a);
            acc[q][r] = a;
          }
        }
      }
#pragma unroll
      for (int r = 0; r < STREAM_RB; ++r) {
        const int p = p0 + r;
        const float fn = p < P ? norms[(size_t)frame * P + p] : 1.f;
#pragma unroll
        for (int q = 0; q < MAXM; ++q) {
          float s = warp_sum(acc[q][r]);
          if (lane == 0 && q < mc && p < P) {
            float v = corr_cos(s, desc_norm[row0 + mb + q], fn);
            maps[(size_t)(map0 + mb + q) * map_stride + p] = fmaxf(v, 0.f);
          }
        }
      }
    }
  }
}

int launch_corr_maps(const FeatView& fv, const float* desc, int desc_rows, const float* desc_norm,
                     const int* grp_frame, const int* grp_row0, const int* grp_m, const int* grp_map0, int n_groups,
                     int total_maps, int max_group_m, float* maps, int map_stride, int* tile_start, float* split_ws,
                     cudaStream_t st, const CorrAssist& assist) {
  if (n_groups <= 0 || total_maps <= 0) return DINOTRK_OK;
  unsigned long long* tkeys = fv.tensor() ? assist.tkeys : nullptr;
  // rows per GEMM M tile: 256 (CTA pairs) by default; 128-row single-CTA tiles when no group can fill more than half a
  // pair tile (10-128 points per call: Tracker.forward-sized batches, small query sets) or when the caller asks for them
  const int tile_rows = fv.tensor() ? ((assist.small_tiles || max_group_m <= 128) ? TC_BM : TC2_BM) : BM;
  const int n_tiles = cdiv(fv.P, CORR_TILE);
  const float* tpc = fv.tpc;
  const float* norms = fv.norms;
  const int C = fv.C, P = fv.P;
  // all_wide: every non-empty group goes through the GEMM, whatever its size (the full-map queue of the exact-window
  // pipeline: a map's arithmetic must not depend on how many other maps of its frame were queued with it)
  const int stream_max = assist.all_wide ? 0 : STREAM_MAX_M;
  if (max_group_m > stream_max || tkeys != nullptr || assist.zero_word != nullptr) {
    ProfRange pr(PROF_MISC, st);
    corr_plan_kernel<<<1, 32, 0, st>>>(grp_m, n_groups, stream_max, tile_rows, tile_start, grp_map0, tkeys, n_tiles,
                                       assist.zero_word);
    DTK_LAUNCHED();
  }
  if (max_group_m > stream_max) {
    // upper bound on sum ceil(m_k / BM) over the wide groups
    int max_tiles = total_maps / tile_rows + n_groups;
    if (fv.tensor()) {
      int rc = launch_corr_gemm_tc(fv.hi, fv.lo, norms, fv.T, C, P, desc, desc_rows, desc_norm, grp_frame, grp_row0,
                                   grp_m, grp_map0, tile_start, n_groups, max_tiles, maps, map_stride, split_ws, st, tkeys,
                                   assist.split_ready, tile_rows, true, nullptr, corr_hilo(fv) ? fv.hilo : nullptr);
      if (rc) return rc;
    } else {
      static PerDev<bool> attr_dev;
      bool& attr_set = attr_dev.get();
      if (!attr_set) {
        DTK_CUDA(cudaFuncSetAttribute(corr_gemm_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, GEMM_SMEM));
        attr_set = true;
      }
      dim3 grid(max_tiles, cdiv(P, BN));
      ProfRange pr(PROF_CORR_GEMM, st);
      corr_gemm_kernel<<<grid, GEMM_THREADS, GEMM_SMEM, st>>>(tpc, norms, C, P, desc, desc_norm, grp_frame,
                                                              grp_row0, grp_m, grp_map0, tile_start, n_groups,
                                                              maps, map_stride);
      DTK_LAUNCHED();
    }
  }
  if (!assist.no_thin && !assist.all_wide) {
    // thin groups (there may be none; CTAs of wide groups exit at once).  Three instantiations: <= 2 or <= 4 descriptors
    // with 8 rows in flight per warp (pure streaming), <= 8 descriptors with 4 rows.
    const int variant = max_group_m <= 2 ? 0 : (max_group_m <= 4 ? 1 : 2);
    const int maxm = variant == 0 ? 2 : (variant == 1 ? 4 : 8);
    size_t smem = (size_t)maxm * C * sizeof(float);
    static PerDev<size_t[3]> attr_smem_dev;
    size_t (&attr_smem)[3] = attr_smem_dev.get();
    auto kern = variant == 0 ? corr_stream_kernel<2, 8> : (variant == 1 ? corr_stream_kernel<4, 8> : corr_stream_kernel<8, 4>);
    if (smem > 48 * 1024 && smem > attr_smem[variant]) {
      DTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      attr_smem[variant] = smem;
    }
    dim3 grid(cdiv(P, STREAM_TOK), n_groups);
    ProfRange pr(PROF_CORR_STREAM, st);
    kern<<<grid, STREAM_THREADS, smem, st>>>(tpc, norms, C, P, desc, desc_norm, grp_frame, grp_row0, grp_m, grp_map0,
                                             stream_max, maps, map_stride);
    DTK_LAUNCHED();
  }
  return DINOTRK_OK;
}

}  // namespace dtk

using namespace dtk;

extern "C" {

int dinotrk_map_stride(const dinotrk_geom* g) { return g ? (int)align_up((size_t)g->h * g->w, 4) : 0; }

size_t dinotrk_corr_maps_workspace_bytes(int total_maps, int n_groups, int C) {
  return align_up(layout_end<CorrMapsWs>(total_maps, n_groups, C), 256) + 1024;
}

int dinotrk_corr_maps(const dinotrk_features* feat, const dinotrk_geom* g, const float* desc, const float* desc_norm,
                      const int* grp_frame, const int* grp_row0, const int* grp_m, const int* grp_map0, int n_groups,
                      int total_maps, int max_group_m, float* maps, void* workspace, size_t workspace_bytes,
                      void* stream) {
  DTK_CHECK_ARG(feat && feat->tpc && feat->norms && g && desc && desc_norm && grp_frame && grp_row0 && grp_m &&
                grp_map0 && maps, "corr_maps: null pointer");
  DTK_CHECK_ARG(feat->T > 0 && feat->C > 0 && feat->C % 4 == 0 && n_groups >= 0 && total_maps >= 0, "corr_maps: bad sizes");
  DTK_CHECK_ARG((feat->hi == nullptr) == (feat->lo == nullptr), "corr_maps: hi and lo must be given together");
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_corr_maps_workspace_bytes(total_maps, n_groups, feat->C),
                "corr_maps: workspace too small");
  Arena ar(workspace);
  const CorrMapsWs ws(ar, total_maps, n_groups, feat->C);
  // rows of desc = total_maps here (one descriptor row per map is the generic contract)
  return launch_corr_maps(make_view(*feat, *g), desc, total_maps, desc_norm, grp_frame, grp_row0, grp_m, grp_map0,
                          n_groups, total_maps, max_group_m, maps, dinotrk_map_stride(g), ws.plan, ws.split,
                          (cudaStream_t)stream);
}

}  // extern "C"

// Foreground masks from DINO features (preprocessing/create_fg_mask.py) and the fg / bg split of the trajectories
// (preprocessing/split_trajectories_to_fg_bg.py).
//
// The reference normalises the T*P x C layer-23 features, centres them and runs torch.pca_lowrank (q = 3, niter = 20),
// which makes three full copies of the features and ~43 tall-skinny GEMM passes over them.  Here the features are read
// in place, token-major [M][C] fp32 (M = T*P may exceed 2^31 elements: every offset is 64-bit), with the row scale s_i
// and the column mean c applied on the fly.  One power pass computes both X = Â P and W = Âᵀ X (Â = diag(s) A - 1cᵀ):
// one warp per row forms the lane partial dots, reduces them with shuffles to x_i and updates per-lane accumulators
// with the rank-1 term (s_i a_i - c) x_iᵀ.  With QR(X) = Q R, Âᵀ Q = W R⁻¹, so a subspace iteration of
// get_approximate_basis (torch/_lowrank.py) costs one read of the features instead of two.
//
// Determinism: the rows are cut into tiles of PCA_TILE rows that depend on M only; a warp accumulates in fp32 over its
// PCA_ROWS rows of a tile, the warps then add into the block's float64 sums one after the other, each block writes its
// float64 partial and one thread per output sums the partials in block order.  Two runs give the same bits.
#include <math.h>

#include <algorithm>

#include "common.cuh"

namespace dtk {

constexpr int PCA_THREADS = 256, PCA_WARPS = PCA_THREADS / 32;
constexpr int PCA_ROWS = 64;                        // rows a warp accumulates in fp32 before the float64 flush
constexpr int PCA_TILE = PCA_WARPS * PCA_ROWS;
constexpr int PCA_MAX_BLOCKS = 1056;                // 8 waves of 132 SMs; a constant, so the sums do not depend on the GPU
constexpr int PCA_MAX_C = 1536, PCA_MAX_Q = 4;

static inline int pca_blocks(long long M) {
  return (int)std::min<long long>((M + PCA_TILE - 1) / PCA_TILE, PCA_MAX_BLOCKS);
}

// Lane l owns the float4 chunks 4 (l + 32 r), r < NCH, of a row (NCH = ceil(C / 128)).
template <int NCH>
__device__ __forceinline__ void load_row(const float* __restrict__ row, int C, int lane, float4 (&v)[NCH]) {
#pragma unroll
  for (int r = 0; r < NCH; ++r) {
    const int k = 4 * (lane + 32 * r);
    v[r] = k < C ? __ldg(reinterpret_cast<const float4*>(row + k)) : make_float4(0.f, 0.f, 0.f, 0.f);
  }
}

__device__ __forceinline__ double warp_sum_f64(double v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}

// The warps of the block add their N per-lane values (lane l's chunk r, element e, component j at
// smem[(4 (l + 32 r) + e) * Q + j]) into the block's float64 sums in warp order.
template <int NCH, int Q, typename Acc>
__device__ __forceinline__ void flush_ordered(double* __restrict__ sum, const Acc (&acc)[NCH][4][Q], int C, int lane,
                                              int warp) {
  for (int w = 0; w < PCA_WARPS; ++w) {
    if (w == warp) {
#pragma unroll
      for (int r = 0; r < NCH; ++r) {
        const int k = 4 * (lane + 32 * r);
        if (k < C) {
#pragma unroll
          for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int j = 0; j < Q; ++j) sum[(k + e) * Q + j] += (double)acc[r][e][j];
        }
      }
    }
    __syncthreads();
  }
}

// ---- row statistics: s_i = 1 / max(|a_i|, 1e-12) (F.normalize's rule) or 1, and the column sums of diag(s) A ------
template <int NCH>
__global__ void __launch_bounds__(PCA_THREADS, 1)
pca_stats_kernel(const float* __restrict__ a, long long M, int C, int normalize, float* __restrict__ s_out,
                 double* __restrict__ part) {
  extern __shared__ double sm_sum[];                  // [C]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < C; i += PCA_THREADS) sm_sum[i] = 0.0;
  __syncthreads();
  const long long tiles = (M + PCA_TILE - 1) / PCA_TILE;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    double acc[NCH][4][1] = {};
    const long long r0 = tile * PCA_TILE + (long long)warp * PCA_ROWS, r1 = min(r0 + PCA_ROWS, M);
    for (long long i = r0; i < r1; ++i) {
      float4 v[NCH];
      load_row<NCH>(a + i * (long long)C, C, lane, v);
      float s = 1.f;
      if (normalize) {
        double ss = 0.0;
#pragma unroll
        for (int r = 0; r < NCH; ++r)
          ss += (double)v[r].x * v[r].x + (double)v[r].y * v[r].y + (double)v[r].z * v[r].z + (double)v[r].w * v[r].w;
        s = (float)(1.0 / fmax(sqrt(warp_sum_f64(ss)), 1e-12));
      }
      if (lane == 0) s_out[i] = s;
#pragma unroll
      for (int r = 0; r < NCH; ++r) {
        acc[r][0][0] += (double)__fmul_rn(s, v[r].x);
        acc[r][1][0] += (double)__fmul_rn(s, v[r].y);
        acc[r][2][0] += (double)__fmul_rn(s, v[r].z);
        acc[r][3][0] += (double)__fmul_rn(s, v[r].w);
      }
    }
    flush_ordered<NCH, 1>(sm_sum, acc, C, lane, warp);
  }
  for (int i = threadIdx.x; i < C; i += PCA_THREADS) part[(size_t)blockIdx.x * C + i] = sm_sum[i];
}

// ---- power pass: X = Â P [M][Q], and the block partials of W = Âᵀ X [C][Q] -------------------------------------------
// A row is read by a team of TEAM warps, warp h of the team owning chunks [h NCHH, (h + 1) NCHH) of it: one warp up to
// C = 1024 at Q = 3 (96 fp32 accumulators per lane), two above, so that no configuration spills.  The two warps of a
// team add their partial dots through shared memory (double-buffered by row parity, one named barrier per row).
template <int Q, int NCH>
struct PowerShape {
  static constexpr int TEAM = NCH * Q > 24 ? 2 : 1;
  static constexpr int NCHH = (NCH + TEAM - 1) / TEAM;
};

template <int Q, int NCH>
__global__ void __launch_bounds__(PCA_THREADS, 1)
pca_power_kernel(const float* __restrict__ a, long long M, int C, const float* __restrict__ s, const float* __restrict__ c,
                 const float* __restrict__ P, float* __restrict__ X, double* __restrict__ part) {
  constexpr int TEAM = PowerShape<Q, NCH>::TEAM, NCHH = PowerShape<Q, NCH>::NCHH, TEAMS = PCA_WARPS / TEAM;
  constexpr int TILE = TEAMS * PCA_ROWS;
  extern __shared__ double sm_sum[];                  // [C][Q] float64, then P [C][Q] and c [C] fp32
  __shared__ float s_x[TEAMS][2][TEAM][Q];
  float* sm_p = reinterpret_cast<float*>(sm_sum + (size_t)C * Q);
  float* sm_c = sm_p + (size_t)C * Q;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, team = warp / TEAM, h = warp % TEAM;
  const int k0 = 128 * NCHH * h;                      // first column of this warp's share of the row
  for (int i = threadIdx.x; i < C * Q; i += PCA_THREADS) { sm_sum[i] = 0.0; sm_p[i] = P[i]; }
  for (int i = threadIdx.x; i < C; i += PCA_THREADS) sm_c[i] = c[i];
  __syncthreads();
  const long long tiles = (M + TILE - 1) / TILE;
  for (long long tile = blockIdx.x; tile < tiles; tile += gridDim.x) {
    float acc[NCHH][4][Q] = {};
    const long long r0 = tile * TILE + (long long)team * PCA_ROWS, r1 = min(r0 + PCA_ROWS, M);
    for (long long i = r0; i < r1; ++i) {
      float4 v[NCHH];
      load_row<NCHH>(a + i * (long long)C + k0, C - k0, lane, v);
      const float si = __ldg(s + i);
      float d[Q] = {};
#pragma unroll
      for (int r = 0; r < NCHH; ++r) {
        const int k = k0 + 4 * (lane + 32 * r);
        if (k < C) {
          const float4 cc = *reinterpret_cast<const float4*>(sm_c + k);
          v[r].x = __fsub_rn(__fmul_rn(si, v[r].x), cc.x);
          v[r].y = __fsub_rn(__fmul_rn(si, v[r].y), cc.y);
          v[r].z = __fsub_rn(__fmul_rn(si, v[r].z), cc.z);
          v[r].w = __fsub_rn(__fmul_rn(si, v[r].w), cc.w);
          const float* p = sm_p + (size_t)k * Q;
          const float ve[4] = {v[r].x, v[r].y, v[r].z, v[r].w};
#pragma unroll
          for (int e = 0; e < 4; ++e)
#pragma unroll
            for (int j = 0; j < Q; ++j) d[j] = fmaf(ve[e], p[e * Q + j], d[j]);
        }
      }
      float x[Q];
#pragma unroll
      for (int j = 0; j < Q; ++j) x[j] = warp_sum(d[j]);
      if (TEAM > 1) {
        const int par = (int)(i & 1);
#pragma unroll
        for (int j = 0; j < Q; ++j)
          if (lane == j) s_x[team][par][h][j] = x[j];
        asm volatile("bar.sync %0, %1;" ::"r"(team + 1), "r"(32 * TEAM) : "memory");
#pragma unroll
        for (int j = 0; j < Q; ++j) x[j] = __fadd_rn(s_x[team][par][0][j], s_x[team][par][TEAM - 1][j]);
      }
      if (h == 0) {
#pragma unroll
        for (int j = 0; j < Q; ++j)
          if (lane == j) X[i * Q + j] = x[j];
      }
#pragma unroll
      for (int r = 0; r < NCHH; ++r) {
        const float ve[4] = {v[r].x, v[r].y, v[r].z, v[r].w};    // zero past C
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
          for (int j = 0; j < Q; ++j) acc[r][e][j] = fmaf(ve[e], x[j], acc[r][e][j]);
      }
    }
    flush_ordered<NCHH, Q>(sm_sum + (size_t)k0 * Q, acc, C - k0, lane, warp);
  }
  for (int i = threadIdx.x; i < C * Q; i += PCA_THREADS) part[(size_t)blockIdx.x * C * Q + i] = sm_sum[i];
}

// out[i] = (sum over blocks b in order of part[b][i]) / div
__global__ void pca_reduce_kernel(const double* __restrict__ part, int blocks, int n, double div, float* __restrict__ out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  double acc = 0.0;
  for (int b = 0; b < blocks; ++b) acc += part[(size_t)b * n + i];
  out[i] = (float)(acc / div);
}

// ---- the mask: colors = diag(s) A V (not centred, create_fg_mask.py:29) and the min / max of every column ----------
// float <-> int keys whose signed order is the float order (atomicMin / atomicMax give the exact extremes)
__device__ __forceinline__ int f2key(float f) { const int b = __float_as_int(f); return b >= 0 ? b : b ^ 0x7fffffff; }
__device__ __forceinline__ float key2f(int k) { return __int_as_float(k >= 0 ? k : k ^ 0x7fffffff); }

template <int Q, int NCH>
__global__ void __launch_bounds__(PCA_THREADS)
pca_project_kernel(const float* __restrict__ a, long long M, int C, const float* __restrict__ s, const float* __restrict__ V,
                   float* __restrict__ colors, int* __restrict__ minmax) {
  extern __shared__ float sm_v[];                     // [C][Q]
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  for (int i = threadIdx.x; i < C * Q; i += PCA_THREADS) sm_v[i] = V[i];
  __syncthreads();
  float mn[Q], mx[Q];
#pragma unroll
  for (int j = 0; j < Q; ++j) { mn[j] = INFINITY; mx[j] = -INFINITY; }
  const long long warps = (long long)gridDim.x * PCA_WARPS;
  for (long long i = (long long)blockIdx.x * PCA_WARPS + warp; i < M; i += warps) {
    float4 v[NCH];
    load_row<NCH>(a + i * (long long)C, C, lane, v);
    const float si = __ldg(s + i);
    float d[Q] = {};
#pragma unroll
    for (int r = 0; r < NCH; ++r) {
      const int k = 4 * (lane + 32 * r);
      if (k < C) {
        const float* p = sm_v + (size_t)k * Q;
        const float ve[4] = {__fmul_rn(si, v[r].x), __fmul_rn(si, v[r].y), __fmul_rn(si, v[r].z), __fmul_rn(si, v[r].w)};
#pragma unroll
        for (int e = 0; e < 4; ++e)
#pragma unroll
          for (int j = 0; j < Q; ++j) d[j] = fmaf(ve[e], p[e * Q + j], d[j]);
      }
    }
#pragma unroll
    for (int j = 0; j < Q; ++j) {
      const float x = warp_sum(d[j]);
      if (lane == j) colors[i * Q + j] = x;
      mn[j] = fminf(mn[j], x);
      mx[j] = fmaxf(mx[j], x);
    }
  }
  if (lane == 0) {
#pragma unroll
    for (int j = 0; j < Q; ++j) {
      atomicMin(minmax + j, f2key(mn[j]));
      atomicMax(minmax + PCA_MAX_Q + j, f2key(mx[j]));
    }
  }
}

__global__ void minmax_init_kernel(int* minmax) {
  const int j = threadIdx.x;
  if (j < PCA_MAX_Q) { minmax[j] = f2key(INFINITY); minmax[PCA_MAX_Q + j] = f2key(-INFINITY); }
}

// create_fg_mask.py:33-34 in fp32: (col0 - min0) / (max0 - min0) < threshold -> 1
__global__ void token_mask_kernel(const float* __restrict__ colors, long long M, int Q, const int* __restrict__ minmax,
                                  float threshold, uint8_t* __restrict__ mask) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= M) return;
  const float mn = key2f(minmax[0]), mx = key2f(minmax[PCA_MAX_Q]);
  mask[i] = __fdiv_rn(__fsub_rn(colors[i * Q], mn), __fsub_rn(mx, mn)) < threshold ? 1 : 0;
}

// F.interpolate(mode="nearest") of a [T][h][w] 0/1 mask to [T][H][W] 0/255: ATen's nearest source index
// min((int)floorf(dst * ((float)in / out)), in - 1)
__global__ void mask_upsample_kernel(const uint8_t* __restrict__ tm, int T, int h, int w, int H, int W,
                                     uint8_t* __restrict__ out) {
  const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long HW = (long long)H * W;
  if (i >= (long long)T * HW) return;
  const int t = (int)(i / HW), rem = (int)(i - t * HW), y = rem / W, x = rem - y * W;
  const float sy = (float)h / (float)H, sx = (float)w / (float)W;
  const int iy = min((int)floorf(__fmul_rn((float)y, sy)), h - 1), ix = min((int)floorf(__fmul_rn((float)x, sx)), w - 1);
  out[i] = tm[((size_t)t * h + iy) * w + ix] ? 255 : 0;
}

// ---- split_trajectories_to_fg_bg.py:55-78 --------------------------------------------------------------------------
constexpr int SPLIT_THREADS = 256;

// cls[n] = 1 (fg: mask at the rounded start > 0), 0 (bg), 2 (no valid step, or the start rounds outside the frame);
// cnt[b] = fg rows of block b; counts[1] = bad rows, counts[2] = the first bad row.
__global__ void __launch_bounds__(SPLIT_THREADS)
split_count_kernel(const float2* __restrict__ traj, int N, int T, const uint8_t* __restrict__ masks, int Tm, int H, int W,
                   uint8_t* __restrict__ cls, int* __restrict__ cnt, int* __restrict__ counts) {
  const int n = blockIdx.x * SPLIT_THREADS + threadIdx.x;
  int c = 0;
  if (n < N) {
    const float2* row = traj + (size_t)n * T;
    int t = 0;
    float2 p = make_float2(NAN, NAN);
    for (; t < T; ++t) {
      p = row[t];
      if (!isnan(p.x) && !isnan(p.y)) break;
    }
    const float x = rintf(p.x), y = rintf(p.y);   // torch.round: half to even
    if (t < T && t < Tm && x >= 0.f && x <= (float)(W - 1) && y >= 0.f && y <= (float)(H - 1)) {
      c = masks[((size_t)t * H + (size_t)y) * W + (size_t)x] > 0 ? 1 : 0;
    } else {
      c = 2;
      atomicAdd(counts + 1, 1);
      atomicMin(counts + 2, n);
    }
    cls[n] = (uint8_t)c;
  }
  const int nf = __syncthreads_count(c == 1);
  if (threadIdx.x == 0) cnt[blockIdx.x] = nf;
}

// Row n of block b -> fg[off[b] + rank among the block's fg rows] or bg[b * 256 - off[b] + rank among its bg rows];
// the warps then copy the block's rows, lanes along the row.
__global__ void __launch_bounds__(SPLIT_THREADS)
split_emit_kernel(const float2* __restrict__ traj, int N, int T, const uint8_t* __restrict__ cls, const int* __restrict__ off,
                  float2* __restrict__ fg, float2* __restrict__ bg) {
  __shared__ long long s_dst[SPLIT_THREADS];          // fg row, or -1 - bg row
  const int n = blockIdx.x * SPLIT_THREADS + threadIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const bool is_fg = n < N && cls[n] == 1;
  const int rank = block_rank<SPLIT_THREADS>(is_fg);
  const int fg0 = off[blockIdx.x], bg0 = blockIdx.x * SPLIT_THREADS - fg0;
  s_dst[threadIdx.x] = is_fg ? (long long)(fg0 + rank) : -1 - (long long)(bg0 + threadIdx.x - rank);
  __syncthreads();
  const int rows = min(SPLIT_THREADS, N - blockIdx.x * SPLIT_THREADS);
  for (int r = warp; r < rows; r += SPLIT_THREADS / 32) {
    const long long d = s_dst[r];
    const float2* src = traj + ((size_t)blockIdx.x * SPLIT_THREADS + r) * T;
    float2* dst = d >= 0 ? fg + (size_t)d * T : bg + (size_t)(-1 - d) * T;
    for (int t = lane; t < T; t += 32) dst[t] = src[t];
  }
}

}  // namespace dtk

using namespace dtk;

#define DTK_PCA_NCH_CASES(F, ...) \
  switch ((C + 127) / 128) {                                                                                       \
    case 1: F(1, __VA_ARGS__); break; case 2: F(2, __VA_ARGS__); break; case 3: F(3, __VA_ARGS__); break;          \
    case 4: F(4, __VA_ARGS__); break; case 5: F(5, __VA_ARGS__); break; case 6: F(6, __VA_ARGS__); break;          \
    case 7: F(7, __VA_ARGS__); break; case 8: F(8, __VA_ARGS__); break; case 9: F(9, __VA_ARGS__); break;          \
    case 10: F(10, __VA_ARGS__); break; case 11: F(11, __VA_ARGS__); break; default: F(12, __VA_ARGS__); break;    \
  }

namespace {

template <typename K>
int allow_smem(K kernel, size_t smem) {
  DTK_CUDA(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
  return DINOTRK_OK;
}

int pca_args_ok(const float* a, long long M, int C, int q) {
  DTK_CHECK_ARG(a && M > 0, "pca: null features or M <= 0");
  DTK_CHECK_ARG(C > 0 && C % 4 == 0 && C <= PCA_MAX_C, "pca: C = %d must be a positive multiple of 4 and <= %d", C, PCA_MAX_C);
  DTK_CHECK_ARG(q >= 1 && q <= PCA_MAX_Q, "pca: q = %d outside [1, %d]", q, PCA_MAX_Q);
  DTK_CHECK_ARG(((uintptr_t)a & 15) == 0, "pca: features must be 16-byte aligned");
  return DINOTRK_OK;
}

template <int NCH>
int run_stats(const float* a, long long M, int C, int normalize, float* s, double* part, cudaStream_t st) {
  const int G = pca_blocks(M);
  const size_t smem = (size_t)C * sizeof(double);
  if (int rc = allow_smem(pca_stats_kernel<NCH>, smem)) return rc;
  pca_stats_kernel<NCH><<<G, PCA_THREADS, smem, st>>>(a, M, C, normalize, s, part);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

template <int Q, int NCH>
int run_power(const float* a, long long M, int C, const float* s, const float* c, const float* P, float* X, double* part,
              cudaStream_t st) {
  const int G = pca_blocks(M);
  const size_t smem = (size_t)C * Q * sizeof(double) + (size_t)C * Q * sizeof(float) + (size_t)C * sizeof(float);
  if (int rc = allow_smem(pca_power_kernel<Q, NCH>, smem)) return rc;
  pca_power_kernel<Q, NCH><<<G, PCA_THREADS, smem, st>>>(a, M, C, s, c, P, X, part);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

template <int Q, int NCH>
int run_project(const float* a, long long M, int C, const float* s, const float* V, float* colors, int* minmax,
                cudaStream_t st) {
  const size_t smem = (size_t)C * Q * sizeof(float);
  const int G = (int)std::min<long long>((M + PCA_WARPS - 1) / PCA_WARPS, 4LL * num_sms());
  if (int rc = allow_smem(pca_project_kernel<Q, NCH>, smem)) return rc;
  pca_project_kernel<Q, NCH><<<G, PCA_THREADS, smem, st>>>(a, M, C, s, V, colors, minmax);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // namespace

extern "C" {

size_t dinotrk_pca_workspace_bytes(long long M, int C, int q) {
  if (M <= 0 || C <= 0 || q <= 0) return 0;
  return align_up((size_t)pca_blocks(M) * C * std::max(q, 1) * sizeof(double), 256) + 256 + 256;
}

int dinotrk_pca_stats(const float* a, long long M, int C, int normalize, float* s, float* c, void* workspace,
                      size_t workspace_bytes, void* stream) {
  if (int rc = pca_args_ok(a, M, C, 1)) return rc;
  DTK_CHECK_ARG(s && c && workspace, "pca_stats: null argument");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_pca_workspace_bytes(M, C, 1), "pca_stats: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  double* part = (double*)workspace;
  ProfRange pr(PROF_FG_MASK, st);
#define DTK_STATS(NCH, ...) if (int rc = run_stats<NCH>(a, M, C, normalize, s, part, st)) return rc
  DTK_PCA_NCH_CASES(DTK_STATS, 0)
#undef DTK_STATS
  pca_reduce_kernel<<<cdiv(C, 256), 256, 0, st>>>(part, pca_blocks(M), C, (double)M, c);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_pca_power(const float* a, long long M, int C, int q, const float* s, const float* c, const float* P, float* X,
                      float* W, void* workspace, size_t workspace_bytes, void* stream) {
  if (int rc = pca_args_ok(a, M, C, q)) return rc;
  DTK_CHECK_ARG(s && c && P && X && W && workspace, "pca_power: null argument");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_pca_workspace_bytes(M, C, q), "pca_power: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  double* part = (double*)workspace;
  ProfRange pr(PROF_FG_MASK, st);
#define DTK_POWER(NCH, Q) if (int rc = run_power<Q, NCH>(a, M, C, s, c, P, X, part, st)) return rc
  switch (q) {
    case 1: DTK_PCA_NCH_CASES(DTK_POWER, 1) break;
    case 2: DTK_PCA_NCH_CASES(DTK_POWER, 2) break;
    case 3: DTK_PCA_NCH_CASES(DTK_POWER, 3) break;
    default: DTK_PCA_NCH_CASES(DTK_POWER, 4) break;
  }
#undef DTK_POWER
  pca_reduce_kernel<<<cdiv(C * q, 256), 256, 0, st>>>(part, pca_blocks(M), C * q, 1.0, W);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_mask_upsample(const uint8_t* token_mask, int T, int h, int w, int H, int W, uint8_t* out, void* stream) {
  DTK_CHECK_ARG(token_mask && out && T > 0 && h > 0 && w > 0 && H > 0 && W > 0, "mask_upsample: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  const long long n = (long long)T * H * W;
  ProfRange pr(PROF_FG_MASK, st);
  mask_upsample_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(token_mask, T, h, w, H, W, out);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_fg_mask(const float* a, int T, int h, int w, int C, int q, const float* s, const float* V, float threshold,
                    int H, int W, float* colors, uint8_t* token_mask, uint8_t* mask, void* workspace, size_t workspace_bytes,
                    void* stream) {
  DTK_CHECK_ARG(T > 0 && h > 0 && w > 0, "fg_mask: T, h, w must be positive");
  const long long M = (long long)T * h * w;
  if (int rc = pca_args_ok(a, M, C, q)) return rc;
  DTK_CHECK_ARG(s && V && colors && token_mask && mask && workspace && H > 0 && W > 0, "fg_mask: bad arguments");
  DTK_CHECK_ARG(workspace_bytes >= 2 * PCA_MAX_Q * sizeof(int), "fg_mask: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  int* minmax = (int*)workspace;
  {
    ProfRange pr(PROF_FG_MASK, st);
    minmax_init_kernel<<<1, 32, 0, st>>>(minmax);
    DTK_LAUNCHED();
#define DTK_PROJECT(NCH, Q) if (int rc = run_project<Q, NCH>(a, M, C, s, V, colors, minmax, st)) return rc
    switch (q) {
      case 1: DTK_PCA_NCH_CASES(DTK_PROJECT, 1) break;
      case 2: DTK_PCA_NCH_CASES(DTK_PROJECT, 2) break;
      case 3: DTK_PCA_NCH_CASES(DTK_PROJECT, 3) break;
      default: DTK_PCA_NCH_CASES(DTK_PROJECT, 4) break;
    }
#undef DTK_PROJECT
    token_mask_kernel<<<(unsigned)((M + 255) / 256), 256, 0, st>>>(colors, M, q, minmax, threshold, token_mask);
    DTK_LAUNCHED();
  }
  return dinotrk_mask_upsample(token_mask, T, h, w, H, W, mask, stream);
}

struct SplitWs {
  uint8_t* cls; int* cnt; int* off; int* counts;
  SplitWs(Arena& ar, int N) {
    const size_t nb = (size_t)(N > 0 ? cdiv(N, SPLIT_THREADS) : 1);
    cls = ar.take<uint8_t>((size_t)std::max(N, 1));
    cnt = ar.take<int>(nb);
    off = ar.take<int>(nb);
    counts = ar.take<int>(4);
  }
};

size_t dinotrk_traj_split_workspace_bytes(int N) { return align_up(layout_end<SplitWs>(N), 256) + 256; }

int dinotrk_traj_split_count(const float* traj, int N, int T, const uint8_t* masks, int Tm, int H, int W, int* n_fg,
                             void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(traj && masks && n_fg && workspace && N > 0 && T > 0 && Tm > 0 && H > 0 && W > 0,
                "traj_split_count: bad arguments");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_traj_split_workspace_bytes(N), "traj_split_count: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = cdiv(N, SPLIT_THREADS);
  Arena ar(workspace);
  const SplitWs w(ar, N);
  const int init[4] = {0, 0, N, 0};
  DTK_CUDA(cudaMemcpyAsync(w.counts, init, sizeof(init), cudaMemcpyHostToDevice, st));
  {
    ProfRange pr(PROF_MISC, st);
    split_count_kernel<<<nb, SPLIT_THREADS, 0, st>>>(reinterpret_cast<const float2*>(traj), N, T, masks, Tm, H, W, w.cls,
                                                      w.cnt, w.counts);
    DTK_LAUNCHED();
    if (int rc = launch_count_scan(w.cnt, nb, 1, w.off, w.counts, st)) return rc;
  }
  int host[4];
  DTK_CUDA(cudaMemcpyAsync(host, w.counts, sizeof(host), cudaMemcpyDeviceToHost, st));
  DTK_CUDA(cudaStreamSynchronize(st));
  DTK_CHECK_ARG(host[1] == 0, "traj_split: %d trajectories have no valid step or start outside the %dx%d frame or past "
                "mask frame %d (first: row %d)", host[1], W, H, Tm - 1, host[2]);
  *n_fg = host[0];
  return DINOTRK_OK;
}

int dinotrk_traj_split_emit(const float* traj, int N, int T, float* fg, float* bg, void* workspace, size_t workspace_bytes,
                            void* stream) {
  DTK_CHECK_ARG(traj && workspace && N > 0 && T > 0, "traj_split_emit: bad arguments");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_traj_split_workspace_bytes(N), "traj_split_emit: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = cdiv(N, SPLIT_THREADS);
  Arena ar(workspace);
  const SplitWs w(ar, N);
  ProfRange pr(PROF_MISC, st);
  split_emit_kernel<<<nb, SPLIT_THREADS, 0, st>>>(reinterpret_cast<const float2*>(traj), N, T, w.cls, w.off,
                                                   reinterpret_cast<float2*>(fg), reinterpret_cast<float2*>(bg));
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // extern "C"

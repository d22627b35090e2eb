// The training-batch sampler (data/dataset.py:56-258 DinoTrackerSampler / LongRangeSampler).
//
// The reference keeps the valid trajectories and a [N'][T] bool can_sample, and on every call builds can_sample.float()
// over the whole set and copies every candidate row twice by boolean indexing, to keep at most `batch` of them.  Here
// the valid rows are compacted once (prepare) next to a bitmask of their valid frames, ceil(T / 32) words per row; a
// call then writes per-block candidate counts and their scan (count), finds the randperm-selected candidates by
// position (select) and copies the drawn points (gather).  Nothing proportional to N' * T is written per call.
//
// The stored rows may live in pinned host memory (the windowed mode): gather and prepare then read and write them
// through the device's mapping of that memory, touching only the rows they need.  Every element offset is 64-bit.
#include <math.h>

#include "common.cuh"

namespace dtk {

constexpr int SMP_THREADS = 256;
constexpr int SMP_MAX_T = 65536;

__host__ __device__ __forceinline__ int smp_words(int T) { return (T + 31) / 32; }

// prepare: row n is valid when more than one step has both coordinates non-NaN (dataset.py:100-106)
__device__ __forceinline__ int valid_steps(const float2* __restrict__ row, int T) {
  int c = 0;
  for (int t = 0; t < T; ++t) {
    const float2 p = row[t];
    c += (!isnan(p.x) && !isnan(p.y)) ? 1 : 0;
  }
  return c;
}

__global__ void __launch_bounds__(SMP_THREADS)
sampler_prepare_count_kernel(const float2* __restrict__ traj, int N, int T, int* __restrict__ block_cnt) {
  const int n = blockIdx.x * SMP_THREADS + threadIdx.x;
  const bool keep = n < N && valid_steps(traj + (size_t)n * T, T) > 1;
  const int c = __syncthreads_count(keep);
  if (threadIdx.x == 0) block_cnt[blockIdx.x] = c;
}

// Valid row n of block b -> stored row off[b] + (rank of n among the block's valid rows): its T positions and its
// frame bits (bit t of word t / 32 set where step t is valid).
__global__ void __launch_bounds__(SMP_THREADS)
sampler_prepare_emit_kernel(const float2* __restrict__ traj, int N, int T, const int* __restrict__ off,
                            float2* __restrict__ rows, uint32_t* __restrict__ bits) {
  const int n = blockIdx.x * SMP_THREADS + threadIdx.x;
  const float2* src = traj + (size_t)n * T;
  const bool keep = n < N && valid_steps(src, T) > 1;
  const int rank = block_rank<SMP_THREADS>(keep);
  if (!keep) return;
  const size_t r = (size_t)off[blockIdx.x] + rank;
  float2* dst = rows + r * T;
  uint32_t* b = bits + r * smp_words(T);
  uint32_t word = 0;
  for (int t = 0; t < T; ++t) {
    const float2 p = src[t];
    dst[t] = p;
    if (!isnan(p.x) && !isnan(p.y)) word |= 1u << (t & 31);
    if ((t & 31) == 31 || t == T - 1) { b[t >> 5] = word; word = 0; }
  }
}

// The frame mask of the drawn frame indices (randperm values: distinct, in [0, T)) in shared memory.
__device__ __forceinline__ void build_mask(uint32_t* s_mask, int W, int T, const int64_t* __restrict__ frames, int k) {
  for (int i = threadIdx.x; i < W; i += blockDim.x) s_mask[i] = 0u;
  __syncthreads();
  for (int i = threadIdx.x; i < k; i += blockDim.x) {
    const int64_t f = frames[i];
    if (f >= 0 && f < T) atomicOr(s_mask + (f >> 5), 1u << (f & 31));
  }
  __syncthreads();
}

// popcount(bits & mask) >= 2 (dataset.py:171)
__device__ __forceinline__ bool is_candidate(const uint32_t* __restrict__ bits, const uint32_t* s_mask, int W, int n) {
  int c = 0;
  const uint32_t* b = bits + (size_t)n * W;
  for (int w = 0; w < W && c < 2; ++w) c += __popc(__ldg(b + w) & s_mask[w]);
  return c >= 2;
}

__global__ void __launch_bounds__(SMP_THREADS)
sampler_count_kernel(const uint32_t* __restrict__ bits, int N, int T, const int64_t* __restrict__ frames, int k,
                     int* __restrict__ block_cnt) {
  extern __shared__ uint32_t s_mask[];
  const int W = smp_words(T);
  build_mask(s_mask, W, T, frames, k);
  const int n = blockIdx.x * SMP_THREADS + threadIdx.x;
  const int c = __syncthreads_count(n < N && is_candidate(bits, s_mask, W, n));
  if (threadIdx.x == 0) block_cnt[blockIdx.x] = c;
}

// One warp per selected position perm[i] (< the candidate total): the block b holding it is the last with
// off[b] <= pos, the row is the (pos - off[b])-th candidate of that block.  Writes row_ids[i] and the multinomial's
// weight row mat[i][t] = 1 where t is a drawn frame and valid on that row, else 0 (dataset.py:180-183).
constexpr int SEL_WARPS = 8;
__global__ void __launch_bounds__(SEL_WARPS * 32)
sampler_select_kernel(const uint32_t* __restrict__ bits, int N, int T, const int64_t* __restrict__ frames, int k,
                      const int* __restrict__ off, int nb, const int64_t* __restrict__ perm, int m,
                      int64_t* __restrict__ row_ids, float* __restrict__ mat) {
  extern __shared__ uint32_t s_mask[];
  const int W = smp_words(T);
  build_mask(s_mask, W, T, frames, k);
  const int lane = threadIdx.x & 31, i = blockIdx.x * SEL_WARPS + (threadIdx.x >> 5);
  if (i >= m) return;
  const int pos = (int)perm[i];
  const int blk = last_le(nb, pos, off);
  const int row = warp_nth_hit(blk * SMP_THREADS, min(blk * SMP_THREADS + SMP_THREADS, N), pos - off[blk],
                               [&](int n) { return is_candidate(bits, s_mask, W, n); });
  if (lane == 0) row_ids[i] = row;
  float* out = mat + (size_t)i * T;
  if (row < 0) {   // a position past the candidate total: no row, no weight
    for (int t = lane; t < T; t += 32) out[t] = 0.f;
    return;
  }
  const uint32_t* b = bits + (size_t)row * W;
  for (int t = lane; t < T; t += 32) out[t] = ((__ldg(b + (t >> 5)) & s_mask[t >> 5]) >> (t & 31)) & 1u ? 1.f : 0.f;
}

// t1[i] = (rows[row_ids[i]][draws[i][0]], draws[i][0]) and t2 likewise with draws[i][1] (dataset.py:184-188)
__global__ void sampler_gather_kernel(const float2* __restrict__ rows, int T, const int64_t* __restrict__ row_ids,
                                      const int64_t* __restrict__ draws, int m, float* __restrict__ t1, float* __restrict__ t2) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= 2 * m) return;
  const int i = j >> 1;
  const int64_t t = draws[j];
  const float2 p = rows[(size_t)row_ids[i] * T + (size_t)t];
  float* o = ((j & 1) ? t2 : t1) + 3 * (size_t)i;
  o[0] = p.x;
  o[1] = p.y;
  o[2] = (float)t;
}

// The device's address of a buffer in device, managed or pinned host memory; null for pageable host memory.
static const void* device_view(const void* p) {
  cudaPointerAttributes a;
  if (cudaPointerGetAttributes(&a, p) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  if (a.type == cudaMemoryTypeDevice || a.type == cudaMemoryTypeManaged) return p;
  if (a.type == cudaMemoryTypeHost) return a.devicePointer;
  return nullptr;
}

struct SamplerWs {
  int* cnt; int* off; int* total;
  SamplerWs(Arena& ar, int N) {
    const size_t nb = (size_t)(N > 0 ? cdiv(N, SMP_THREADS) : 1);
    cnt = ar.take<int>(nb);
    off = ar.take<int>(nb);
    total = ar.take<int>(1);
  }
};

static int read_total(const SamplerWs& w, int* out, cudaStream_t st) {
  int host = 0;
  DTK_CUDA(cudaMemcpyAsync(&host, w.total, sizeof(int), cudaMemcpyDeviceToHost, st));
  DTK_CUDA(cudaStreamSynchronize(st));
  *out = host;
  return DINOTRK_OK;
}

}  // namespace dtk

using namespace dtk;

extern "C" {

size_t dinotrk_sampler_workspace_bytes(int N) { return align_up(layout_end<SamplerWs>(N), 256) + 256; }

int dinotrk_sampler_prepare_count(const float* traj, int N, int T, int* n_valid, void* workspace, size_t workspace_bytes,
                                  void* stream) {
  DTK_CHECK_ARG(traj && n_valid && workspace && N > 0 && T > 0 && T <= SMP_MAX_T,
                "sampler_prepare_count: bad arguments (N = %d, T = %d)", N, T);
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_sampler_workspace_bytes(N), "sampler_prepare_count: workspace too small");
  const float2* src = (const float2*)device_view(traj);
  DTK_CHECK_ARG(src, "sampler_prepare_count: trajectories must be in device or pinned host memory");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = cdiv(N, SMP_THREADS);
  Arena ar(workspace);
  const SamplerWs w(ar, N);
  {
    ProfRange pr(PROF_SAMPLER, st);
    sampler_prepare_count_kernel<<<nb, SMP_THREADS, 0, st>>>(src, N, T, w.cnt);
    DTK_LAUNCHED();
    if (int rc = launch_count_scan(w.cnt, nb, 1, w.off, w.total, st)) return rc;
  }
  return read_total(w, n_valid, st);
}

int dinotrk_sampler_prepare_emit(const float* traj, int N, int T, float* rows, uint32_t* bits, void* workspace,
                                 size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(traj && rows && bits && workspace && N > 0 && T > 0 && T <= SMP_MAX_T,
                "sampler_prepare_emit: bad arguments (N = %d, T = %d)", N, T);
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_sampler_workspace_bytes(N), "sampler_prepare_emit: workspace too small");
  const float2* src = (const float2*)device_view(traj);
  float2* dst = (float2*)device_view(rows);
  uint32_t* b = (uint32_t*)device_view(bits);
  DTK_CHECK_ARG(src && dst && b, "sampler_prepare_emit: buffers must be in device or pinned host memory");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = cdiv(N, SMP_THREADS);
  Arena ar(workspace);
  const SamplerWs w(ar, N);
  ProfRange pr(PROF_SAMPLER, st);
  sampler_prepare_emit_kernel<<<nb, SMP_THREADS, 0, st>>>(src, N, T, w.off, dst, b);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_sampler_count(const uint32_t* bits, int N, int T, const int64_t* frames, int n_frames, int* n_cand,
                          void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(bits && frames && n_cand && workspace && N > 0 && T > 0 && T <= SMP_MAX_T && n_frames > 0 && n_frames <= T,
                "sampler_count: bad arguments (N = %d, T = %d, frames = %d)", N, T, n_frames);
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_sampler_workspace_bytes(N), "sampler_count: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = cdiv(N, SMP_THREADS);
  Arena ar(workspace);
  const SamplerWs w(ar, N);
  {
    ProfRange pr(PROF_SAMPLER, st);
    sampler_count_kernel<<<nb, SMP_THREADS, smp_words(T) * 4, st>>>(bits, N, T, frames, n_frames, w.cnt);
    DTK_LAUNCHED();
    if (int rc = launch_count_scan(w.cnt, nb, 1, w.off, w.total, st)) return rc;
  }
  return read_total(w, n_cand, st);
}

int dinotrk_sampler_select(const uint32_t* bits, int N, int T, const int64_t* frames, int n_frames, const int64_t* perm,
                           int m, int64_t* row_ids, float* mat, void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(bits && frames && perm && row_ids && mat && workspace && N > 0 && T > 0 && T <= SMP_MAX_T &&
                n_frames > 0 && n_frames <= T && m > 0 && m <= N,
                "sampler_select: bad arguments (N = %d, T = %d, frames = %d, m = %d)", N, T, n_frames, m);
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_sampler_workspace_bytes(N), "sampler_select: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = cdiv(N, SMP_THREADS);
  Arena ar(workspace);
  const SamplerWs w(ar, N);
  ProfRange pr(PROF_SAMPLER, st);
  sampler_select_kernel<<<cdiv(m, SEL_WARPS), SEL_WARPS * 32, smp_words(T) * 4, st>>>(bits, N, T, frames, n_frames, w.off,
                                                                                      nb, perm, m, row_ids, mat);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_sampler_gather(const float* rows, int T, const int64_t* row_ids, const int64_t* draws, int m, float* t1,
                           float* t2, void* stream) {
  DTK_CHECK_ARG(rows && row_ids && draws && t1 && t2 && T > 0 && T <= SMP_MAX_T && m > 0,
                "sampler_gather: bad arguments (T = %d, m = %d)", T, m);
  const float2* src = (const float2*)device_view(rows);
  DTK_CHECK_ARG(src, "sampler_gather: rows must be in device or pinned host memory");
  cudaStream_t st = (cudaStream_t)stream;
  ProfRange pr(PROF_SAMPLER, st);
  sampler_gather_kernel<<<cdiv(2 * m, 256), 256, 0, st>>>(src, T, row_ids, draws, m, t1, t2);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // extern "C"

// Shared helpers for libdinotrk (sm_90a).  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include <string.h>

#include <type_traits>

#include <nvtx3/nvToolsExt.h>   // header-only; ranges cost nothing unless a profiler injects itself

#include "dinotrk.h"

namespace dtk {

void set_error(const char* fmt, ...);
extern unsigned long long g_launches;

#define DTK_CHECK_ARG(cond, ...)              \
  do {                                        \
    if (!(cond)) {                            \
      dtk::set_error(__VA_ARGS__);            \
      return DINOTRK_EINVAL;                  \
    }                                         \
  } while (0)

// Supported token grids of the tracker's entry points (head, inference, training backward): h <= 256, w <= 256 and
// h * w <= 32,768 (1274 x 1274 px at patch 14 / stride 7).  Shared-memory map buffers and per-map key arrays are sized
// for it.
constexpr int DTK_GRID_MAX_SIDE = 256, DTK_GRID_MAX_TOKENS = 32768;
#define DTK_CHECK_GRID(g, what)                                                                                          \
  DTK_CHECK_ARG((g).h > 0 && (g).w > 0 && (g).h <= dtk::DTK_GRID_MAX_SIDE && (g).w <= dtk::DTK_GRID_MAX_SIDE &&          \
                    (g).h * (g).w <= dtk::DTK_GRID_MAX_TOKENS,                                                           \
                "%s: token grid %d x %d outside the supported envelope (h, w <= %d, h * w <= %d tokens)", what, (g).h,  \
                (g).w, dtk::DTK_GRID_MAX_SIDE, dtk::DTK_GRID_MAX_TOKENS)

#define DTK_CUDA(call)                                                              \
  do {                                                                              \
    cudaError_t e__ = (call);                                                       \
    if (e__ != cudaSuccess) {                                                       \
      dtk::set_error("%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e__)); \
      return DINOTRK_ECUDA;                                                         \
    }                                                                               \
  } while (0)

// count + check a kernel launch
#define DTK_LAUNCHED()                 \
  do {                                 \
    ++dtk::g_launches;                 \
    DTK_CUDA(cudaPeekAtLastError());   \
  } while (0)

// ---- optional per-kernel-class timing with CUDA events on the launching stream (bench.py roofline) ----
enum ProfClass {
  PROF_SAMPLE = 0, PROF_CORR_GEMM, PROF_CORR_STREAM, PROF_HEAD, PROF_COS, PROF_ANCHOR_LIST, PROF_OCCLUSION,
  PROF_PACK, PROF_CONV, PROF_BLUR, PROF_ALIGN, PROF_MISC, PROF_BB, PROF_VIT_GEMM, PROF_VIT_ATTN, PROF_VIT_MISC, PROF_HEAD_FULL,
  PROF_XW_COARSE, PROF_XW_PLAN, PROF_XW_GEMM, PROF_XW_HEAD, PROF_TRAIN_BWD,
  PROF_DELTA_TRAIN_CONV, PROF_DELTA_BN, PROF_DELTA_DGRAD, PROF_DELTA_WGRAD, PROF_FG_MASK, PROF_CONTRASTIVE,
  PROF_SAMPLER, PROF_CYCLE, PROF_EMB_REG, PROF_COUNT
};
extern bool g_prof_on;
void prof_begin(int cls, cudaStream_t st);
void prof_end(cudaStream_t st);
// ranges do not nest; a negative class records nothing (for code that runs inside the caller's range)
struct ProfRange {
  cudaStream_t st;
  bool on;
  ProfRange(int cls, cudaStream_t s) : st(s), on(g_prof_on && cls >= 0) { if (on) prof_begin(cls, st); }
  ~ProfRange() { if (on) prof_end(st); }
};

// per-device cache slot for values that belong to a device's context (function attributes, occupancy queries,
// auxiliary streams): indexed by the CURRENT device, so a second GPU in the same process gets its own
constexpr int DTK_MAX_DEVICES = 64;
template <typename T>
struct PerDev {
  T v[DTK_MAX_DEVICES] = {};
  T& get() {
    int d = 0;
    cudaGetDevice(&d);
    return v[(d >= 0 && d < DTK_MAX_DEVICES) ? d : 0];
  }
};

// NVTX range over a host-side phase (nsys / ncu --nvtx): the four phases of dinotrk_infer, the ViT and delta-DINO stages
struct NvtxRange {
  explicit NvtxRange(const char* name) { nvtxRangePushA(name); }
  ~NvtxRange() { nvtxRangePop(); }
};

// multiprocessors of the current device (cached per device; corr_tc.cu)
int num_sms();

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }
static inline int cdiv(int a, int b) { return (a + b - 1) / b; }

// bump allocator over a caller-provided workspace
struct Arena {
  char* base;
  size_t off;
  explicit Arena(void* p) : base((char*)p), off(0) {}
  template <typename T>
  T* take(size_t count) {
    off = align_up(off, 256);
    T* p = (T*)(base + off);
    off += count * sizeof(T);
    return p;
  }
};

// A workspace's layout is a struct whose constructor takes every buffer from an Arena.  Its size function is a dry run of
// that constructor on a null base, so the size and the carve cannot disagree: this returns where the last buffer ends.
template <typename Layout, typename... Args>
static inline size_t layout_end(const Args&... args) {
  Arena ar(nullptr);
  const Layout layout(ar, args...);
  (void)layout;
  return ar.off;
}

// element-wise IEEE fp32 operations on pairs (two FFMA / FMUL / FADD: bit for bit what a packed instruction would give)
__device__ __forceinline__ float2 f2fma(float2 a, float2 b, float2 c) { return make_float2(__fmaf_rn(a.x, b.x, c.x), __fmaf_rn(a.y, b.y, c.y)); }
__device__ __forceinline__ float2 f2mul(float2 a, float2 b) { return make_float2(__fmul_rn(a.x, b.x), __fmul_rn(a.y, b.y)); }
__device__ __forceinline__ float2 f2add(float2 a, float2 b) { return make_float2(__fadd_rn(a.x, b.x), __fadd_rn(a.y, b.y)); }

__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
  return v;
}

// ---- compaction: count per block (__syncthreads_count), scan the block counts, then emit or select by rank ----------
// The largest k in [0, n) with key(k) <= x, or 0 if there is none; key (an array or a functor) is ascending.
template <typename K>
__device__ __forceinline__ int last_le(int n, int x, K key) {
  int lo = 0, hi = n - 1;
  while (lo < hi) {
    const int mid = (lo + hi + 1) >> 1;
    int k;
    if constexpr (std::is_pointer<K>::value) k = key[mid]; else k = key(mid);
    if (k <= x) lo = mid; else hi = mid - 1;
  }
  return lo;
}

// The exclusive rank of this thread's pred among the block's THREADS threads in thread order; *total = the block's
// count.  One barrier, so every thread of the block calls it; a loop over it needs a barrier before the next call.
template <int THREADS>
__device__ __forceinline__ int block_rank(bool pred, int* total = nullptr) {
  __shared__ int s_warp[THREADS / 32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const unsigned ball = __ballot_sync(0xffffffffu, pred);
  if (lane == 0) s_warp[warp] = __popc(ball);
  __syncthreads();
  int rank = __popc(ball & ((1u << lane) - 1u)), sum = 0;
#pragma unroll
  for (int k = 0; k < THREADS / 32; ++k) { rank += k < warp ? s_warp[k] : 0; sum += s_warp[k]; }
  if (total) *total = sum;
  return rank;
}

// The index of the n-th (from 0) i in [begin, end) with hit(i), or -1 if there is none.  The whole warp calls it with
// the same arguments and tests 32 indices at a time.
template <typename F>
__device__ __forceinline__ int warp_nth_hit(int begin, int end, int n, F hit) {
  const int lane = threadIdx.x & 31;
  for (int base = begin; base < end; base += 32) {
    const bool h = base + lane < end && hit(base + lane);
    const unsigned ball = __ballot_sync(0xffffffffu, h);
    if (n < __popc(ball)) {
      const unsigned sel = __ballot_sync(0xffffffffu, h && __popc(ball & ((1u << lane) - 1u)) == n);
      return base + __ffs(sel) - 1;
    }
    n -= __popc(ball);
  }
  return -1;
}

// Exclusive scan of `rows` count arrays of nb entries, one block each (features.cu): row r scans cnt + r * nb into
// off + r * nb and writes its sum to total[r].
int launch_count_scan(const int* cnt, int nb, int rows, int* off, int* total, cudaStream_t stream);

// ---- exact restatement of the reference's coordinate arithmetic ---------------------------
// models/tracker.py:84-93: a, b are computed in Python doubles and stored as fp32.
struct PointAffine {
  float aw, ah, bw, bh;
};
static inline PointAffine make_point_affine(const dinotrk_geom& g) {
  double p = g.patch, s = g.stride;
  double last_h = double((g.H - g.patch) / g.stride) * s + p / 2;
  double last_w = double((g.W - g.patch) / g.stride) * s + p / 2;
  PointAffine a;
  a.ah = (float)(2.0 / (last_h - p / 2));
  a.aw = (float)(2.0 / (last_w - p / 2));
  a.bh = (float)(1.0 - last_h * 2.0 / (last_h - p / 2));
  a.bw = (float)(1.0 - last_w * 2.0 / (last_w - p / 2));
  return a;
}

// ATen grid_sampler (align_corners=True, padding_mode=border): unnormalise then clip.
__device__ __forceinline__ float gs_unnorm_clip(float coord, int size) {
  float x = __fmul_rn(__fdiv_rn(__fadd_rn(coord, 1.f), 2.f), (float)(size - 1));
  return fminf(fmaxf(x, 0.f), (float)(size - 1));
}

// Trilinear sampling set-up for one point: 8 corners in ATen order
// (tnw, tne, tsw, tse, bnw, bne, bsw, bse) -> token index, set slot (z) and weight; weight 0 and
// token -1 for corners ATen skips as out of bounds.
struct TriCorners {
  int tok[4];     // (x0,y0) (x1,y0) (x0,y1) (x1,y1); -1 if out of bounds
  float wxy[4][2];  // [corner][z0|z1] full 3-factor weights in ATen's multiplication order
  int z0, z1;     // set slots; -1 if out of bounds
};
__device__ __forceinline__ TriCorners tri_setup(float xn, float yn, float set_idx, int N, int h, int w) {
  // utils.py:96-99: idx / (N-1) (skipped when N == 1), * 2 - 1
  float tn = set_idx;
  if (N > 1) tn = __fdiv_rn(tn, (float)(N - 1));
  tn = __fadd_rn(__fmul_rn(tn, 2.f), -1.f);
  float ix = gs_unnorm_clip(xn, w), iy = gs_unnorm_clip(yn, h), iz = gs_unnorm_clip(tn, N);
  float x0 = floorf(ix), y0 = floorf(iy), z0 = floorf(iz);
  float x1 = x0 + 1.f, y1 = y0 + 1.f, z1 = z0 + 1.f;
  float wx0 = __fsub_rn(x1, ix), wx1 = __fsub_rn(ix, x0);
  float wy0 = __fsub_rn(y1, iy), wy1 = __fsub_rn(iy, y0);
  float wz0 = __fsub_rn(z1, iz), wz1 = __fsub_rn(iz, z0);
  TriCorners c;
  int X0 = (int)x0, Y0 = (int)y0, X1 = X0 + 1, Y1 = Y0 + 1;
  bool okx1 = X1 <= w - 1, oky1 = Y1 <= h - 1;
  c.tok[0] = Y0 * w + X0;
  c.tok[1] = okx1 ? Y0 * w + X1 : -1;
  c.tok[2] = oky1 ? Y1 * w + X0 : -1;
  c.tok[3] = (okx1 && oky1) ? Y1 * w + X1 : -1;
  float wx[4] = {wx0, wx1, wx0, wx1};
  float wy[4] = {wy0, wy0, wy1, wy1};
#pragma unroll
  for (int k = 0; k < 4; ++k) {
    c.wxy[k][0] = __fmul_rn(__fmul_rn(wx[k], wy[k]), wz0);
    c.wxy[k][1] = __fmul_rn(__fmul_rn(wx[k], wy[k]), wz1);
  }
  c.z0 = (int)z0;
  c.z1 = ((int)z0 + 1 <= N - 1) ? (int)z0 + 1 : -1;
  return c;
}

}  // namespace dtk

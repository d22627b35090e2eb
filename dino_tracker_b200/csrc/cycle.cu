// The cycle-consistency term of the training step (models/tracker.py:182-301, dino_tracker.py:346-353).
//
// The reference draws, per (source, target) pair of the frame set, a host randperm over the source frame's foreground
// pixels and one over its background pixels, keeps the first 179 / 77 of each, tracks them source -> target -> source
// and keeps the points that return within cyc_thresh px.  Here:
//   * dinotrk_randperm_prefix (host) writes the first k entries of torch's CPU randperm(n) in O(k) and advances the
//     generator past the n - 1 draws randperm makes, without tempering them;
//   * mask_count / scan (once per mask set) give per-frame, per-block foreground counts in row-major pixel order, and
//     cycle_select maps each drawn rank to its pixel (binary search over the block scan, ballot rank in the block);
//   * both legs of all pairs run as one batch each on the tracker's kernels; cycle_unnorm turns the first leg's output
//     into the second leg's input and cycle_keep applies the reference's fp32 distance test and compacts the survivors.
#include <math.h>

#include <unordered_map>

#include "common.cuh"

namespace dtk {

constexpr int CYC_THREADS = 256;   // pixels per count block
constexpr int CYC_SEL_WARPS = 8;
constexpr int CYC_KEEP_THREADS = 1024;

// ---- host: torch's CPU randperm (aten/src/ATen/native/TensorFactories.cpp randperm_cpu, n < 2^32 / 20) -------------
// The generator is mt19937 as at::mt19937 keeps it: `left` draws until the next twist, `next` the index of the next
// state word.  A draw: if (--left == 0) { twist; left = 624; next = 0; } y = temper(state[next++]).
constexpr int MT_N = 624, MT_M = 397;
struct Mt {
  uint32_t s[MT_N];
  int32_t left;
  uint64_t next;
  static uint32_t mix(uint32_t u, uint32_t v, uint32_t far) {
    const uint32_t y = (u & 0x80000000u) | (v & 0x7fffffffu);
    return far ^ (y >> 1) ^ ((0u - (y & 1u)) & 0x9908b0dfu);
  }
  // the in-place twist, split at the wrap-arounds (skipping a large randperm is ~n / 624 of these)
  void twist() {
    int i = 0;
    for (; i < MT_N - MT_M; ++i) s[i] = mix(s[i], s[i + 1], s[i + MT_M]);
    for (; i < MT_N - 1; ++i) s[i] = mix(s[i], s[i + 1], s[i + MT_M - MT_N]);
    s[MT_N - 1] = mix(s[MT_N - 1], s[0], s[MT_M - 1]);
    left = MT_N;
    next = 0;
  }
  uint32_t draw() {
    if (--left == 0) twist();
    uint32_t y = s[next++];
    y ^= y >> 11;
    y ^= (y << 7) & 0x9d2c5680u;
    y ^= (y << 15) & 0xefc60000u;
    y ^= y >> 18;
    return y;
  }
  // m draws whose values are not needed: only the twists and the bookkeeping
  void skip(uint64_t m) {
    while (m > 0) {
      if (left > 1) {
        const uint64_t step = m < (uint64_t)(left - 1) ? m : (uint64_t)(left - 1);
        left -= (int32_t)step;
        next += step;
        m -= step;
      } else {
        twist();
        next = 1;
        --m;
      }
    }
  }
};

// CPUGeneratorImpl::get_state(): seed u64, left i32, seeded i32, next u64, state[624] as u64, then the normal-sampling
// cache this helper leaves alone
constexpr size_t RNG_LEFT = 8, RNG_NEXT = 16, RNG_STATE = 24;

// ---- device: pixel draws ------------------------------------------------------------------------------------------
// cnt[t][b] = foreground pixels (fg[t][p] != 0) of block b of frame t
__global__ void __launch_bounds__(CYC_THREADS)
cycle_mask_count_kernel(const uint8_t* __restrict__ fg, int P, int nb, int* __restrict__ cnt) {
  const int t = blockIdx.y, p = blockIdx.x * CYC_THREADS + threadIdx.x;
  const int c = __syncthreads_count(p < P && fg[(size_t)t * P + p] != 0);
  if (threadIdx.x == 0) cnt[(size_t)t * nb + blockIdx.x] = c;
}

// Row i of a draw: rows[i] = {t_src, is_fg, rank, src_slot, tgt_slot, t_tgt, there_pos, back_pos}.  One warp per row:
// the pixel is the rank-th foreground (or background) pixel of frame t_src in row-major order.  Writes start[i] =
// (x, y, t_src) and the first leg's input there_pts[there_pos] = (x, y, src_slot).
__global__ void __launch_bounds__(CYC_SEL_WARPS * 32)
cycle_select_kernel(const uint8_t* __restrict__ fg, int W, int P, int nb, const int* __restrict__ off,
                    const int* __restrict__ rows, int R, float* __restrict__ start, float* __restrict__ there_pts) {
  const int lane = threadIdx.x & 31, i = blockIdx.x * CYC_SEL_WARPS + (threadIdx.x >> 5);
  if (i >= R) return;
  const int* r = rows + (size_t)i * 8;
  const int t = r[0], want = r[1];
  const int* o = off + (size_t)t * nb;
  const uint8_t* m = fg + (size_t)t * P;
  // pixels of the wanted kind before block b: off[b] (foreground) or b * CYC_THREADS - off[b] (background)
  auto before = [&](int b) { return want ? o[b] : b * CYC_THREADS - o[b]; };
  const int b = last_le(nb, r[2], before);
  const int pix = warp_nth_hit(b * CYC_THREADS, min(b * CYC_THREADS + CYC_THREADS, P), r[2] - before(b),
                               [&](int p) { return (m[p] != 0) == (want != 0); });
  if (lane != 0) return;
  // the host draws ranks below the frame's count, so pix >= 0
  const float x = (float)(pix % W), y = (float)(pix / W);
  float* s = start + (size_t)i * 3;
  s[0] = x; s[1] = y; s[2] = (float)t;
  float* q = there_pts + (size_t)r[6] * 3;
  q[0] = x; q[1] = y; q[2] = (float)r[3];
}

// RangeNormalizer.unnormalize(c, src=(-1, 1), dims=[0, 1]) in its fp32 op order: (c + 1) / 2 * (size - 1)
__device__ __forceinline__ float unnorm(float c, float size_m1) {
  return __fmul_rn(__fdiv_rn(__fadd_rn(c, 1.f), 2.f), size_m1);
}

// First leg's output there_out[i] (normalised, reference row order) -> there_px[i] = (x_px, y_px, t_tgt) and the second
// leg's input back_pts[back_pos] = (x_px, y_px, tgt_slot)
__global__ void cycle_unnorm_kernel(const float* __restrict__ there_out, const int* __restrict__ rows, int R, float w_m1,
                                    float h_m1, float* __restrict__ there_px, float* __restrict__ back_pts) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= R) return;
  const int* r = rows + (size_t)i * 8;
  const float x = unnorm(there_out[2 * i], w_m1), y = unnorm(there_out[2 * i + 1], h_m1);
  float* a = there_px + (size_t)i * 3;
  a[0] = x; a[1] = y; a[2] = (float)r[5];
  float* b = back_pts + (size_t)r[7] * 3;
  b[0] = x; b[1] = y; b[2] = (float)r[4];
}

// keep[i] = torch.norm(start[i, :2] - back_px[i], dim=1) <= thresh as the reference evaluates it on the device: the
// difference, then each square rounded, their sum, a correctly rounded sqrt.  One block; survivors in row order:
// keep_rows[k] = i, cycle_px[k] = back_px[i], *n_keep = their number.
__global__ void __launch_bounds__(CYC_KEEP_THREADS)
cycle_keep_kernel(const float* __restrict__ start, const float* __restrict__ back_out, int R, float w_m1, float h_m1,
                  float thresh, int* __restrict__ keep_rows, float* __restrict__ cycle_px, int* __restrict__ n_keep) {
  int base = 0;
  for (int i0 = 0; i0 < R; i0 += CYC_KEEP_THREADS) {
    const int i = i0 + threadIdx.x;
    bool keep = false;
    float bx = 0.f, by = 0.f;
    if (i < R) {
      bx = unnorm(back_out[2 * i], w_m1);
      by = unnorm(back_out[2 * i + 1], h_m1);
      const float dx = __fsub_rn(start[3 * i], bx), dy = __fsub_rn(start[3 * i + 1], by);
      keep = __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy))) <= thresh;
    }
    int total;
    const int k = base + block_rank<CYC_KEEP_THREADS>(keep, &total);
    if (keep) {
      keep_rows[k] = i;
      cycle_px[2 * k] = bx;
      cycle_px[2 * k + 1] = by;
    }
    base += total;
    __syncthreads();   // the next chunk's block_rank rewrites the warp counts
  }
  if (threadIdx.x == 0) *n_keep = base;
}

struct CycleMaskWs {
  int* cnt;   // [T][cdiv(P, CYC_THREADS)] foreground pixels per block
  CycleMaskWs(Arena& ar, int T, int P) { cnt = ar.take<int>((size_t)T * cdiv(P, CYC_THREADS)); }
};

}  // namespace dtk

using namespace dtk;

extern "C" {

int dinotrk_randperm_prefix(uint8_t* state, size_t state_bytes, int64_t n, int64_t k, int64_t* out) {
  DTK_CHECK_ARG(state && state_bytes == DINOTRK_CPU_RNG_STATE_BYTES,
                "randperm_prefix: generator state of %zu bytes (expected %d)", state_bytes, DINOTRK_CPU_RNG_STATE_BYTES);
  DTK_CHECK_ARG(n >= 0 && n < (int64_t)(UINT32_MAX / 20) && k >= 0 && (out || k == 0 || n == 0),
                "randperm_prefix: bad arguments (n = %lld, k = %lld)", (long long)n, (long long)k);
  Mt mt;
  int32_t left;
  uint64_t next;
  memcpy(&left, state + RNG_LEFT, 4);
  memcpy(&next, state + RNG_NEXT, 8);
  DTK_CHECK_ARG(left >= 1 && left <= MT_N && next <= (uint64_t)MT_N, "randperm_prefix: corrupt generator state");
  mt.left = left;
  mt.next = next;
  for (int i = 0; i < MT_N; ++i) {
    uint64_t v;
    memcpy(&v, state + RNG_STATE + 8 * (size_t)i, 8);
    mt.s[i] = (uint32_t)v;
  }
  // forward Fisher-Yates: step i swaps positions i and i + z; position i is final after step i.  `moved` holds the
  // values of the positions a swap displaced (every other position still holds its own index).
  const int64_t draws = n > 0 ? n - 1 : 0, kk = k < n ? k : n, steps = kk < draws ? kk : draws;
  std::unordered_map<int64_t, int64_t> moved;
  moved.reserve((size_t)steps * 2);
  auto value = [&](int64_t p) {
    auto it = moved.find(p);
    return it == moved.end() ? p : it->second;
  };
  for (int64_t i = 0; i < steps; ++i) {
    const int64_t j = i + (int64_t)(mt.draw() % (uint64_t)(n - i));
    const int64_t vi = value(i);
    out[i] = value(j);
    moved[j] = vi;
  }
  if (kk > steps) out[kk - 1] = value(kk - 1);   // the whole permutation: its last entry takes no draw
  mt.skip((uint64_t)(draws - steps));
  memcpy(state + RNG_LEFT, &mt.left, 4);
  memcpy(state + RNG_NEXT, &mt.next, 8);
  for (int i = 0; i < MT_N; ++i) {
    const uint64_t v = mt.s[i];
    memcpy(state + RNG_STATE + 8 * (size_t)i, &v, 8);
  }
  return DINOTRK_OK;
}

size_t dinotrk_cycle_mask_workspace_bytes(int T, int P) {
  if (T <= 0 || P <= 0) return 0;
  return align_up(layout_end<CycleMaskWs>(T, P), 256);
}

int dinotrk_cycle_mask_scan(const uint8_t* fg, int T, int P, int* off, int* n_fg, void* workspace, size_t workspace_bytes,
                            void* stream) {
  DTK_CHECK_ARG(fg && off && n_fg && workspace && T > 0 && P > 0, "cycle_mask_scan: bad arguments (T = %d, P = %d)", T, P);
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_cycle_mask_workspace_bytes(T, P), "cycle_mask_scan: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const int nb = cdiv(P, CYC_THREADS);
  Arena ar(workspace);
  int* cnt = CycleMaskWs(ar, T, P).cnt;
  ProfRange pr(PROF_CYCLE, st);
  cycle_mask_count_kernel<<<dim3(nb, T), CYC_THREADS, 0, st>>>(fg, P, nb, cnt);
  DTK_LAUNCHED();
  return launch_count_scan(cnt, nb, T, off, n_fg, st);
}

int dinotrk_cycle_select(const uint8_t* fg, int T, int H, int W, const int* off, const int* rows, int R, float* start,
                         float* there_pts, void* stream) {
  DTK_CHECK_ARG(fg && off && rows && start && there_pts && T > 0 && H > 0 && W > 0 && R > 0,
                "cycle_select: bad arguments (T = %d, %d x %d, R = %d)", T, H, W, R);
  cudaStream_t st = (cudaStream_t)stream;
  const int P = H * W;
  ProfRange pr(PROF_CYCLE, st);
  cycle_select_kernel<<<cdiv(R, CYC_SEL_WARPS), CYC_SEL_WARPS * 32, 0, st>>>(fg, W, P, cdiv(P, CYC_THREADS), off, rows, R,
                                                                             start, there_pts);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_cycle_unnorm(const float* there_out, const int* rows, int R, int H, int W, float* there_px, float* back_pts,
                         void* stream) {
  DTK_CHECK_ARG(there_out && rows && there_px && back_pts && R > 0 && H > 1 && W > 1, "cycle_unnorm: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  ProfRange pr(PROF_CYCLE, st);
  cycle_unnorm_kernel<<<cdiv(R, 256), 256, 0, st>>>(there_out, rows, R, (float)(W - 1), (float)(H - 1), there_px, back_pts);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_cycle_keep(const float* start, const float* back_out, int R, int H, int W, float thresh, int* keep_rows,
                       float* cycle_px, int* n_keep, void* stream) {
  DTK_CHECK_ARG(start && back_out && keep_rows && cycle_px && n_keep && R > 0 && H > 1 && W > 1, "cycle_keep: bad arguments");
  cudaStream_t st = (cudaStream_t)stream;
  ProfRange pr(PROF_CYCLE, st);
  cycle_keep_kernel<<<1, CYC_KEEP_THREADS, 0, st>>>(start, back_out, R, (float)(W - 1), (float)(H - 1), thresh, keep_rows,
                                                     cycle_px, n_keep);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // extern "C"

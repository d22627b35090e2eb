// Optical-flow trajectories (preprocessing/extract_trajectories.py) and the optical-flow filter of the best buddies
// (preprocessing_dino_bb/of_filter_dino_best_buddies.py).  The flows come from the caller (RAFT stays outside the
// library); everything the reference does with them runs here.
//
// Chaining: the reference walks all h*w pixels of a start frame s through frames s..T-1 with ~15 tensor ops per step,
// copies the padded (h*w) x T x 2 block to the host and grows the result with torch.cat.  Here one thread walks one
// pixel in registers and stops at its first failed check (every check is cumulative: the trajectory is a valid prefix
// followed by NaN).  A second pass re-walks only the kept pixels (forward sampling only) and writes them, compacted in
// (row-major pixel) order, straight into the caller's [n][T][2] output; it also marks their rounded positions in a
// per-frame occupancy bitmap that later start frames read as the reference's look-behind.
#include <math.h>

#include "common.cuh"

namespace dtk {

constexpr int TRAJ_THREADS = 256;

// data/data_utils.py:62-76 bilinear_sampler (grid_sample, bilinear, zeros padding, align_corners=True) of one
// [2][H][W] flow at pixel (x, y): the grid is normalised as 2*x/(W-1) - 1 in fp32 and unnormalised as ATen does,
// ((g + 1) / 2) * (size - 1); corner weights and the accumulation order are ATen's (nw, ne, sw, se).  A tensor divided
// by a Python number on CUDA is multiplied by the fp32 reciprocal (ATen div_true_kernel_cuda); so is this one, since the
// reference runs on CUDA.  (The CPU divides; for W - 1 a power of two both are exact.)
__device__ __forceinline__ float2 flow_at(const float* __restrict__ f, int H, int W, float x, float y) {
  const float gx = __fsub_rn(__fmul_rn(__fmul_rn(2.f, x), __frcp_rn((float)(W - 1))), 1.f);
  const float gy = __fsub_rn(__fmul_rn(__fmul_rn(2.f, y), __frcp_rn((float)(H - 1))), 1.f);
  const float ix = __fmul_rn(__fdiv_rn(__fadd_rn(gx, 1.f), 2.f), (float)(W - 1));
  const float iy = __fmul_rn(__fdiv_rn(__fadd_rn(gy, 1.f), 2.f), (float)(H - 1));
  float2 acc = make_float2(0.f, 0.f);
  // no corner in bounds (also NaN): ATen adds nothing
  if (!(ix >= -1.f && ix < (float)W && iy >= -1.f && iy < (float)H)) return acc;
  const float x0 = floorf(ix), y0 = floorf(iy), x1 = x0 + 1.f, y1 = y0 + 1.f;
  const int X0 = (int)x0, Y0 = (int)y0, X1 = X0 + 1, Y1 = Y0 + 1;
  const float nw = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(y1, iy));
  const float ne = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(y1, iy));
  const float sw = __fmul_rn(__fsub_rn(x1, ix), __fsub_rn(iy, y0));
  const float se = __fmul_rn(__fsub_rn(ix, x0), __fsub_rn(iy, y0));
  const size_t plane = (size_t)H * W;
  auto add = [&](int X, int Y, float wt) {
    if (X >= 0 && X < W && Y >= 0 && Y < H) {
      const size_t o = (size_t)Y * W + X;
      acc.x = fmaf(__ldg(f + o), wt, acc.x);
      acc.y = fmaf(__ldg(f + plane + o), wt, acc.y);
    }
  };
  add(X0, Y0, nw);
  add(X1, Y0, ne);
  add(X0, Y1, sw);
  add(X1, Y1, se);
  return acc;
}

// torch.norm of a 2-vector as the reference evaluates it, without contraction: sqrt(dx*dx + dy*dy)
__device__ __forceinline__ float norm2(float dx, float dy) {
  return __fsqrt_rn(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
}

// ---- extract_trajectories.py:61-95 get_flows_with_masks ------------------------------------------------------------
// masks[i + 1][q] = 1 where some pixel of frame i lands on q (rounded forward warp, in bounds).  masks is zeroed first.
__global__ void flow_cover_kernel(const float* __restrict__ fwd, int T, int H, int W, uint8_t* __restrict__ masks) {
  const size_t P = (size_t)H * W, i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)(T - 1) * P) return;
  const size_t pair = i / P, q = i - pair * P;
  const float* f = fwd + pair * 2 * P;
  const float gx = rintf(__fadd_rn((float)(q % W), f[q])), gy = rintf(__fadd_rn((float)(q / W), f[P + q]));
  if (gx >= 0.f && gx <= (float)(W - 1) && gy >= 0.f && gy <= (float)(H - 1))
    masks[(pair + 1) * P + (size_t)gy * W + (size_t)gx] = 1;
}

// masks[i + 1][q] &= |c - (c + b + F(c + b))| < threshold, with b the backward flow of pair i at q and F its forward
// flow sampled at c + b (the round trip frame i+1 -> i -> i+1).
__global__ void flow_consistency_kernel(const float* __restrict__ fwd, const float* __restrict__ bwd, int T, int H, int W,
                                        float threshold, uint8_t* __restrict__ masks) {
  const size_t P = (size_t)H * W, i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)(T - 1) * P) return;
  const size_t pair = i / P, q = i - pair * P;
  const float cx = (float)(q % W), cy = (float)(q / W);
  const float c1x = __fadd_rn(cx, bwd[pair * 2 * P + q]), c1y = __fadd_rn(cy, bwd[pair * 2 * P + P + q]);
  const float2 w = flow_at(fwd + pair * 2 * P, H, W, c1x, c1y);
  const float err = norm2(__fsub_rn(cx, __fadd_rn(c1x, w.x)), __fsub_rn(cy, __fadd_rn(c1y, w.y)));
  uint8_t& m = masks[(pair + 1) * P + q];
  m = (m && err < threshold) ? 1 : 0;
}

// ---- extract_trajectories.py:203-266 chaining of one start frame s -------------------------------------------------
struct ChainArgs {
  const float* fwd;    // [T-1][2][H][W]
  const float* bwd;
  const float* dfwd;   // [T-1-s][2][H][W] direct flows s -> s+1+k, or null
  const float* dbwd;   // [T-1-s][2][H][W] direct flows s+1+k -> s
  const uint8_t* masks;
  int T, H, W, s, min_len;
  float threshold, direct_threshold;
};

// The direct-flow check of step k for the walk started at pixel (x0, y0) at position (cx, cy) after the step
// (extract_trajectories.py:98-160 for the mask, :234-255 for its use).  The backward direct flow is sampled through
// utils.bilinear_interpolate_video: the 5-D grid_sample (border, align_corners) of the (T-1-s)-frame volume at
// (x / (W-1) * 2 - 1, y / (H-1) * 2 - 1, k / (T-2-s) * 2 - 1), including its fp32 temporal-weight leak.
__device__ __forceinline__ bool direct_ok(const ChainArgs& a, int k, float x0, float y0, size_t p, float cx, float cy) {
  const int D = a.T - 1 - a.s;
  const size_t P = (size_t)a.H * a.W;
  const float d1x = __fadd_rn(x0, __ldg(a.dfwd + (size_t)k * 2 * P + p));
  const float d1y = __fadd_rn(y0, __ldg(a.dfwd + (size_t)k * 2 * P + P + p));
  const float xn = __fsub_rn(__fmul_rn(__fmul_rn(d1x, __frcp_rn((float)(a.W - 1))), 2.f), 1.f);
  const float yn = __fsub_rn(__fmul_rn(__fmul_rn(d1y, __frcp_rn((float)(a.H - 1))), 2.f), 1.f);
  const TriCorners c = tri_setup(xn, yn, (float)k, D, a.H, a.W);
  float bx = 0.f, by = 0.f;
#pragma unroll
  for (int z = 0; z < 2; ++z) {
    const int f = z == 0 ? c.z0 : c.z1;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      if (f >= 0 && c.tok[j] >= 0) {
        const size_t o = (size_t)f * 2 * P + c.tok[j];
        bx = fmaf(__ldg(a.dbwd + o), c.wxy[j][z], bx);
        by = fmaf(__ldg(a.dbwd + o + P), c.wxy[j][z], by);
      }
    }
  }
  const float err = norm2(__fsub_rn(x0, __fadd_rn(d1x, bx)), __fsub_rn(y0, __fadd_rn(d1y, by)));
  const bool reliable = err < a.threshold && d1x >= 0.f && d1x <= (float)(a.W - 1) && d1y >= 0.f && d1y <= (float)(a.H - 1);
  const float e = __fmul_rn(norm2(__fsub_rn(cx, d1x), __fsub_rn(cy, d1y)), reliable ? 1.f : 0.f);
  return e < a.direct_threshold;
}

// len[p] = number of valid frames of the trajectory started at pixel p (0 when it does not start or is shorter than
// min_len); block_cnt[b] = kept pixels of block b.
__global__ void __launch_bounds__(TRAJ_THREADS)
traj_chain_kernel(ChainArgs a, const uint8_t* __restrict__ occ, int* __restrict__ len, int* __restrict__ block_cnt) {
  const size_t P = (size_t)a.H * a.W, p = (size_t)blockIdx.x * TRAJ_THREADS + threadIdx.x;
  int L = 0;
  // start where the flow from the previous frame is not consistent, or where no kept trajectory passes (look-behind)
  if (p < P && (!a.masks[(size_t)a.s * P + p] || !occ[(size_t)a.s * P + p])) {
    const float x0 = (float)(p % a.W), y0 = (float)(p / a.W);
    float cx = x0, cy = y0;
    L = 1;
    for (int k = 0; k < a.T - 1 - a.s; ++k) {
      const size_t f = (size_t)(a.s + k) * 2 * P;
      const float2 w12 = flow_at(a.fwd + f, a.H, a.W, cx, cy);
      const float c1x = __fadd_rn(cx, w12.x), c1y = __fadd_rn(cy, w12.y);
      const float2 w21 = flow_at(a.bwd + f, a.H, a.W, c1x, c1y);
      const float err = norm2(__fsub_rn(cx, __fadd_rn(c1x, w21.x)), __fsub_rn(cy, __fadd_rn(c1y, w21.y)));
      bool ok = err < a.threshold && c1x <= (float)(a.W - 1) && c1y <= (float)(a.H - 1) && c1x >= 0.f && c1y >= 0.f;
      cx = c1x;
      cy = c1y;
      if (ok && a.dfwd != nullptr) ok = direct_ok(a, k, x0, y0, p, cx, cy);
      if (!ok) break;
      ++L;
    }
    if (L < a.min_len) L = 0;
  }
  if (p < P) len[p] = L;
  const int n = __syncthreads_count(L > 0);
  if (threadIdx.x == 0) block_cnt[blockIdx.x] = n;
}

// Kept pixel p of block b -> out row off[b] + (rank of p among the block's kept pixels): NaN before s, the walk's
// positions on [s, s + len), NaN after; marks occ[t][round(y)][round(x)] for t in (s, s + len).
__global__ void __launch_bounds__(TRAJ_THREADS)
traj_emit_kernel(const float* __restrict__ fwd, int T, int H, int W, int s, const int* __restrict__ len,
                 const int* __restrict__ off, uint8_t* __restrict__ occ, float* __restrict__ out) {
  const size_t P = (size_t)H * W, p = (size_t)blockIdx.x * TRAJ_THREADS + threadIdx.x;
  const int L = p < P ? len[p] : 0;
  const int rank = block_rank<TRAJ_THREADS>(L > 0);
  if (L == 0) return;
  float2* row = reinterpret_cast<float2*>(out) + (size_t)(off[blockIdx.x] + rank) * T;
  const float2 nan2 = make_float2(NAN, NAN);
  for (int t = 0; t < s; ++t) row[t] = nan2;
  float cx = (float)(p % W), cy = (float)(p / W);
  row[s] = make_float2(cx, cy);
  for (int k = 1; k < L; ++k) {
    const float2 w = flow_at(fwd + (size_t)(s + k - 1) * 2 * P, H, W, cx, cy);
    cx = __fadd_rn(cx, w.x);
    cy = __fadd_rn(cy, w.y);
    row[s + k] = make_float2(cx, cy);
    const float rx = rintf(cx), ry = rintf(cy);   // positions are in bounds: the walk checked them
    if (rx >= 0.f && rx <= (float)(W - 1) && ry >= 0.f && ry <= (float)(H - 1))
      occ[(size_t)(s + k) * P + (size_t)ry * W + (size_t)rx] = 1;
  }
  for (int t = s + L; t < T; ++t) row[t] = nan2;
}

// ---- of_filter_dino_best_buddies.py:9-29 get_closest_traj_idx_batch -------------------------------------------------
__global__ void traj_transpose_kernel(const float2* __restrict__ traj, int M, int T, float2* __restrict__ posT) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (size_t)M * T) return;
  const size_t n = i / T, t = i - n * T;
  posT[t * M + n] = traj[i];
}

__global__ void fill_u64_kernel(unsigned long long* p, size_t n, unsigned long long v) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) p[i] = v;
}

// Block (grid-point tile, frame t, slice of trajectories): every thread keeps NEAR_PTS grid points; the valid
// positions of the slice are compacted through shared memory (a NaN position is +inf: never nearer) and scanned in
// index order.  The candidate's distance is sqrt(dx*dx + dy*dy) in fp32 without contraction and comparisons are on it
// (ties -> lowest index); the squared sum only skips candidates that cannot be nearer.  Slices merge by atomicMin on
// (distance bits, index) keys, so the result does not depend on the launch shape.
constexpr int NEAR_THREADS = 256, NEAR_PTS = 2;
__global__ void __launch_bounds__(NEAR_THREADS)
traj_nearest_kernel(const float2* __restrict__ posT, int M, int gh, int gw, float start, float step, int slice,
                    unsigned long long* __restrict__ keys) {
  __shared__ float2 s_pos[NEAR_THREADS];
  __shared__ int s_idx[NEAR_THREADS];
  const int G = gh * gw, t = blockIdx.y;
  float px[NEAR_PTS], py[NEAR_PTS], best_r[NEAR_PTS], best_s[NEAR_PTS];
  int best_n[NEAR_PTS];
#pragma unroll
  for (int j = 0; j < NEAR_PTS; ++j) {
    const int g = min(blockIdx.x * NEAR_THREADS * NEAR_PTS + j * NEAR_THREADS + threadIdx.x, G - 1);
    px[j] = __fadd_rn(start, __fmul_rn(step, (float)(g % gw)));
    py[j] = __fadd_rn(start, __fmul_rn(step, (float)(g / gw)));
    best_r[j] = INFINITY; best_s[j] = INFINITY; best_n[j] = 0;
  }
  const float2* pos = posT + (size_t)t * M;
  const int n0 = blockIdx.z * slice, n1 = min(n0 + slice, M);
  for (int base = n0; base < n1; base += NEAR_THREADS) {
    const int n = base + threadIdx.x;
    float2 q = make_float2(NAN, NAN);
    if (n < n1) q = pos[n];
    const bool valid = !isnan(q.x) && !isnan(q.y);
    int cnt;
    const int slot = block_rank<NEAR_THREADS>(valid, &cnt);
    if (valid) { s_pos[slot] = q; s_idx[slot] = n; }
    __syncthreads();
    for (int i = 0; i < cnt; ++i) {
      const float2 c = s_pos[i];
#pragma unroll
      for (int j = 0; j < NEAR_PTS; ++j) {
        const float dx = __fsub_rn(c.x, px[j]), dy = __fsub_rn(c.y, py[j]);
        const float sq = __fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy));
        if (sq < best_s[j]) {
          const float r = __fsqrt_rn(sq);
          if (r < best_r[j]) { best_r[j] = r; best_s[j] = sq; best_n[j] = s_idx[i]; }
        }
      }
    }
    __syncthreads();
  }
#pragma unroll
  for (int j = 0; j < NEAR_PTS; ++j) {
    const int g = blockIdx.x * NEAR_THREADS * NEAR_PTS + j * NEAR_THREADS + threadIdx.x;
    if (g < G && best_r[j] < INFINITY)
      atomicMin(keys + (size_t)t * G + g, ((unsigned long long)__float_as_uint(best_r[j]) << 32) | (unsigned)best_n[j]);
  }
}

__global__ void key_index_kernel(const unsigned long long* __restrict__ keys, size_t n, int* __restrict__ idx) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) idx[i] = (int)(keys[i] & 0xffffffffu);
}

// ---- of_filter_dino_best_buddies.py:86-97 the pair filter ----------------------------------------------------------
// torch's floor division of floats (Python semantics, aten div_floor_floating)
__device__ __forceinline__ float py_floordiv(float a, float b) {
  const float mod = fmodf(a, b);
  float div = __fdiv_rn(__fsub_rn(a, mod), b);
  if (mod != 0.f && ((b < 0.f) != (mod < 0.f))) div = __fsub_rn(div, 1.f);
  if (div == 0.f) return copysignf(0.f, __fdiv_rn(a, b));
  float fd = floorf(div);
  if (__fsub_rn(div, fd) > 0.5f) fd = __fadd_rn(fd, 1.f);
  return fd;
}

// ((p - 7) // stride).long() as an index into a dimension of n (negative indices wrap as in torch indexing)
__device__ __forceinline__ int grid_index(float p, float stride, int n) {
  const float q = py_floordiv(__fsub_rn(p, 7.f), stride);
  int i = fabsf(q) < 2e9f ? (int)q : (q < 0.f ? -n - 1 : n);
  if (i < 0) i += n;
  return min(max(i, 0), n - 1);   // out of range: torch raises; clamp keeps the read inside the table
}

__global__ void of_filter_kernel(const float* __restrict__ traj, int T, const int* __restrict__ nearest, int gh, int gw,
                                 float stride, const float* __restrict__ src_xy, const float* __restrict__ tgt_xy,
                                 const int* __restrict__ pair_src, const int* __restrict__ pair_tgt,
                                 const int* __restrict__ offsets, int n_pairs, int n_pts, uint8_t* __restrict__ keep) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n_pts) return;
  const int lo = last_le(n_pairs, i, offsets);   // pair k: offsets[k] <= i < offsets[k + 1]
  const int ts = pair_src[lo], tt = pair_tgt[lo], G = gh * gw;
  const int ns = nearest[(size_t)ts * G + grid_index(src_xy[2 * i + 1], stride, gh) * gw + grid_index(src_xy[2 * i], stride, gw)];
  const int nt = nearest[(size_t)tt * G + grid_index(tgt_xy[2 * i + 1], stride, gh) * gw + grid_index(tgt_xy[2 * i], stride, gw)];
  const float* a = traj + ((size_t)ns * T + tt) * 2;
  const float* b = traj + ((size_t)nt * T + ts) * 2;
  // keep the pairs the flow does NOT cover: neither point's trajectory reaches the other frame
  keep[i] = ((isnan(a[0]) || isnan(a[1])) && (isnan(b[0]) || isnan(b[1]))) ? 1 : 0;
}

}  // namespace dtk

using namespace dtk;

extern "C" {

static int flow_video_ok(const dinotrk_flow_video* fv) {
  return fv && fv->fwd && fv->bwd && fv->T >= 2 && fv->H >= 2 && fv->W >= 2;
}

int dinotrk_flow_masks(const dinotrk_flow_video* fv, float threshold, uint8_t* masks, void* stream) {
  DTK_CHECK_ARG(flow_video_ok(fv) && masks, "flow_masks: bad arguments (T, H, W >= 2 and non-null flows / masks)");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t P = (size_t)fv->H * fv->W, n = (size_t)(fv->T - 1) * P;
  DTK_CUDA(cudaMemsetAsync(masks, 0, (size_t)(fv->T + 1) * P, st));
  ProfRange pr(PROF_MISC, st);
  flow_cover_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(fv->fwd, fv->T, fv->H, fv->W, masks);
  DTK_LAUNCHED();
  flow_consistency_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(fv->fwd, fv->bwd, fv->T, fv->H, fv->W, threshold, masks);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

struct TrajWs {
  uint8_t* occ; int* len; int* cnt; int* off;
  TrajWs(Arena& ar, int T, int H, int W) {
    const size_t P = (size_t)H * W, nb = (P + TRAJ_THREADS - 1) / TRAJ_THREADS;
    occ = ar.take<uint8_t>((size_t)T * P);
    len = ar.take<int>(P);
    cnt = ar.take<int>(nb);
    off = ar.take<int>(nb);
  }
};

size_t dinotrk_traj_workspace_bytes(int T, int H, int W) { return align_up(layout_end<TrajWs>(T, H, W), 256) + 256; }

int dinotrk_traj_chain(const dinotrk_flow_video* fv, const uint8_t* masks, int s, float threshold, int min_len,
                       const float* direct_fwd, const float* direct_bwd, float direct_threshold, int* n_kept,
                       void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(flow_video_ok(fv) && masks && n_kept && workspace, "traj_chain: null argument");
  DTK_CHECK_ARG(s >= 0 && s < fv->T && min_len >= 1, "traj_chain: start frame %d outside [0, %d) or min_len %d < 1", s, fv->T, min_len);
  DTK_CHECK_ARG((direct_fwd == nullptr) == (direct_bwd == nullptr), "traj_chain: give both direct flows or neither");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_traj_workspace_bytes(fv->T, fv->H, fv->W), "traj_chain: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t P = (size_t)fv->H * fv->W, nb = (P + TRAJ_THREADS - 1) / TRAJ_THREADS;
  Arena ar(workspace);
  const TrajWs w(ar, fv->T, fv->H, fv->W);
  ChainArgs a{fv->fwd, fv->bwd, direct_fwd, direct_bwd, masks, fv->T, fv->H, fv->W, s, min_len, threshold, direct_threshold};
  ProfRange pr(PROF_MISC, st);
  traj_chain_kernel<<<(unsigned)nb, TRAJ_THREADS, 0, st>>>(a, w.occ, w.len, w.cnt);
  DTK_LAUNCHED();
  return launch_count_scan(w.cnt, (int)nb, 1, w.off, n_kept, st);
}

int dinotrk_traj_emit(const dinotrk_flow_video* fv, int s, float* out, void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(flow_video_ok(fv) && workspace && s >= 0 && s < fv->T, "traj_emit: bad arguments");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_traj_workspace_bytes(fv->T, fv->H, fv->W), "traj_emit: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  const size_t P = (size_t)fv->H * fv->W, nb = (P + TRAJ_THREADS - 1) / TRAJ_THREADS;
  Arena ar(workspace);
  const TrajWs w(ar, fv->T, fv->H, fv->W);
  ProfRange pr(PROF_MISC, st);
  traj_emit_kernel<<<(unsigned)nb, TRAJ_THREADS, 0, st>>>(fv->fwd, fv->T, fv->H, fv->W, s, w.len, w.off, w.occ, out);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

struct NearestWs {
  float2* posT; unsigned long long* keys;
  NearestWs(Arena& ar, int M, int T, int gh, int gw) {
    posT = ar.take<float2>((size_t)M * T);
    keys = ar.take<unsigned long long>((size_t)T * gh * gw);
  }
};

size_t dinotrk_traj_nearest_workspace_bytes(int M, int T, int gh, int gw) {
  return align_up(layout_end<NearestWs>(M, T, gh, gw), 256) + 256;
}

int dinotrk_traj_nearest(const float* traj, int M, int T, int gh, int gw, float start, float step, int* nearest,
                         void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(traj && nearest && workspace && M > 0 && T > 0 && gh > 0 && gw > 0, "traj_nearest: bad arguments");
  DTK_CHECK_ARG(workspace_bytes >= dinotrk_traj_nearest_workspace_bytes(M, T, gh, gw), "traj_nearest: workspace too small");
  cudaStream_t st = (cudaStream_t)stream;
  Arena ar(workspace);
  const NearestWs w(ar, M, T, gh, gw);
  const size_t G = (size_t)gh * gw, nk = (size_t)T * G;
  ProfRange pr(PROF_MISC, st);
  const size_t nt = (size_t)M * T;
  traj_transpose_kernel<<<(unsigned)((nt + 255) / 256), 256, 0, st>>>(reinterpret_cast<const float2*>(traj), M, T, w.posT);
  DTK_LAUNCHED();
  // an all-NaN frame keeps (inf, 0): index 0, as torch.argmin over all-inf distances
  fill_u64_kernel<<<(unsigned)((nk + 255) / 256), 256, 0, st>>>(w.keys, nk, (unsigned long long)0x7f800000u << 32);
  DTK_LAUNCHED();
  const int gx = cdiv((int)G, NEAR_THREADS * NEAR_PTS);
  // enough slices of the trajectories to fill the GPU about four times over, none shorter than 4096
  int slices = cdiv(4 * num_sms(), gx * T);
  slices = max(1, min(slices, cdiv(M, 4096)));
  const int slice = cdiv(cdiv(M, slices), NEAR_THREADS) * NEAR_THREADS;
  slices = cdiv(M, slice);
  traj_nearest_kernel<<<dim3(gx, T, slices), NEAR_THREADS, 0, st>>>(w.posT, M, gh, gw, start, step, slice, w.keys);
  DTK_LAUNCHED();
  key_index_kernel<<<(unsigned)((nk + 255) / 256), 256, 0, st>>>(w.keys, nk, nearest);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_of_filter(const float* traj, int M, int T, const int* nearest, int gh, int gw, int stride, const float* src_xy,
                      const float* tgt_xy, const int* pair_src, const int* pair_tgt, const int* offsets, int n_pairs, int n_pts,
                      uint8_t* keep, void* stream) {
  DTK_CHECK_ARG(traj && nearest && M > 0 && T > 0 && gh > 0 && gw > 0 && stride > 0 && n_pairs >= 0 && n_pts >= 0,
                "of_filter: bad arguments");
  if (n_pts == 0) return DINOTRK_OK;
  DTK_CHECK_ARG(src_xy && tgt_xy && pair_src && pair_tgt && offsets && keep && n_pairs > 0, "of_filter: null argument");
  cudaStream_t st = (cudaStream_t)stream;
  ProfRange pr(PROF_MISC, st);
  of_filter_kernel<<<cdiv(n_pts, 256), 256, 0, st>>>(traj, T, nearest, gh, gw, (float)stride, src_xy, tgt_xy, pair_src, pair_tgt,
                                                     offsets, n_pairs, n_pts, keep);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // extern "C"

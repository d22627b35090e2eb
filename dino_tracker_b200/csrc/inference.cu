// Inference driver on the device: trajectories, trajectory cosine similarities, anchor re-tracking and
// occlusion (models/model_inference.py:8-216) + the generic grouped correlation/head entry point behind
// Tracker.forward (models/tracker.py:303-325).
//
// The reference walks query points and anchor frames in Python, one model() call per (query, anchor):
// each call gathers (T+1) x C x h x w twice and runs a B x N einsum.  Here every phase is a handful of
// launches over work lists grouped by target frame:
//   A  trajectories : descriptors s_n (N of them)          x every frame t        -> traj[n][t]
//   B  cos-sims     : d[n][i] sampled along the trajectory . d[n][t_q]            -> cos[n][i]
//   C  anchors      : for every anchor frame a, descriptors e[n][i] (a in A_n)    -> anchors[n][a][i]
//   D  occlusion    : lower medians over anchors, threshold, OR with cos < th     -> occ[n][i]
#include <algorithm>
#include <vector>

#include "common.cuh"
#include "corr.cuh"
#include "head.cuh"
#include "sample.cuh"
#include "xwin.cuh"

namespace dtk {

constexpr int TC2_BM_ROWS = 256;   // M tile of the CTA-pair GEMM (tcgemm.cuh: TC2_BM)

// ---------------------------------------------------------------------------------- phase A helpers
// descriptors of the query points: frames_set = [t_q, s..e-1], set index 0 (model_inference.py:8-34)
__global__ void sample_query_kernel(const float* __restrict__ tpc, int T, int C, int P, int h, int w, PointAffine pa,
                                    const float* __restrict__ qp, float* __restrict__ desc, float* __restrict__ dnorm) {
  int n = blockIdx.x;
  float x = __fadd_rn(__fmul_rn(pa.aw, qp[n * 3 + 0]), pa.bw);
  float y = __fadd_rn(__fmul_rn(pa.ah, qp[n * 3 + 1]), pa.bh);
  int tq = (int)qp[n * 3 + 2];
  tq = min(max(tq, 0), T - 1);
  // set index 0 of a set with N >= 2 slots: t_n = -1 exactly -> slot 0 with weight 1, slot 1 with weight 0.
  // The weight-0 corner is skipped (0 * finite), so only frame t_q contributes.
  TriCorners c = tri_setup(x, y, 0.f, 2, h, w);
  sample_point(tpc, C, P, c, tq, -1, desc + (size_t)n * C, dnorm + n);
}

// out_index / t column for phase A maps of one chunk: map j -> group k -> (n, t)
__global__ void index_traj_kernel(const int* __restrict__ grp_frame, const int* __restrict__ grp_row0,
                                  const int* __restrict__ grp_map0, int n_groups, int n_maps, int T,
                                  int* __restrict__ out_index, float* __restrict__ traj) {
  int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_maps) return;
  const int lo = last_le(n_groups, j, grp_map0);
  int n = grp_row0[lo] + (j - grp_map0[lo]);
  int t = grp_frame[lo];
  out_index[j] = n * T + t;
  traj[((size_t)n * T + t) * 3 + 2] = (float)t;
}

// ---------------------------------------------------------------------------------- phase B
// cos[n][i] = F.cosine_similarity(d[n][t_q], d[n][i]) with d sampled from the full T-frame set
// (model_inference.py:110-126): x / max(|x|, eps) . y / max(|y|, eps), eps = 1e-8.
__global__ void traj_cos_kernel(const float* __restrict__ tpc, int T, int C, int P, int h, int w, PointAffine pa,
                                const float* __restrict__ traj, const float* __restrict__ qp,
                                float* __restrict__ cos_out) {
  extern __shared__ __align__(16) float sm[];  // dq[C], di[C]
  __shared__ float nrm[2];
  __shared__ float red[SAMPLE_THREADS / 32];
  const int n = blockIdx.y, i = blockIdx.x;
  int tq = (int)qp[n * 3 + 2];
  tq = min(max(tq, 0), T - 1);
  for (int which = 0; which < 2; ++which) {
    const float* pt = traj + ((size_t)n * T + (which == 0 ? tq : i)) * 3;
    float x = __fadd_rn(__fmul_rn(pa.aw, pt[0]), pa.bw);
    float y = __fadd_rn(__fmul_rn(pa.ah, pt[1]), pa.bh);
    TriCorners c = tri_setup(x, y, pt[2], T, h, w);  // frames_set = identity over the T frames
    sample_point(tpc, C, P, c, c.z0, c.z1, sm + which * C, nrm + which);
    __syncthreads();
  }
  const float nq = fmaxf(nrm[0], 1e-8f), ni = fmaxf(nrm[1], 1e-8f);
  float acc = 0.f;
  for (int c = threadIdx.x; c < C; c += SAMPLE_THREADS) acc = fmaf(__fdiv_rn(sm[c], nq), __fdiv_rn(sm[C + c], ni), acc);
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = acc;
  __syncthreads();
  if (threadIdx.x == 0) {
    float s = 0.f;
    for (int k = 0; k < SAMPLE_THREADS / 32; ++k) s += red[k];
    cos_out[(size_t)n * T + i] = s;
  }
}

// ---------------------------------------------------------------------------------- phase C helpers
// per anchor frame a: ordered list of the query points n with cos[n][a] >= th, and its length
constexpr int ANCHOR_LIST_THREADS = 256;
__global__ void __launch_bounds__(ANCHOR_LIST_THREADS)
anchor_lists_kernel(const float* __restrict__ cos_sims, int N, int T, float th, int* __restrict__ cnt,
                    int* __restrict__ qlist) {
  const int a = blockIdx.x;
  int base = 0;
  for (int n0 = 0; n0 < N; n0 += ANCHOR_LIST_THREADS) {
    const int n = n0 + threadIdx.x;
    const bool v = n < N && cos_sims[(size_t)n * T + a] >= th;
    int total;
    const int rank = block_rank<ANCHOR_LIST_THREADS>(v, &total);
    if (v) qlist[(size_t)a * N + base + rank] = n;
    base += total;
    __syncthreads();   // the next chunk's block_rank rewrites the warp counts
  }
  if (threadIdx.x == 0) cnt[a] = base;
}

// Anchor work item of map j of a chunk, whose group is lo.  Group k of the chunk covers items
// [grp_item0[k], grp_item0[k] + grp_m[k]) of anchor frame grp_frame[k]; item u = (query slot u / T, frame u % T):
// anchor frame a, query n = qlist[a][slot], source frame i.
struct AnchorItem { int a, slot, i, n; };
__device__ __forceinline__ AnchorItem anchor_item(int j, int lo, int T, const int* __restrict__ qlist, int N,
                                                  const int* __restrict__ grp_frame, const int* __restrict__ grp_map0,
                                                  const int* __restrict__ grp_item0) {
  AnchorItem it;
  it.a = grp_frame[lo];
  const int uu = grp_item0[lo] + (j - grp_map0[lo]);
  it.slot = uu / T; it.i = uu - it.slot * T;
  it.n = qlist[(size_t)it.a * N + it.slot];
  return it;
}

// Trajectory point pt = traj[n][i] (it lives in frame i) sampled from the frame set [a, i0..e-1] at slot i - i0 + 1
// (model_inference.py:138-143): its corners and the frames of its two slots.  Slot 0 is the anchor frame a; without one
// (NoAnchor: the unique table, which samples only points that give slot 0 no weight) it is numbered like the others.
struct NoAnchor {};
__device__ __forceinline__ int slot_frame(int z, int i0, int a) { return z == 0 ? a : i0 + z - 1; }
__device__ __forceinline__ int slot_frame(int z, int i0, NoAnchor) { return i0 + z - 1; }
struct SetSample { TriCorners c; int f0, f1; };
template <class Anchor>
__device__ __forceinline__ SetSample frame_set_sample(const float* __restrict__ pt, int i, int T, int frame_batch, int h, int w,
                                                      const PointAffine& pa, Anchor a) {
  const int i0 = (i / frame_batch) * frame_batch, e = min(i0 + frame_batch, T);
  float x = __fadd_rn(__fmul_rn(pa.aw, pt[0]), pa.bw);
  float y = __fadd_rn(__fmul_rn(pa.ah, pt[1]), pa.bh);
  SetSample s;
  s.c = tri_setup(x, y, (float)(i - i0 + 1), e - i0 + 1, h, w);
  s.f0 = slot_frame(s.c.z0, i0, a);
  s.f1 = s.c.z1 < 0 ? -1 : slot_frame(s.c.z1, i0, a);
  return s;
}

// descriptors of one chunk of anchor work items (see anchor_item)
__global__ void sample_anchor_kernel(const float* __restrict__ tpc, int T, int C, int P, int h, int w, PointAffine pa,
                                     const float* __restrict__ traj, const int* __restrict__ qlist, int N,
                                     const int* __restrict__ grp_frame, const int* __restrict__ grp_map0,
                                     const int* __restrict__ grp_item0, int n_groups, int frame_batch,
                                     float* __restrict__ desc, float* __restrict__ dnorm, int* __restrict__ out_index,
                                     __half* __restrict__ desc_hi, __half* __restrict__ desc_lo) {
  const int j = blockIdx.x;
  const AnchorItem it = anchor_item(j, last_le(n_groups, j, grp_map0), T, qlist, N, grp_frame, grp_map0, grp_item0);
  const SetSample s = frame_set_sample(traj + ((size_t)it.n * T + it.i) * 3, it.i, T, frame_batch, h, w, pa, it.a);
  sample_point(tpc, C, P, s.c, s.f0, s.f1, desc + (size_t)j * C, dnorm + j, desc_hi ? desc_hi + (size_t)j * C : nullptr,
               desc_lo ? desc_lo + (size_t)j * C : nullptr);
  if (threadIdx.x == 0) out_index[j] = (it.n * T + it.a) * T + it.i;
}

// The descriptor of work item (n, i, a) -- trajectory point traj[n][i] sampled from the frame set [a, i0..e-1] at slot
// i - i0 + 1 -- does not depend on the anchor frame a unless the fp32 round trip of the slot index (utils.py:96-99) leaks
// weight onto slot 0.  So every (n, i) is sampled ONCE (fp16 hi / lo halves + norm, what the tensor-path GEMMs consume) and
// flagged if slot 0 takes part; per chunk, unflagged items are row copies, flagged ones are sampled as before.
// int8 row of the coarse pass from a descriptor's hi / lo halves and norm, which the block has just stored (plain loads,
// not the read-only path): warp 0 quantises d = hi + lo; returns rho on lane 0 of warp 0
__device__ __forceinline__ float quant_desc(const __half* hi, const __half* lo, int C, const float* norm, int8_t* q, float* fac) {
  __syncthreads();   // the block's hi / lo stores and the norm (sample_point) are visible
  if (threadIdx.x >= 32) return 0.f;
  const float nrm = *norm;
  return xw_quant_row([&](int k) {
    const uint2 a = *reinterpret_cast<const uint2*>(hi + k), b = *reinterpret_cast<const uint2*>(lo + k);
    const float2 a0 = __half22float2(*reinterpret_cast<const __half2*>(&a.x)), a1 = __half22float2(*reinterpret_cast<const __half2*>(&a.y));
    const float2 b0 = __half22float2(*reinterpret_cast<const __half2*>(&b.x)), b1 = __half22float2(*reinterpret_cast<const __half2*>(&b.y));
    return make_float4(a0.x + b0.x, a0.y + b0.y, a1.x + b1.x, a1.y + b1.y);
  }, C, nrm, q, fac);
}

__global__ void sample_unique_kernel(const float* __restrict__ tpc, int T, int C, int P, int h, int w, PointAffine pa,
                                     const float* __restrict__ traj, int frame_batch, __half* __restrict__ u_hi,
                                     __half* __restrict__ u_lo, float* __restrict__ u_norm, int* __restrict__ u_flag,
                                     int8_t* __restrict__ u_q8, float* __restrict__ u_fac, float* __restrict__ u_rho) {
  const int u = blockIdx.x;                 // n * T + i
  const SetSample s = frame_set_sample(traj + (size_t)u * 3, u % T, T, frame_batch, h, w, pa, NoAnchor{});
  bool slot0 = false;
#pragma unroll
  for (int k = 0; k < 4; ++k) slot0 = slot0 || (s.c.z0 == 0 && s.c.tok[k] >= 0 && s.c.wxy[k][0] != 0.f);
  if (threadIdx.x == 0) u_flag[u] = slot0 ? 1 : 0;
  if (slot0) return;                        // depends on the anchor frame: sampled per work item
  sample_point(tpc, C, P, s.c, s.f0, s.f1, nullptr, u_norm + u, u_hi + (size_t)u * C, u_lo + (size_t)u * C);
  if (u_q8) {   // (+ the int8 row of the coarse pass)
    const float r = quant_desc(u_hi + (size_t)u * C, u_lo + (size_t)u * C, C, u_norm + u, u_q8 + (size_t)u * C, u_fac + u);
    if (threadIdx.x == 0) u_rho[u] = r;
  }
}

// Per-map scalars of one chunk of anchor work items, one thread per map: the output slot, the map's row in the GEMMs' A
// arrays (arow) and, for an unflagged source point, the norm and the coarse bound eps (from the descriptor's residual and
// its anchor frame's rho_f; with_eps: the int8 coarse pass runs) of its unique sample.  A group whose first row lies below
// n_unique is read IN PLACE from the unique table (its rows there are consecutive, the planner saw to that); the maps of
// the other groups get row chunk_row0 + map of the chunk's own descriptor arrays, which gather_anchor_kernel fills.
__global__ void anchor_scalars_kernel(int T, const int* __restrict__ qlist, int N, const int* __restrict__ grp_frame,
                                      const int* __restrict__ grp_row0, const int* __restrict__ grp_map0,
                                      const int* __restrict__ grp_item0, int n_groups, int n_maps, int n_unique, int chunk_row0,
                                      const float* __restrict__ u_norm, const int* __restrict__ u_flag,
                                      const float* __restrict__ u_rho, const float* __restrict__ rho_f, float eps_slack, bool with_eps,
                                      int* __restrict__ out_index, int* __restrict__ arow, float* __restrict__ dnorm,
                                      float* __restrict__ desc_eps) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n_maps) return;
  const int lo = last_le(n_groups, j, grp_map0);
  const AnchorItem it = anchor_item(j, lo, T, qlist, N, grp_frame, grp_map0, grp_item0);
  const size_t u = (size_t)it.n * T + it.i;
  out_index[j] = (it.n * T + it.a) * T + it.i;
  const int r0 = grp_row0[lo];
  arow[j] = r0 < n_unique ? r0 + (j - grp_map0[lo]) : chunk_row0 + j;
  if (u_flag[u]) return;   // sampled per work item: gather_anchor_kernel writes the norm and eps
  dnorm[j] = u_norm[u];
  if (with_eps) desc_eps[j] = xw_eps_s8(u_rho[u], rho_f[it.a], eps_slack);
}

// descriptors (fp16 hi / lo; with desc_q8: + the int8 row and its factor) of the GATHERED maps of one chunk of anchor work
// items: row copies from the unique samples, or, for a flagged source point, the sample itself with its norm and eps.
// One block per map of [map_lo, map_lo + gridDim.x); maps of in-place groups are left alone.  desc_* / dnorm / desc_fac /
// desc_eps are the chunk's arrays (row = map).
__global__ void gather_anchor_kernel(const float* __restrict__ tpc, int T, int C, int P, int h, int w, PointAffine pa,
                                     const float* __restrict__ traj, const int* __restrict__ qlist, int N,
                                     const int* __restrict__ grp_frame, const int* __restrict__ grp_row0,
                                     const int* __restrict__ grp_map0, const int* __restrict__ grp_item0, int n_groups,
                                     int n_unique, int map_lo, int frame_batch, const __half* __restrict__ u_hi,
                                     const __half* __restrict__ u_lo, const int* __restrict__ u_flag,
                                     float* __restrict__ dnorm, __half* __restrict__ desc_hi,
                                     __half* __restrict__ desc_lo, const int8_t* __restrict__ u_q8,
                                     const float* __restrict__ u_fac, const float* __restrict__ rho_f, float eps_slack,
                                     int8_t* __restrict__ desc_q8, float* __restrict__ desc_fac,
                                     float* __restrict__ desc_eps) {
  const int j = map_lo + blockIdx.x;
  const int lo = last_le(n_groups, j, grp_map0);
  if (grp_row0[lo] < n_unique) return;   // read in place
  const AnchorItem it = anchor_item(j, lo, T, qlist, N, grp_frame, grp_map0, grp_item0);
  const size_t u = (size_t)it.n * T + it.i;
  if (!u_flag[u]) {
    const uint4* sh = reinterpret_cast<const uint4*>(u_hi + u * C);
    const uint4* sl = reinterpret_cast<const uint4*>(u_lo + u * C);
    uint4* dh = reinterpret_cast<uint4*>(desc_hi + (size_t)j * C);
    uint4* dl = reinterpret_cast<uint4*>(desc_lo + (size_t)j * C);
    for (int k = threadIdx.x; k < C / 8; k += blockDim.x) { dh[k] = __ldg(sh + k); dl[k] = __ldg(sl + k); }
    if (desc_q8) {
      const uint4* sq = reinterpret_cast<const uint4*>(u_q8 + u * C);
      uint4* dq = reinterpret_cast<uint4*>(desc_q8 + (size_t)j * C);
      for (int k = threadIdx.x; k < C / 16; k += blockDim.x) dq[k] = __ldg(sq + k);
      if (threadIdx.x == 0) desc_fac[j] = u_fac[u];
    }
    return;
  }
  const SetSample s = frame_set_sample(traj + u * 3, it.i, T, frame_batch, h, w, pa, it.a);
  sample_point(tpc, C, P, s.c, s.f0, s.f1, nullptr, dnorm + j, desc_hi + (size_t)j * C, desc_lo + (size_t)j * C);
  if (desc_q8) {
    const float r = quant_desc(desc_hi + (size_t)j * C, desc_lo + (size_t)j * C, C, dnorm + j, desc_q8 + (size_t)j * C, desc_fac + j);
    if (threadIdx.x == 0) desc_eps[j] = xw_eps_s8(r, rho_f[it.a], eps_slack);
  }
}

// ---------------------------------------------------------------------------------- phase D
// model_inference.py:169-177.  One block per query point, one warp per column i.
// D[a][i] = |anchors[n][a][i] - traj[n][a]| for a in A_n; med[i] = lower median over a
// (torch.median: sorted position (M-1)/2); th = max_{i in A_n} med[i];
// occ[i] = med[i] > th || cos[n][i] < cos_th.
constexpr int OCC_THREADS = 256;
__global__ void occlusion_kernel(const float* __restrict__ traj, const float* __restrict__ cos_sims,
                                 const float* __restrict__ anchors, int T, float anchor_th, float cos_th,
                                 uint8_t* __restrict__ occ) {
  extern __shared__ float sm[];  // med[T] | alist[T] | ax[T] | ay[T] | col[nwarps][T]
  float* med = sm;
  int* alist = reinterpret_cast<int*>(sm + T);
  float* ax = sm + 2 * T;
  float* ay = sm + 3 * T;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = OCC_THREADS / 32;
  float* col = sm + 4 * T + warp * T;
  __shared__ int M;
  __shared__ float th_s;
  const int n = blockIdx.x;
  if (threadIdx.x == 0) {
    int m = 0;
    for (int a = 0; a < T; ++a)
      if (cos_sims[(size_t)n * T + a] >= anchor_th) {
        alist[m] = a;
        ax[m] = traj[((size_t)n * T + a) * 3 + 0];
        ay[m] = traj[((size_t)n * T + a) * 3 + 1];
        ++m;
      }
    M = m;
  }
  __syncthreads();
  const int m = M, want = (m - 1) / 2;
  for (int i = warp; i < T; i += nw) {
    for (int p = lane; p < m; p += 32) {
      const float* g = anchors + (((size_t)n * T + alist[p]) * T + i) * 2;
      float dx = __fsub_rn(g[0], ax[p]), dy = __fsub_rn(g[1], ay[p]);
      col[p] = sqrtf(__fadd_rn(__fmul_rn(dx, dx), __fmul_rn(dy, dy)));
    }
    __syncwarp();
    for (int p = lane; p < m; p += 32) {
      const float dp = col[p];
      int rank = 0;
      for (int q = 0; q < m; ++q) {
        float dq = col[q];
        rank += (dq < dp) || (dq == dp && q < p);
      }
      if (rank == want) med[i] = dp;
    }
    __syncwarp();
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    float th = -INFINITY;
    for (int p = 0; p < m; ++p) th = fmaxf(th, med[alist[p]]);
    th_s = th;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < T; i += blockDim.x)
    occ[(size_t)n * T + i] = (m > 0 && (med[i] > th_s || cos_sims[(size_t)n * T + i] < cos_th)) ? 1 : 0;
}

struct GroupBuf {  // host mirror of the per-chunk group arrays: [frame | row0 | m | map0 | item0] x cap
  std::vector<int> v;
  int cap, n;
  bool overflow = false;   // a push beyond cap (dropped): the caller's bound on the groups of a chunk was wrong
  explicit GroupBuf(int c) : v((size_t)5 * c), cap(c), n(0) {}
  void clear() { n = 0; }
  void push(int frame, int row0, int m, int map0, int item0) {
    if (n >= cap) { overflow = true; return; }
    v[n] = frame; v[cap + n] = row0; v[2 * cap + n] = m; v[3 * cap + n] = map0; v[4 * cap + n] = item0; ++n;
  }
};

// ---- chunk planning (host only) ---------------------------------------------------------------------------------
// A phase's work items are cut into chunks of <= ch correlation maps; inside a chunk, items of the same target
// frame form one group = [frame | first descriptor row | number of rows m | first map | first item] (GroupBuf order).
//   kind 0 (trajectories): items = (frame t, query row n), t-major; descriptor rows are the N query rows.
//   kind 1 (anchors): items of anchor frame a = cnt[a] * T pairs (slot, i), a-major; descriptor rows are per chunk
//   (row = map), or, with AnchorRows, rows of one array that holds the unique table and the chunks' own rows behind it.
struct ChunkMeta { int used, maxm, n_groups; bool no_thin; int n_gathered, gather_lo, gather_hi; };   // gathered maps lie in [lo, hi)
// Descriptor rows of the exact-window pipeline.  The descriptor of item (slot, i) of anchor frame a is row n T + i of the
// unique table, n = qlist[a][slot], unless query n is flagged (qflag: some source frame's sample depends on the anchor
// frame).  So the T-item cells of consecutive unflagged queries are consecutive rows there and a GEMM can read them in
// place.  A frame's span of a chunk is cut into groups at the runs of consecutive unflagged queries; a run is read in place
// when padding it to whole 256-row tiles of the coarse GEMM costs at most 1 / XW_INPLACE_PAD_DIV of its rows.  Shorter runs
// and flagged queries are gathered into the chunk's own rows (row gather_row0 + ring slot * ring_stride + map), adjacent
// ones as one group.
constexpr int XW_INPLACE_PAD_DIV = 16;
constexpr int XW_INPLACE_MIN_ROWS = TC2_BM_ROWS - TC2_BM_ROWS / (XW_INPLACE_PAD_DIV + 1);   // 241: the shortest such run
struct AnchorRows { const int* qlist; const unsigned char* qflag; int gather_row0, ring, ring_stride; };
// align: anchor-phase chunks are cut at multiples of `align` items per frame (T for the exact-window path: whole cells).
// first_cap > 0: capacity of the first anchor-phase chunk only (the probe chunk of the exact-window pipeline).
// rows (with align = T): see AnchorRows; the chunks hold the same items with or without it.  False: gcap was too small.
static bool plan_chunks(int kind, int T, int N, const int* cnt, int ch_all, int gcap, std::vector<ChunkMeta>& metas,
                        std::vector<int>& plan_host, int align = 1, int first_cap = 0, const AnchorRows* rows = nullptr) {
  int ch = ch_all;
  metas.clear(); plan_host.clear();
  GroupBuf gb(gcap);
  int n_gathered = 0, gather_lo = 0, gather_hi = 0;
  auto commit_chunk = [&](int used) {
    bool no_thin = true;
    int maxm = 0;
    for (int k = 0; k < gb.n; ++k) {
      no_thin = no_thin && gb.v[2 * gb.cap + k] > STREAM_MAX_M;
      maxm = std::max(maxm, gb.v[2 * gb.cap + k]);
    }
    metas.push_back(ChunkMeta{used, maxm, gb.n, no_thin, n_gathered, gather_lo, gather_hi});
    plan_host.insert(plan_host.end(), gb.v.begin(), gb.v.end());
    n_gathered = gather_lo = gather_hi = 0;
  };
  // groups of the span [item0, item0 + m) of anchor frame a, maps map0 .. of the chunk being filled
  auto push_span = [&](int a, int map0, int m, int item0) {
    if (!rows) { gb.push(a, map0, m, map0, item0); return; }
    const int* ql = rows->qlist + (size_t)a * N;
    const int chunk_row0 = rows->gather_row0 + (int)(metas.size() % rows->ring) * rows->ring_stride;
    const int s0 = item0 / T, s1 = (item0 + m) / T;
    int gs = -1;   // first slot of the gathered group being collected
    auto close_gathered = [&](int s_end) {
      if (gs < 0) return;
      const int gm = (s_end - gs) * T, gmap = map0 + (gs - s0) * T;
      gb.push(a, chunk_row0 + gmap, gm, gmap, gs * T);
      if (n_gathered == 0) gather_lo = gmap;
      n_gathered += gm; gather_hi = gmap + gm;
      gs = -1;
    };
    for (int s = s0; s < s1;) {
      const bool flagged = rows->qflag[ql[s]] != 0;
      int e = s + 1;
      while (!flagged && e < s1 && ql[e] == ql[e - 1] + 1 && !rows->qflag[ql[e]]) ++e;
      const int r = (e - s) * T, pad = (r + TC2_BM_ROWS - 1) / TC2_BM_ROWS * TC2_BM_ROWS - r;
      if (!flagged && (long long)pad * XW_INPLACE_PAD_DIV <= r) {
        close_gathered(s);
        gb.push(a, ql[s] * T, r, map0 + (s - s0) * T, s * T);
      } else if (gs < 0) {
        gs = s;
      }
      s = e;
    }
    close_gathered(s1);
  };
  if (kind == 0) {
    int t = 0, row = 0;  // next work item: (frame t, query row)
    while (t < T) {
      gb.clear();
      int used = 0;
      while (t < T && used < ch && gb.n < gcap) {
        int m = N - row;
        if (m > ch - used) m = ch - used;
        gb.push(t, row, m, used, 0);
        used += m; row += m;
        if (row == N) { row = 0; ++t; }
      }
      commit_chunk(used);
    }
  } else {
    int a = 0;
    long long item = 0;  // next work item: anchor frame a, item index within a (slot * T + i)
    while (a < T) {
      gb.clear();
      int used = 0;
      ch = (metas.empty() && first_cap > 0 && first_cap < ch_all) ? first_cap : ch_all;
      while (a < T && used < ch && gb.n < gcap) {
        long long tot = (long long)cnt[a] * T;
        long long m = tot - item;
        if (m > ch - used) {
          m = (long long)((ch - used) / align) * align;
          if (m == 0 && used > 0) break;            // chunk full up to the alignment
          if (m == 0) m = align;                    // (ch >= align is guaranteed by the caller)
        }
        if (m > 0) {
          push_span(a, used, (int)m, (int)item);
          used += (int)m; item += m;
        }
        if (item >= tot) { item = 0; ++a; }
      }
      if (used == 0) break;
      commit_chunk(used);
    }
  }
  return !gb.overflow;
}

// ---- cells of the exact-window path (xwin.cuh): the <= 128 source frames of one (query slot, anchor frame) ----
struct CellPlan {
  std::vector<int> v;               // per chunk: [first map | m | frame | group | first A row] x (cells of the chunk), chunks back to back
  std::vector<size_t> first;        // first cell of chunk k in v's cell numbering (size chunks + 1)
  std::vector<int> tiles;           // per chunk: (gcap + 1) prefix of ceil(m / 256) per group (coarse GEMM)
  int max_m = 0;
};
static void plan_cells(int T, int gcap, const std::vector<ChunkMeta>& metas, const std::vector<int>& plan_host, CellPlan& cp) {
  const int nb = (T + XW_MAX_CELL - 1) / XW_MAX_CELL, rb = (T + nb - 1) / nb;
  cp.v.clear(); cp.first.assign(1, 0); cp.tiles.clear(); cp.max_m = 0;
  std::vector<int> r0, mm, fr, gr, ar;
  for (size_t k = 0; k < metas.size(); ++k) {
    const int* gb = plan_host.data() + k * 5 * gcap;
    r0.clear(); mm.clear(); fr.clear(); gr.clear(); ar.clear();
    int pre = 0;
    for (int g = 0; g < metas[k].n_groups; ++g) {
      const int frame = gb[g], row0 = gb[gcap + g], m = gb[2 * gcap + g], map0 = gb[3 * gcap + g];
      cp.tiles.push_back(pre);
      pre += (m + TC2_BM_ROWS - 1) / TC2_BM_ROWS;
      for (int s0 = 0; s0 < m; s0 += T)
        for (int b = 0; b < T; b += rb) {
          const int cm = std::min(rb, T - b);
          r0.push_back(map0 + s0 + b); mm.push_back(cm); fr.push_back(frame); gr.push_back(g); ar.push_back(row0 + s0 + b);
          cp.max_m = std::max(cp.max_m, cm);
        }
    }
    for (int g = metas[k].n_groups; g <= gcap; ++g) cp.tiles.push_back(pre);
    const size_t n = r0.size();
    cp.v.insert(cp.v.end(), r0.begin(), r0.end());
    cp.v.insert(cp.v.end(), mm.begin(), mm.end());
    cp.v.insert(cp.v.end(), fr.begin(), fr.end());
    cp.v.insert(cp.v.end(), gr.begin(), gr.end());
    cp.v.insert(cp.v.end(), ar.begin(), ar.end());
    cp.first.push_back(cp.first.back() + n);
  }
}

// side stream + events of the anchor phase's pipelining (one set per device; see dinotrk_infer_set_overlap)
struct InferAsync {
  cudaStream_t side;   // sampling stream
  cudaEvent_t fork, join, sample[2], gemm[2];
};
static int g_overlap_mode = -1;   // -1: the default (1); see dinotrk_infer_set_overlap
struct InferAsyncSlot { InferAsync ia; int state; };   // state 0: not created, 1: ready, -1: creation failed
static InferAsync* infer_async() {
  static PerDev<InferAsyncSlot> slots;   // streams and events belong to the device they were created on
  if (g_overlap_mode == 0) return nullptr;
  InferAsyncSlot& slot = slots.get();
  InferAsync& ia = slot.ia;
  if (slot.state == 0) {
    slot.state = -1;
    if (cudaStreamCreateWithFlags(&ia.side, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    cudaEvent_t* evs[] = {&ia.fork, &ia.join, &ia.sample[0], &ia.sample[1], &ia.gemm[0], &ia.gemm[1]};
    for (cudaEvent_t* ev : evs)
      if (cudaEventCreateWithFlags(ev, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    slot.state = 1;
  }
  return slot.state == 1 ? &ia : nullptr;
}

// events, pinned counters and selection of the exact-window pipeline (one set per device)
constexpr int XW_RING = 4;
constexpr int XW_PROBE_MAPS = 4096;   // size of the probe chunk (automatic pipeline choice)
constexpr int INFER_A_COUNTED = 16;   // trajectory-phase chunks whose uncertified maps the anchor phase's choice reads
// host_cnt: [XW_RING][XW_CNT_CHUNK] queue total / uncertified / extent tokens / box-GEMM cells of the chunks in flight |
// [INFER_A_COUNTED] trajectory-phase uncertified counts | the video's smallest token norm
constexpr int XW_CNT_CHUNK = 4, XW_CNT_A = XW_CNT_CHUNK * XW_RING, XW_CNT_MINNORM = XW_CNT_A + INFER_A_COUNTED;
struct XwAsync {
  int state;                                   // 0: not created, 1: ready, -1: failed
  cudaEvent_t sample[XW_RING], done[XW_RING], freed[XW_RING];
  int* host_cnt;                               // pinned (see XW_CNT_*)
};
static XwAsync* xw_async() {
  static PerDev<XwAsync> slots;
  XwAsync& xa = slots.get();
  if (xa.state == 0) {
    xa.state = -1;
    for (int k = 0; k < XW_RING; ++k) {
      if (cudaEventCreateWithFlags(&xa.sample[k], cudaEventDisableTiming) != cudaSuccess) return nullptr;
      if (cudaEventCreateWithFlags(&xa.done[k], cudaEventDisableTiming) != cudaSuccess) return nullptr;
      if (cudaEventCreateWithFlags(&xa.freed[k], cudaEventDisableTiming) != cudaSuccess) return nullptr;
    }
    if (cudaHostAlloc(&xa.host_cnt, (XW_CNT_MINNORM + 4) * sizeof(int), cudaHostAllocDefault) != cudaSuccess) return nullptr;
    xa.state = 1;
  }
  return xa.state == 1 ? &xa : nullptr;
}
static int g_xw_path = -1;                     // -1: automatic, 0: full-map path only, 1: exact-window path
static int g_xw_coarse = -1;                   // -1: automatic, 0: fp16 coarse pass, 1: int8 coarse pass
// Slots of dinotrk_infer_last_stats, named as the keys of _lib.infer_stats(): anchor-phase maps | finished on the
// exact-window path | re-done on the full-map path | pipeline used | of those re-done, queued by the certificate |
// tensor-core contraction | int8 coarse pass | bits of the largest per-frame int8 residual | exact-window maps whose
// descriptor was read in place from the unique table | those gathered into the chunk's rows | cells the exact box GEMM
// ran on | the tokens of their extents (xwin.cuh, XwChunk::box_ext)
namespace infer_stat {
enum { anchor_maps, exact_window, full_map, pipeline, full_map_by_certificate, contraction, coarse, coarse_rho_f,
       desc_in_place, desc_gathered, exact_box_cells, exact_box_tokens, count };
}
static long long g_infer_stats[infer_stat::count] = {};
// the probe chunk queues more than this fraction of its maps on the int8 coarse pass: the rest of the phase runs the fp16
// pass.  A queued map costs a full-map split-precision GEMM, ~3 fp16 coarse passes, while the int8 pass saves about half
// of one per map: int8 loses above ~1/6 extra queued maps.  1/16 leaves a wide margin.
constexpr int XW_S8_PROBE_QUEUE_DIV = 16;

// Which pipeline the anchor phase runs, and the exact-window pipeline's coarse pass.  Every rule of the choice is here, in
// the order it is applied: what the call can run (before the host sync), what the video and the trajectory phase showed
// (after it), and the verdict of the probe chunk.
struct AnchorChoice {
  XwAsync* xa = nullptr;   // events and pinned counters of the exact-window pipeline; nullptr: it cannot run
  bool xw = false;         // the exact-window pipeline: coarse pass + exact window (xwin.cuh)
  bool probe = false;      // automatic: its first chunk is a probe whose verdict may change the rest of the phase
  bool s8 = false;         // its coarse pass on int8 tensor cores

  // Before the host sync: the exact-window pipeline needs the tensor-core contraction, the disc inside the window box, not
  // to be switched off, and its events.
  AnchorChoice(const FeatView& fv, const dinotrk_geom& g) {
    if (fv.tensor() && disc_fits_box(g) && g_xw_path != 0) xa = xw_async();
    xw = xa != nullptr;
    probe = g_xw_path < 0;
  }
  // the int8 rows of the unique table are sampled whenever the int8 coarse pass can still be chosen
  static bool q8_rows(const FeatView& fv) { return fv.s8() && g_xw_coarse != 0 && fv.C % 16 == 0 && fv.C <= XW_S8_MAX_C; }
  // After the host sync.  A token below the split's faithful range (a zero one included) voids the coarse pass's error
  // bound.  Automatic mode: head weights the certificate cannot handle send (almost) every map to the full-map kernels
  // anyway; the trajectory phase just showed it when more than a quarter of its first chunks' maps went uncertified.
  void after_sync(int C, int n_counted_A, long long maps_A) {
    if (!xw) return;
    float mn;
    memcpy(&mn, xa->host_cnt + XW_CNT_MINNORM, sizeof(float));
    if (!(mn >= split_min_norm(C))) xw = false;
    if (xw && probe && n_counted_A > 0) {
      long long unc = 0;
      for (int k = 0; k < n_counted_A; ++k) unc += xa->host_cnt[XW_CNT_A + k];
      if (unc * 4 > maps_A) xw = false;
    }
  }
  // Once xw is final: int8 when the features carry their int8 operands (forced: required), unless in automatic mode a
  // frame's residual rho_f makes the bound too loose.
  int coarse_pass(const FeatView& fv, float rho_max) {
    DTK_CHECK_ARG(g_xw_coarse != 1 || !xw || fv.s8(), "infer: int8 coarse pass forced without the int8 features");
    s8 = xw && fv.s8() && g_xw_coarse != 0;
    DTK_CHECK_ARG(!s8 || (fv.C % 16 == 0 && fv.C <= XW_S8_MAX_C), "infer: int8 coarse pass needs C %% 16 == 0 and C <= %d",
                  XW_S8_MAX_C);
    if (g_xw_coarse < 0 && !(rho_max <= XW_S8_RHO_MAX)) s8 = false;
    return DINOTRK_OK;
  }
  // The probe chunk's verdict from its maps queued for the full-map kernels.  More than a quarter queued by the certificate
  // (refiner weights whose outside-the-box logit bound needs the exact map): the rest of the phase runs the full-map
  // pipeline (true).  Else, automatic coarse mode, more than 1 / XW_S8_PROBE_QUEUE_DIV queued: the fp16 coarse pass.
  bool probe_says_full_maps(long long by_certificate, long long queued, int maps) {
    if (by_certificate * 4 > maps) return true;
    if (s8 && g_xw_coarse < 0 && queued * XW_S8_PROBE_QUEUE_DIV > maps) s8 = false;
    return false;
  }
};

// workspace of dinotrk_corr_track: the maps, the correlation's plan and split, the head's list of uncertified maps
struct CorrTrackWs {
  float* maps; CorrMapsWs corr; int* hscratch;
  CorrTrackWs(Arena& ar, int total_maps, int n_groups, int C, int map_stride)
      : maps(ar.take<float>((size_t)total_maps * map_stride)), corr(ar, total_maps, n_groups, C),
        hscratch(ar.take<int>(total_maps + 1)) {}
};

struct ChunkBufs {   // everything one chunk in flight owns
  float* maps; float* desc; float* norm; int* plan; float* split; int* hscratch; unsigned long long* tkeys;
  ChunkBufs() = default;
  ChunkBufs(Arena& ar, int C, int N, int P, int ms, int ch, int gcap) {
    maps = ar.take<float>((size_t)ch * ms);
    desc = ar.take<float>((size_t)ch * C);
    norm = ar.take<float>(ch);
    plan = ar.take<int>(gcap + 1);
    split = ar.take<float>(corr_tc_workspace_bytes(ch > N ? ch : N, C) / 4);
    hscratch = ar.take<int>(ch + 1);
    tkeys = ar.take<unsigned long long>((size_t)ch * cdiv(P, CORR_TILE));
  }
};

// One ring slot of the exact-window pipeline: its rows [row0, row0 + ch) of the descriptor table and its per-map arrays
// (norm: per map; for a gathered map also its row's).
struct XwSet {
  int row0; float* norm; int* out_index; int* arow; float* eps; XwChunk xc;
  XwSet() = default;
  XwSet(Arena& ar, int row0_, float* u_norm, int P, int ch, int gcap) : row0(row0_), norm(u_norm + row0_) {
    out_index = ar.take<int>(ch);
    arow = ar.take<int>(ch);
    eps = ar.take<float>(ch);
    xc = XwChunk(ar, ch, (size_t)ch + 2, cdiv(P, XW_TILE), gcap);   // cells have >= 1 row
  }
};

// The workspace of dinotrk_infer for chunks of ch maps, gcap groups per chunk and at most max_chunks chunks per phase.
struct InferWs {
  float* descA; float* normA;
  ChunkBufs cb[2];
  int* out_index_ring[4];   // written by the sampler of chunk k, read by both head kernels of chunk k (the second one late)
  int* d_groups; int* d_cnt; int* d_qlist;
  // Descriptor rows of the exact-window GEMMs, one row numbering for every per-row array: rows [0, N T) are the unique
  // table (row n T + i: trajectory point i of query n), rows N T + k ch + j the gathered map j of ring slot k.  One A
  // tensor map per operand covers both, so a group reads its rows wherever they are.
  size_t xw_rows;
  __half* u_hi; __half* u_lo; int8_t* u_q8; float* u_norm; float* u_fac; int* u_flag; float* u_rho;
  float* d_rnorms; unsigned* d_minnorm;
  XwSet xr[XW_RING];
  int cell_nb;   // cells per trajectory
  int* d_cells; int* d_tiles;
  int sg_cap;    // groups of the accumulated full-map queue
  int* d_cgrp; int* d_splan; int* d_cntA;
  InferWs(Arena& ar, int T, int C, int N, int P, int ms, int ch, int gcap, size_t max_chunks) {
    descA = ar.take<float>((size_t)N * C);
    normA = ar.take<float>(N);
    for (ChunkBufs& b : cb) b = ChunkBufs(ar, C, N, P, ms, ch, gcap);
    for (int*& r : out_index_ring) r = ar.take<int>(ch);
    d_groups = ar.take<int>(max_chunks * 5 * gcap);
    d_cnt = ar.take<int>(T);
    d_qlist = ar.take<int>((size_t)T * N);
    const int n_unique = N * T;
    xw_rows = (size_t)n_unique + (size_t)XW_RING * ch;
    u_hi = ar.take<__half>(xw_rows * C);
    u_lo = ar.take<__half>(xw_rows * C);
    u_q8 = ar.take<int8_t>(xw_rows * C);
    u_norm = ar.take<float>(xw_rows);
    u_fac = ar.take<float>(xw_rows);
    u_flag = ar.take<int>((size_t)N * T);
    u_rho = ar.take<float>((size_t)N * T);
    d_rnorms = ar.take<float>((size_t)T * P);
    d_minnorm = ar.take<unsigned>(4);
    for (int k = 0; k < XW_RING; ++k) xr[k] = XwSet(ar, n_unique + k * ch, u_norm, P, ch, gcap);
    cell_nb = (T + XW_MAX_CELL - 1) / XW_MAX_CELL;
    d_cells = ar.take<int>((size_t)N * T * cell_nb * 5 + 16);
    d_tiles = ar.take<int>(max_chunks * (gcap + 1));
    sg_cap = (int)std::min<size_t>(max_chunks * (size_t)gcap, 16384);
    d_cgrp = ar.take<int>((size_t)4 * sg_cap);
    d_splan = ar.take<int>((size_t)sg_cap + 1);
    d_cntA = ar.take<int>(64);
  }
};

// What every phase of one dinotrk_infer call reads, and the host plan of the phase's chunks.
struct InferCtx {
  const FeatView& fv; const dinotrk_geom& g; const dinotrk_head_weights& hw;
  InferWs& ws; cudaStream_t st;
  int T, C, N, P, ms, ch, gcap, fb;   // fb: frames per batch of the anchor phase's frame sets
  size_t max_chunks;
  PointAffine pa;
  // The chunks of a phase are planned on the host in one go and their group arrays uploaded with ONE copy, so the
  // per-chunk launches never block the host (a pageable cudaMemcpyAsync per chunk would).
  std::vector<ChunkMeta> metas;
  std::vector<int> plan_host;
  int upload_plan() {
    DTK_CHECK_ARG(metas.size() <= max_chunks, "infer: chunk plan exceeds its bound (%zu > %zu)", metas.size(), max_chunks);
    if (!plan_host.empty())
      DTK_CUDA(cudaMemcpyAsync(ws.d_groups, plan_host.data(), plan_host.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    return DINOTRK_OK;
  }
  struct Grp { const int *f, *r, *m, *map0, *item; };
  Grp grp_of(size_t k) const {   // the device group arrays of chunk k
    const int* b = ws.d_groups + k * 5 * gcap;
    return Grp{b, b + gcap, b + 2 * gcap, b + 3 * gcap, b + 4 * gcap};
  }
};

// ---- phase A: trajectories.  The uncertified maps of the first INFER_A_COUNTED chunks are counted into ws.d_cntA, for the
// anchor phase's choice; n_counted: how many chunks.
static int infer_trajectories(InferCtx& c, const float* query_points, float* traj, int& n_counted) {
  NvtxRange nv("dinotrk.infer.A.trajectories");
  InferWs& ws = c.ws;
  const bool tensor = c.fv.tensor();   // tensor-core GEMM: tile keys for the head
  {
    ProfRange pr(PROF_SAMPLE, c.st);
    sample_query_kernel<<<c.N, SAMPLE_THREADS, 0, c.st>>>(c.fv.tpc, c.T, c.C, c.P, c.g.h, c.g.w, c.pa, query_points, ws.descA,
                                                           ws.normA);
    DTK_LAUNCHED();
  }
  if (tensor) {   // the query descriptors are reused by every chunk: split them once (layout of desc_rows = N)
    for (int k = 0; k < 2; ++k) {
      const DescSplit a(ws.cb[k].split, c.N, c.C);
      int rc = corr_hilo(c.fv) ? launch_split_hilo(ws.descA, a.hi, c.N, c.C, c.st)
                               : launch_split_f16(ws.descA, a.hi, a.lo, (size_t)c.N * c.C, c.st);
      if (rc) return rc;
    }
  }
  plan_chunks(0, c.T, c.N, nullptr, c.ch, c.gcap, c.metas, c.plan_host);
  int rc = c.upload_plan();
  if (rc) return rc;
  for (size_t k = 0; k < c.metas.size(); ++k) {
    const ChunkMeta& cm = c.metas[k];
    const ChunkBufs& b = ws.cb[k & 1];
    const InferCtx::Grp gp = c.grp_of(k);
    {
      ProfRange pr(PROF_MISC, c.st);
      index_traj_kernel<<<cdiv(cm.used, 256), 256, 0, c.st>>>(gp.f, gp.r, gp.map0, cm.n_groups, cm.used, c.T,
                                                              ws.out_index_ring[k & 3], traj);
      DTK_LAUNCHED();
    }
    CorrAssist as;
    as.tkeys = tensor ? b.tkeys : nullptr; as.zero_word = b.hscratch; as.split_ready = tensor; as.no_thin = cm.no_thin;
    rc = launch_corr_maps(c.fv, ws.descA, c.N, ws.normA, gp.f, gp.r, gp.m, gp.map0, cm.n_groups, cm.used, cm.maxm, b.maps, c.ms,
                          b.plan, b.split, c.st, as);
    if (rc) return rc;
    rc = launch_head(b.maps, cm.used, c.ms, c.g, c.hw, ws.out_index_ring[k & 3], traj, 3, 0, nullptr, b.hscratch, c.st, as.tkeys,
                     true);
    if (rc) return rc;
    if (k < INFER_A_COUNTED)
      DTK_CUDA(cudaMemcpyAsync(ws.d_cntA + k, b.hscratch, sizeof(int), cudaMemcpyDeviceToDevice, c.st));
  }
  n_counted = (int)std::min<size_t>(c.metas.size(), INFER_A_COUNTED);
  return DINOTRK_OK;
}

// ---- phase C, exact-window pipeline (xwin.cuh): XW_RING chunks in flight, each with its ring slot of per-map arrays and
// gathered descriptor rows.  The sampling stream sb fills a chunk's scalars and gathered rows; the caller's stream runs its
// coarse pass, cell plan, exact-window GEMM and head.  The maps the head cannot certify go to the full-map queue: their
// descriptors are appended to ONE compact array (buffer set ws.cb[0]), which is worked off -- split-precision GEMM over all
// tokens on 128-row tiles + the head kernels of head.cu -- when it is full and at the end of the phase.
struct ExactWindow {
  InferCtx& c;
  const AnchorChoice& choice;
  const CellPlan& cp;
  bool ovl;             // sb is the side stream
  cudaStream_t sb;
  const float* traj;
  float* anchors;
  int q_rows = 0, q_groups = 0;   // the full-map queue

  XwCells cells_of(size_t k) const {
    XwCells x;
    const int n = (int)(cp.first[k + 1] - cp.first[k]);
    const int* base = c.ws.d_cells + 5 * cp.first[k];
    x.row0 = base; x.m = base + n; x.frame = base + 2 * n; x.group = base + 3 * n; x.arow = base + 4 * n;
    x.n_cells = n; x.max_m = cp.max_m;
    return x;
  }
  // the per-map scalars of chunk k and its gathered descriptor rows, on sb
  int sample(size_t k) {
    InferWs& ws = c.ws;
    const ChunkMeta& cm = c.metas[k];
    const XwSet& x = ws.xr[k % XW_RING];
    const InferCtx::Grp gp = c.grp_of(k);
    if (ovl && k >= XW_RING) DTK_CUDA(cudaStreamWaitEvent(sb, choice.xa->freed[k % XW_RING], 0));   // chunk k - 4 is through
    {
      ProfRange pr(PROF_SAMPLE, sb);
      anchor_scalars_kernel<<<cdiv(cm.used, 256), 256, 0, sb>>>(c.T, ws.d_qlist, c.N, gp.f, gp.r, gp.map0, gp.item, cm.n_groups,
                                                               cm.used, c.N * c.T, x.row0, ws.u_norm, ws.u_flag, ws.u_rho,
                                                               c.fv.q_rho, xw_s8_slack(c.C), choice.s8, x.out_index, x.arow,
                                                               x.norm, x.eps);
      DTK_LAUNCHED();
      if (cm.n_gathered > 0) {
        const size_t r0 = (size_t)x.row0;
        gather_anchor_kernel<<<cm.gather_hi - cm.gather_lo, SAMPLE_THREADS, 0, sb>>>(
            c.fv.tpc, c.T, c.C, c.P, c.g.h, c.g.w, c.pa, traj, ws.d_qlist, c.N, gp.f, gp.r, gp.map0, gp.item, cm.n_groups,
            c.N * c.T, cm.gather_lo, c.fb, ws.u_hi, ws.u_lo, ws.u_flag, x.norm, ws.u_hi + r0 * c.C, ws.u_lo + r0 * c.C, ws.u_q8,
            ws.u_fac, c.fv.q_rho, xw_s8_slack(c.C), choice.s8 ? ws.u_q8 + r0 * c.C : nullptr, ws.u_fac + r0, x.eps);
        DTK_LAUNCHED();
      }
    }
    if (ovl) DTK_CUDA(cudaEventRecord(choice.xa->sample[k % XW_RING], sb));
    return DINOTRK_OK;
  }
  // works off the full-map queue
  int flush() {
    if (q_rows == 0) return DINOTRK_OK;
    const ChunkBufs& b = c.ws.cb[0];
    CorrAssist as;
    as.tkeys = b.tkeys; as.zero_word = b.hscratch; as.split_ready = true; as.no_thin = true; as.all_wide = true; as.small_tiles = true;
    const int* cg = c.ws.d_cgrp;
    const int sg = c.ws.sg_cap;
    int rc = launch_corr_maps(c.fv, nullptr, c.ch, b.norm, cg, cg + sg, cg + 2 * sg, cg + 3 * sg, q_groups, q_rows, q_rows,
                              b.maps, c.ms, c.ws.d_splan, b.split, c.st, as);
    if (rc) return rc;
    rc = launch_head(b.maps, q_rows, c.ms, c.g, c.hw, c.ws.out_index_ring[0], anchors, 2, 0, nullptr, b.hscratch, c.st, b.tkeys,
                     true);
    q_rows = q_groups = 0;
    return rc;
  }
  // waits for chunk j's head, counts its maps and appends the ones it queued to the full-map queue
  int finish(size_t j) {
    InferWs& ws = c.ws;
    XwAsync* xa = choice.xa;
    DTK_CUDA(cudaEventSynchronize(xa->done[j % XW_RING]));
    const int* cnt = xa->host_cnt + XW_CNT_CHUNK * (j % XW_RING);
    const int n_slow = cnt[0];
    g_infer_stats[infer_stat::full_map_by_certificate] += cnt[1];
    g_infer_stats[infer_stat::exact_box_tokens] += cnt[2]; g_infer_stats[infer_stat::exact_box_cells] += cnt[3];
    const ChunkMeta& cm = c.metas[j];
    const XwSet& x = ws.xr[j % XW_RING];
    const InferCtx::Grp gp = c.grp_of(j);
    DTK_CHECK_ARG(n_slow >= 0 && n_slow <= cm.used, "infer: corrupt full-map queue (%d of %d)", n_slow, cm.used);
    g_infer_stats[infer_stat::exact_window] += cm.used - n_slow; g_infer_stats[infer_stat::full_map] += n_slow;
    if (n_slow > 0) {
      if (q_rows + n_slow > c.ch || q_groups + cm.n_groups > ws.sg_cap) {
        int rc = flush();
        if (rc) return rc;
      }
      const ChunkBufs& b = ws.cb[0];
      const DescSplit d(b.split, c.ch, c.C);   // layout of a descriptor array of `ch` rows
      int rc = launch_xw_compact(nullptr, ws.u_hi, ws.u_lo, x.arow, x.norm, x.out_index, c.C, gp.f, gp.map0, cm.n_groups, n_slow,
                                 x.xc, nullptr, d.hi, d.lo, b.norm, ws.out_index_ring[0], ws.d_cgrp, ws.sg_cap, c.st, q_rows,
                                 q_groups, corr_hilo(c.fv));
      if (rc) return rc;
      q_rows += n_slow; q_groups += cm.n_groups;
    }
    DTK_CUDA(cudaEventRecord(xa->freed[j % XW_RING], c.st));
    return DINOTRK_OK;
  }
};

// Runs the exact-window pipeline over the planned chunks; done: how many it finished.  With a probe, chunk 0 is finished
// first, and its verdict may end the pipeline there (the caller then runs the rest on full maps) or move the rest to the
// fp16 coarse pass.
static int anchors_exact_window(InferCtx& c, AnchorChoice& choice, const float* traj, float* anchors, size_t& done) {
  InferWs& ws = c.ws;
  const cudaStream_t st = c.st;
  XwAsync* xa = choice.xa;
  CellPlan cp;
  plan_cells(c.T, c.gcap, c.metas, c.plan_host, cp);
  DTK_CHECK_ARG(cp.first.back() * 5 <= (size_t)c.N * c.T * ws.cell_nb * 5 + 16, "infer: cell plan exceeds its bound");
  if (!cp.v.empty()) DTK_CUDA(cudaMemcpyAsync(ws.d_cells, cp.v.data(), cp.v.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  if (!cp.tiles.empty()) DTK_CUDA(cudaMemcpyAsync(ws.d_tiles, cp.tiles.data(), cp.tiles.size() * sizeof(int), cudaMemcpyHostToDevice, st));
  InferAsync* ia = infer_async();
  const bool ovl = ia != nullptr && c.metas.size() > 1;
  ExactWindow pipe{c, choice, cp, ovl, ovl ? ia->side : st, traj, anchors};
  if (ovl) {
    DTK_CUDA(cudaEventRecord(ia->fork, st));
    DTK_CUDA(cudaStreamWaitEvent(pipe.sb, ia->fork, 0));
  }
  int rc;
  if (!c.metas.empty() && (rc = pipe.sample(0))) return rc;
  size_t n_finished = 0;
  done = c.metas.size();
  for (size_t k = 0; k < c.metas.size(); ++k) {
    const ChunkMeta& cm = c.metas[k];
    const XwSet& x = ws.xr[k % XW_RING];
    const InferCtx::Grp gp = c.grp_of(k);
    const XwCells cells = pipe.cells_of(k);
    if (ovl) DTK_CUDA(cudaStreamWaitEvent(st, xa->sample[k % XW_RING], 0));
    const float* eps = choice.s8 ? x.eps : nullptr;   // (nullptr: the fp16 pass's XW_EPS)
    g_infer_stats[infer_stat::desc_in_place] += cm.used - cm.n_gathered; g_infer_stats[infer_stat::desc_gathered] += cm.n_gathered;
    if ((rc = launch_xw_coarse(c.fv, ws.u_hi, (int)ws.xw_rows, ws.u_norm, gp.f, gp.r, gp.m, gp.map0, ws.d_tiles + k * (c.gcap + 1),
                               cm.n_groups, cm.used / TC2_BM_ROWS + cm.n_groups, x.xc, st, ws.d_rnorms,
                               choice.s8 ? ws.u_q8 : nullptr, ws.u_fac))) return rc;
    if ((rc = launch_xw_plan(cells, x.norm, cm.n_groups, c.g, x.xc, st, cm.used, split_min_norm(c.C), eps))) return rc;
    if ((rc = launch_xw_gemm(c.fv, c.g, ws.u_hi, ws.u_lo, (int)ws.xw_rows, cells, x.xc, st))) return rc;
    if ((rc = launch_xw_head(c.fv, c.g, c.hw, cells, x.norm, gp.map0, cm.used, x.out_index, anchors, 2, 0, x.xc, st, cm.n_groups,
                             eps)))
      return rc;
    DTK_CUDA(cudaMemcpyAsync(xa->host_cnt + XW_CNT_CHUNK * (k % XW_RING), x.xc.slow_cnt + cm.n_groups, XW_CNT_CHUNK * sizeof(int),
                             cudaMemcpyDeviceToHost, st));
    DTK_CUDA(cudaEventRecord(xa->done[k % XW_RING], st));
    if (k == 0 && choice.probe && c.metas.size() > 1) {   // the probe: wait for it, look at the certificate's verdicts
      if ((rc = pipe.finish(0))) return rc;
      n_finished = 1;
      if (choice.probe_says_full_maps(g_infer_stats[infer_stat::full_map_by_certificate], g_infer_stats[infer_stat::full_map], cm.used)) {
        done = 1;
        break;
      }
      g_infer_stats[infer_stat::coarse] = choice.s8 ? 1 : 0;
    }
    if (k + 1 < c.metas.size() && (rc = pipe.sample(k + 1))) return rc;
    while (n_finished + 2 <= k)
      if ((rc = pipe.finish(n_finished++))) return rc;
  }
  while (n_finished < done)
    if ((rc = pipe.finish(n_finished++))) return rc;
  if ((rc = pipe.flush())) return rc;
  if (ovl) {
    DTK_CUDA(cudaEventRecord(ia->join, pipe.sb));
    DTK_CUDA(cudaStreamWaitEvent(st, ia->join, 0));
  }
  return DINOTRK_OK;
}

// ---- phase C, full-map pipeline over chunks k0.. of the plan: the descriptors of chunk k + 1 are sampled on the side
// stream (buffer set (k + 1) & 1) while the caller's stream runs the split-precision GEMM over all tokens and the head's
// fast path of chunk k.  The full-map head of chunk j (usually an empty list) runs two chunks later, between two GEMMs: it
// needs ~70 KB of shared memory per CTA and could not co-reside with a GEMM anyway.
static int anchors_full_map(InferCtx& c, size_t k0, const float* traj, float* anchors) {
  InferWs& ws = c.ws;
  const cudaStream_t st = c.st;
  const bool tensor = c.fv.tensor();
  FeatView fv_split = c.fv;   // the sampler writes the separate halves: F16X3 here
  fv_split.hilo = nullptr;
  InferAsync* ia = infer_async();
  const bool ovl = ia != nullptr && c.metas.size() > k0 + 1;
  const cudaStream_t sb = ovl ? ia->side : st;   // sampling stream
  if (ovl) {
    DTK_CUDA(cudaEventRecord(ia->fork, st));
    DTK_CUDA(cudaStreamWaitEvent(sb, ia->fork, 0));
  }
  auto sample = [&](size_t k) -> int {   // descriptors of chunk k (buffer set k & 1)
    const ChunkMeta& cm = c.metas[k];
    const ChunkBufs& b = ws.cb[k & 1];
    const InferCtx::Grp gp = c.grp_of(k);
    if (ovl && k >= k0 + 2) DTK_CUDA(cudaStreamWaitEvent(sb, ia->gemm[k & 1], 0));   // GEMM k-2 read the descriptors of this set
    {
      ProfRange pr(PROF_SAMPLE, sb);
      const DescSplit d(b.split, cm.used, c.C);   // the split layout of launch_corr_gemm_tc for desc_rows = used
      __half* d_hi = tensor ? reinterpret_cast<__half*>(d.hi) : nullptr;
      __half* d_lo = tensor ? reinterpret_cast<__half*>(d.lo) : nullptr;
      sample_anchor_kernel<<<cm.used, SAMPLE_THREADS, 0, sb>>>(c.fv.tpc, c.T, c.C, c.P, c.g.h, c.g.w, c.pa, traj, ws.d_qlist, c.N,
                                                              gp.f, gp.map0, gp.item, cm.n_groups, c.fb, b.desc, b.norm,
                                                              ws.out_index_ring[k & 3], d_hi, d_lo);
      DTK_LAUNCHED();
    }
    if (ovl) DTK_CUDA(cudaEventRecord(ia->sample[k & 1], sb));
    return DINOTRK_OK;
  };
  auto head_full = [&](size_t j) {   // the last reader of chunk j's maps / keys / list
    const ChunkBufs& b = ws.cb[j & 1];
    return launch_head(b.maps, c.metas[j].used, c.ms, c.g, c.hw, ws.out_index_ring[j & 3], anchors, 2, 0, nullptr, b.hscratch,
                       st, tensor ? b.tkeys : nullptr, true, 2);
  };
  int rc;
  if (k0 < c.metas.size() && (rc = sample(k0))) return rc;
  for (size_t k = k0; k < c.metas.size(); ++k) {
    const ChunkMeta& cm = c.metas[k];
    const ChunkBufs& b = ws.cb[k & 1];
    const InferCtx::Grp gp = c.grp_of(k);
    if (ovl) DTK_CUDA(cudaStreamWaitEvent(st, ia->sample[k & 1], 0));
    if (k >= k0 + 2 && (rc = head_full(k - 2))) return rc;
    CorrAssist as;
    as.tkeys = tensor ? b.tkeys : nullptr; as.zero_word = b.hscratch; as.split_ready = tensor; as.no_thin = cm.no_thin;
    rc = launch_corr_maps(fv_split, b.desc, cm.used, b.norm, gp.f, gp.r, gp.m, gp.map0, cm.n_groups, cm.used, cm.maxm, b.maps,
                          c.ms, b.plan, b.split, st, as);
    if (rc) return rc;
    if (ovl) DTK_CUDA(cudaEventRecord(ia->gemm[k & 1], st));
    if (k + 1 < c.metas.size() && (rc = sample(k + 1))) return rc;
    rc = launch_head(b.maps, cm.used, c.ms, c.g, c.hw, ws.out_index_ring[k & 3], anchors, 2, 0, nullptr, b.hscratch, st, as.tkeys,
                     true, 1);
    if (rc) return rc;
  }
  for (size_t j = std::max(k0, c.metas.size() >= 2 ? c.metas.size() - 2 : 0); j < c.metas.size(); ++j)
    if ((rc = head_full(j))) return rc;
  return DINOTRK_OK;
}

// ---- phase C: anchor re-tracking.  The anchor lists, the choice of pipeline around the one host sync, then the exact-window
// pipeline and, when it does not run or its probe turns it down, the full-map pipeline.
static int infer_anchors(InferCtx& c, const float* traj, const float* cos_sims, float anchor_th, float* anchors, int n_counted_A) {
  NvtxRange nv("dinotrk.infer.C.anchors");
  InferWs& ws = c.ws;
  const cudaStream_t st = c.st;
  const int T = c.T, N = c.N;
  {
    ProfRange pr(PROF_ANCHOR_LIST, st);
    anchor_lists_kernel<<<T, ANCHOR_LIST_THREADS, 0, st>>>(cos_sims, N, T, anchor_th, ws.d_cnt, ws.d_qlist);
    DTK_LAUNCHED();
  }
  AnchorChoice choice(c.fv, c.g);
  XwAsync* xa = choice.xa;
  if (xa) {   // reciprocal token norms for the coarse epilogue + the smallest norm of the video (the choice reads it)
    int rc = launch_xw_rnorms(c.fv, ws.d_rnorms, ws.d_minnorm, st);
    if (rc) return rc;
    DTK_CUDA(cudaMemcpyAsync(xa->host_cnt + XW_CNT_MINNORM, ws.d_minnorm, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    if (n_counted_A > 0)
      DTK_CUDA(cudaMemcpyAsync(xa->host_cnt + XW_CNT_A, ws.d_cntA, (size_t)n_counted_A * sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  std::vector<int> cnt(T);
  DTK_CUDA(cudaMemcpyAsync(cnt.data(), ws.d_cnt, (size_t)T * sizeof(int), cudaMemcpyDeviceToHost, st));
  std::vector<float> rho_f(c.fv.s8() ? T : 0);
  if (c.fv.s8()) DTK_CUDA(cudaMemcpyAsync(rho_f.data(), c.fv.q_rho, (size_t)T * sizeof(float), cudaMemcpyDeviceToHost, st));
  std::vector<int> qlist_h, uflag_h;
  if (choice.xw) {
    // every (query, source frame) descriptor once, before the host waits (it depends on the trajectories only).  The
    // planner needs the anchor lists and the flags.
    {
      ProfRange pr(PROF_SAMPLE, st);
      sample_unique_kernel<<<N * T, SAMPLE_THREADS, 0, st>>>(c.fv.tpc, T, c.C, c.P, c.g.h, c.g.w, c.pa, traj, c.fb, ws.u_hi, ws.u_lo,
                                                             ws.u_norm, ws.u_flag, AnchorChoice::q8_rows(c.fv) ? ws.u_q8 : nullptr,
                                                             ws.u_fac, ws.u_rho);
      DTK_LAUNCHED();
    }
    qlist_h.resize((size_t)T * N); uflag_h.resize((size_t)N * T);
    DTK_CUDA(cudaMemcpyAsync(qlist_h.data(), ws.d_qlist, qlist_h.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
    DTK_CUDA(cudaMemcpyAsync(uflag_h.data(), ws.u_flag, uflag_h.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
  }
  DTK_CUDA(cudaStreamSynchronize(st));  // the one host sync: the anchor work lists
  choice.after_sync(c.C, n_counted_A, (long long)N * T);
  long long maps_C = 0;
  for (int a = 0; a < T; ++a) maps_C += (long long)cnt[a] * T;
  long long* stats = g_infer_stats;
  stats[infer_stat::anchor_maps] = maps_C; stats[infer_stat::exact_window] = 0; stats[infer_stat::full_map] = 0;
  stats[infer_stat::pipeline] = choice.xw ? 1 : 0; stats[infer_stat::full_map_by_certificate] = 0;
  stats[infer_stat::contraction] = c.fv.tensor() ? 1 : 0; stats[infer_stat::desc_in_place] = 0; stats[infer_stat::desc_gathered] = 0;
  stats[infer_stat::exact_box_cells] = 0; stats[infer_stat::exact_box_tokens] = 0;
  float rho_max = 0.f;
  for (float r : rho_f) rho_max = std::max(rho_max, r);
  int rc = choice.coarse_pass(c.fv, rho_max);
  if (rc) return rc;
  unsigned bits;
  memcpy(&bits, &rho_max, sizeof(bits));
  stats[infer_stat::coarse] = choice.s8 ? 1 : 0; stats[infer_stat::coarse_rho_f] = bits;
  // The probe is the same set of work items for every chunk size >= XW_PROBE_MAPS.
  const int probe_cap = choice.probe ? std::max(T, (XW_PROBE_MAPS / T) * T) : 0;
  size_t k0 = 0;   // first chunk of the full-map pipeline (> 0 after an exact-window probe)
  if (choice.xw) {
    std::vector<unsigned char> qflag(N, 0);   // a query with a flagged source frame is never read in place
    for (size_t u = 0; u < uflag_h.size(); ++u)
      if (uflag_h[u]) qflag[u / T] = 1;
    const AnchorRows rows{qlist_h.data(), qflag.data(), N * T, XW_RING, c.ch};
    DTK_CHECK_ARG(plan_chunks(1, T, N, cnt.data(), c.ch, c.gcap, c.metas, c.plan_host, T, probe_cap, &rows),
                  "infer: a chunk of the anchor phase has more than %d groups", c.gcap);
    if ((rc = c.upload_plan())) return rc;
    if ((rc = anchors_exact_window(c, choice, traj, anchors, k0))) return rc;
    if (k0 == c.metas.size()) return DINOTRK_OK;
    // switched: chunks k0.. on the full-map pipeline.  The same chunks, their rows per chunk again.  (Everything that read
    // the plan is in the caller's stream by now, so the upload is ordered behind it.)
    stats[infer_stat::pipeline] = 0; stats[infer_stat::coarse] = 0;
    plan_chunks(1, T, N, cnt.data(), c.ch, c.gcap, c.metas, c.plan_host, T, probe_cap);
  } else {
    plan_chunks(1, T, N, cnt.data(), c.ch, c.gcap, c.metas, c.plan_host);
  }
  if ((rc = c.upload_plan())) return rc;
  return anchors_full_map(c, k0, traj, anchors);
}

}  // namespace dtk

using namespace dtk;

extern "C" {

int dinotrk_infer_set_path(int path) {
  DTK_CHECK_ARG(path >= -1 && path <= 1, "infer_set_path: -1 (automatic), 0 (full-map GEMM + head) or 1 (coarse pass + exact window)");
  g_xw_path = path;
  return DINOTRK_OK;
}

int dinotrk_infer_set_coarse(int mode) {
  DTK_CHECK_ARG(mode >= -1 && mode <= 1, "infer_set_coarse: -1 (automatic), 0 (fp16) or 1 (int8)");
  g_xw_coarse = mode;
  return DINOTRK_OK;
}

int dinotrk_infer_last_stats(long long* out, int n) {
  DTK_CHECK_ARG(out && n >= 4, "infer_last_stats: need at least 4 slots");
  for (int i = 0; i < (n < infer_stat::count ? n : infer_stat::count); ++i) out[i] = g_infer_stats[i];
  return DINOTRK_OK;
}

static int infer_chunk_maps(int chunk_maps) { return chunk_maps > 0 ? chunk_maps : 4096; }
// chunks of the anchor phase hold whole (query, anchor frame) cells of T maps: never smaller than T
static int infer_chunk_eff(int chunk_maps, int T) { const int c = infer_chunk_maps(chunk_maps); return c > T ? c : T; }
// capacity of a chunk's group arrays.  Trajectory phase and full-map anchor phase: one group per frame.  Exact-window anchor
// phase: a frame's span is cut at its in-place runs, each of >= XW_INPLACE_MIN_ROWS rows, with at most one gathered group
// before each and one behind the last: <= T + 2 (ch / XW_INPLACE_MIN_ROWS) groups.
static int infer_gcap(int T, int ch) { return T + 2 + 2 * (ch / XW_INPLACE_MIN_ROWS + 1); }
// upper bound on the number of chunks of one phase (phase C has the most work items: N * T * T)
// (anchor-phase chunks are cut at whole cells of T maps: a full chunk holds at least the largest multiple of T <= ch)
static size_t infer_max_chunks(int T, int N, size_t ch) {
  size_t cap = (ch / (size_t)T) * (size_t)T;
  if (cap < (size_t)T) cap = T;
  return ((size_t)N * T * T + cap - 1) / cap + 2;
}

// (planner entry point: plain chunks of `chunk_maps` maps, cut anywhere)
size_t dinotrk_infer_max_chunks(int T, int N, int chunk_maps) {
  const size_t ch = (size_t)infer_chunk_maps(chunk_maps);
  return ((size_t)N * T * T + ch - 1) / ch + 2;
}

int dinotrk_infer_plan(int kind, int T, int N, const int* anchor_counts, int chunk_maps, int* groups, int* meta,
                       int max_chunks, int* n_chunks) {
  DTK_CHECK_ARG((kind == 0 || kind == 1) && T > 0 && N >= 0 && n_chunks, "infer_plan: bad arguments");
  DTK_CHECK_ARG(kind == 0 || anchor_counts, "infer_plan: kind 1 needs the per-frame anchor counts");
  const int ch = infer_chunk_maps(chunk_maps), gcap = T + 2;
  std::vector<ChunkMeta> metas;
  std::vector<int> plan_host;
  plan_chunks(kind, T, N, anchor_counts, ch, gcap, metas, plan_host);
  *n_chunks = (int)metas.size();
  DTK_CHECK_ARG((int)metas.size() <= max_chunks || (!groups && !meta), "infer_plan: %zu chunks, room for %d", metas.size(), max_chunks);
  if (groups) std::copy(plan_host.begin(), plan_host.end(), groups);
  if (meta)
    for (size_t k = 0; k < metas.size(); ++k) {
      meta[4 * k] = metas[k].used; meta[4 * k + 1] = metas[k].maxm; meta[4 * k + 2] = metas[k].n_groups;
      meta[4 * k + 3] = metas[k].no_thin ? 1 : 0;
    }
  return DINOTRK_OK;
}

int dinotrk_infer_anchor_gcap(int T, int chunk_maps) { return T > 0 ? infer_gcap(T, infer_chunk_eff(chunk_maps, T)) : 0; }

int dinotrk_infer_plan_anchors(int T, int N, const int* anchor_counts, const int* qlist, const unsigned char* query_flag,
                               int chunk_maps, int probe, int* groups, int* meta, int max_chunks, int* n_chunks) {
  DTK_CHECK_ARG(T > 0 && N >= 0 && anchor_counts && qlist && query_flag && n_chunks, "infer_plan_anchors: bad arguments");
  for (int a = 0; a < T; ++a) {
    DTK_CHECK_ARG(anchor_counts[a] >= 0 && anchor_counts[a] <= N, "infer_plan_anchors: count of frame %d out of range", a);
    for (int k = 0; k < anchor_counts[a]; ++k)
      DTK_CHECK_ARG(qlist[(size_t)a * N + k] >= 0 && qlist[(size_t)a * N + k] < N, "infer_plan_anchors: query out of range");
  }
  const int ch = infer_chunk_eff(chunk_maps, T), gcap = infer_gcap(T, ch);
  const AnchorRows rows{qlist, query_flag, N * T, XW_RING, ch};
  std::vector<ChunkMeta> metas;
  std::vector<int> plan_host;
  const bool fits = plan_chunks(1, T, N, anchor_counts, ch, gcap, metas, plan_host, T,
                                probe ? std::max(T, (XW_PROBE_MAPS / T) * T) : 0, &rows);
  DTK_CHECK_ARG(fits, "infer_plan_anchors: a chunk has more than %d groups", gcap);
  *n_chunks = (int)metas.size();
  DTK_CHECK_ARG((int)metas.size() <= max_chunks || (!groups && !meta), "infer_plan_anchors: %zu chunks, room for %d", metas.size(), max_chunks);
  if (groups) std::copy(plan_host.begin(), plan_host.end(), groups);
  if (meta)
    for (size_t k = 0; k < metas.size(); ++k) {
      meta[5 * k] = metas[k].used; meta[5 * k + 1] = metas[k].maxm; meta[5 * k + 2] = metas[k].n_groups;
      meta[5 * k + 3] = metas[k].no_thin ? 1 : 0; meta[5 * k + 4] = metas[k].n_gathered;
    }
  return DINOTRK_OK;
}

int dinotrk_infer_set_overlap(int mode) {
  DTK_CHECK_ARG(mode >= -1 && mode <= 1, "infer_set_overlap: mode must be -1 (default), 0 or 1");
  g_overlap_mode = mode;
  return DINOTRK_OK;
}

size_t dinotrk_corr_track_workspace_bytes(int total_maps, int n_groups, int C, const dinotrk_geom* g) {
  if (!g) return 0;
  return align_up(layout_end<CorrTrackWs>(total_maps, n_groups, C, dinotrk_map_stride(g)), 256) + 1024;
}

int dinotrk_corr_track(const dinotrk_features* feat, const dinotrk_geom* g,
                       const dinotrk_head_weights* hw, const float* desc, const float* desc_norm,
                       const int* grp_frame, const int* grp_row0, const int* grp_m, const int* grp_map0,
                       int n_groups, int total_maps, int max_group_m, const int* out_index, float* out,
                       int out_stride, int out_mode, void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(feat && feat->tpc && feat->norms && g && hw && desc && desc_norm && grp_frame && grp_row0 && grp_m &&
                grp_map0 && out, "corr_track: null pointer");
  const int C = feat->C;
  DTK_CHECK_ARG(feat->T > 0 && C > 0 && C % 4 == 0 && n_groups >= 0 && total_maps >= 0, "corr_track: bad sizes");
  DTK_CHECK_ARG((feat->hi == nullptr) == (feat->lo == nullptr), "corr_track: hi and lo must be given together");
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_corr_track_workspace_bytes(total_maps, n_groups, C, g),
                "corr_track: workspace too small");
  if (total_maps == 0) return DINOTRK_OK;
  const int ms = dinotrk_map_stride(g);
  Arena ar(workspace);
  const CorrTrackWs ws(ar, total_maps, n_groups, C, ms);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = launch_corr_maps(make_view(*feat, *g), desc, total_maps, desc_norm, grp_frame, grp_row0, grp_m, grp_map0,
                            n_groups, total_maps, max_group_m, ws.maps, ms, ws.corr.plan, ws.corr.split, st);
  if (rc) return rc;
  return launch_head(ws.maps, total_maps, ms, *g, *hw, out_index, out, out_stride, out_mode, nullptr, ws.hscratch, st);
}


size_t dinotrk_infer_workspace_bytes(int T, int C, const dinotrk_geom* g, int N, int chunk_maps) {
  if (!g) return 0;
  const int ch = infer_chunk_eff(chunk_maps, T);
  const size_t end = layout_end<InferWs>(T, C, N, g->h * g->w, dinotrk_map_stride(g), ch, infer_gcap(T, ch),
                                         infer_max_chunks(T, N, (size_t)ch));
  return align_up(end, 256) + 25088;
}

int dinotrk_traj_cos_sims(const float* tpc, int T, int C, const dinotrk_geom* g, const float* traj,
                          const float* query_points, int N, float* cos_sims, void* workspace,
                          size_t workspace_bytes, void* stream) {
  (void)workspace; (void)workspace_bytes;
  DTK_CHECK_ARG(tpc && g && traj && query_points && cos_sims, "traj_cos_sims: null pointer");
  DTK_CHECK_ARG(T > 0 && C > 0 && C % 4 == 0 && N >= 0, "traj_cos_sims: bad sizes");
  if (N == 0) return DINOTRK_OK;
  size_t smem = (size_t)2 * C * sizeof(float);
  static PerDev<size_t> attr_dev;
  size_t& attr = attr_dev.get();
  if (smem > 48 * 1024 && smem > attr) {
    DTK_CUDA(cudaFuncSetAttribute(traj_cos_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  ProfRange pr(PROF_COS, (cudaStream_t)stream);
  traj_cos_kernel<<<dim3(T, N), SAMPLE_THREADS, smem, (cudaStream_t)stream>>>(
      tpc, T, C, g->h * g->w, g->h, g->w, make_point_affine(*g), traj, query_points, cos_sims);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_occlusion(const float* traj, const float* cos_sims, const float* anchors, int N, int T,
                      float anchor_th, float cos_th, uint8_t* occ, void* stream) {
  DTK_CHECK_ARG(traj && cos_sims && anchors && occ && N >= 0 && T > 0, "occlusion: bad args");
  if (N == 0) return DINOTRK_OK;
  size_t smem = (size_t)(4 + OCC_THREADS / 32) * T * sizeof(float);
  DTK_CHECK_ARG(smem <= 200 * 1024, "occlusion: T=%d too large", T);
  static PerDev<size_t> attr_dev;
  size_t& attr = attr_dev.get();
  if (smem > 48 * 1024 && smem > attr) {
    DTK_CUDA(cudaFuncSetAttribute(occlusion_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr = smem;
  }
  ProfRange pr(PROF_OCCLUSION, (cudaStream_t)stream);
  occlusion_kernel<<<N, OCC_THREADS, smem, (cudaStream_t)stream>>>(traj, cos_sims, anchors, T, anchor_th, cos_th, occ);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_infer(const dinotrk_features* feat, const dinotrk_geom* g,
                  const dinotrk_head_weights* hw, const float* query_points, int N, float anchor_th, float cos_th,
                  int frame_batch, int start_phase, int stop_after, int chunk_maps, float* traj, float* cos_sims,
                  float* anchors,
                  uint8_t* occ, void* workspace, size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(feat && feat->tpc && feat->norms && g && hw && query_points && traj, "infer: null pointer");
  const int T = feat->T, C = feat->C;
  DTK_CHECK_ARG(T > 0 && C > 0 && C % 4 == 0 && N >= 0, "infer: bad sizes");
  DTK_CHECK_GRID(*g, "infer");
  DTK_CHECK_ARG((feat->hi == nullptr) == (feat->lo == nullptr), "infer: hi and lo must be given together");
  const FeatView fv = make_view(*feat, *g);
  DTK_CHECK_ARG(start_phase >= 0 && start_phase <= stop_after && stop_after <= 3,
                "infer: need 0 <= start_phase <= stop_after <= 3");
  DTK_CHECK_ARG((stop_after < 1 || cos_sims) && (stop_after < 2 || anchors) && (stop_after < 3 || occ),
                "infer: missing output buffer for the requested phases");
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_infer_workspace_bytes(T, C, g, N, chunk_maps),
                "infer: workspace too small (%zu < %zu)", workspace_bytes,
                dinotrk_infer_workspace_bytes(T, C, g, N, chunk_maps));
  if (N == 0) return DINOTRK_OK;
  const int P = g->h * g->w, ms = dinotrk_map_stride(g);
  const int ch = infer_chunk_eff(chunk_maps, T);
  const int fb = frame_batch > 0 ? (frame_batch < T ? frame_batch : T) : T;
  const int gcap = infer_gcap(T, ch);
  const size_t max_chunks = infer_max_chunks(T, N, (size_t)ch);
  Arena ar(workspace);
  InferWs ws(ar, T, C, N, P, ms, ch, gcap, max_chunks);
  DTK_CHECK_ARG(ws.xw_rows <= 0x7fffffffu, "infer: %zu descriptor rows exceed the row index", ws.xw_rows);
  InferCtx c{fv, *g, *hw, ws, (cudaStream_t)stream, T, C, N, P, ms, ch, gcap, fb, max_chunks, make_point_affine(*g)};

  int rc, n_counted_A = 0;
  if (start_phase <= 0 && (rc = infer_trajectories(c, query_points, traj, n_counted_A))) return rc;
  if (stop_after < 1) return DINOTRK_OK;
  if (start_phase <= 1) {   // ---- phase B: cosine similarities along the trajectories
    NvtxRange nv("dinotrk.infer.B.cos_sims");
    if ((rc = dinotrk_traj_cos_sims(feat->tpc, T, C, g, traj, query_points, N, cos_sims, nullptr, 0, stream))) return rc;
  }
  if (stop_after < 2) return DINOTRK_OK;
  if (start_phase <= 2 && (rc = infer_anchors(c, traj, cos_sims, anchor_th, anchors, n_counted_A))) return rc;
  if (stop_after < 3) return DINOTRK_OK;
  NvtxRange nv("dinotrk.infer.D.occlusion");   // ---- phase D: occlusion
  return dinotrk_occlusion(traj, cos_sims, anchors, N, T, anchor_th, cos_th, occ, stream);
}

}  // extern "C"

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

// descriptors of one chunk of anchor work items.  Group k of the chunk covers items
// [grp_item0[k], grp_item0[k] + grp_m[k]) of anchor frame grp_frame[k]; item u = (query slot u / T, frame u % T).
// Source point traj[n][i] lives in frame i; frames_set = [a, i0..e-1] (model_inference.py:138-143).
__global__ void sample_anchor_kernel(const float* __restrict__ tpc, int T, int C, int P, int h, int w, PointAffine pa,
                                     const float* __restrict__ traj, const int* __restrict__ qlist, int N,
                                     const int* __restrict__ grp_frame, const int* __restrict__ grp_map0,
                                     const int* __restrict__ grp_item0, int n_groups, int frame_batch,
                                     float* __restrict__ desc, float* __restrict__ dnorm, int* __restrict__ out_index,
                                     __half* __restrict__ desc_hi, __half* __restrict__ desc_lo) {
  const int j = blockIdx.x;
  const int lo = last_le(n_groups, j, grp_map0);
  const int a = grp_frame[lo];
  const int u = grp_item0[lo] + (j - grp_map0[lo]);
  const int slot = u / T, i = u - slot * T;
  const int n = qlist[(size_t)a * N + slot];
  const int i0 = (i / frame_batch) * frame_batch, e = min(i0 + frame_batch, T);
  const int Nset = e - i0 + 1;
  const float* pt = traj + ((size_t)n * T + i) * 3;
  float x = __fadd_rn(__fmul_rn(pa.aw, pt[0]), pa.bw);
  float y = __fadd_rn(__fmul_rn(pa.ah, pt[1]), pa.bh);
  TriCorners c = tri_setup(x, y, (float)(i - i0 + 1), Nset, h, w);
  int f0 = c.z0 == 0 ? a : i0 + c.z0 - 1;
  int f1 = c.z1 < 0 ? -1 : (c.z1 == 0 ? a : i0 + c.z1 - 1);
  sample_point(tpc, C, P, c, f0, f1, desc + (size_t)j * C, dnorm + j, desc_hi ? desc_hi + (size_t)j * C : nullptr,
               desc_lo ? desc_lo + (size_t)j * C : nullptr);
  if (threadIdx.x == 0) out_index[j] = (n * T + a) * T + i;
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
  const int i = u % T;
  const int i0 = (i / frame_batch) * frame_batch, e = min(i0 + frame_batch, T);
  const float* pt = traj + (size_t)u * 3;
  float x = __fadd_rn(__fmul_rn(pa.aw, pt[0]), pa.bw);
  float y = __fadd_rn(__fmul_rn(pa.ah, pt[1]), pa.bh);
  TriCorners c = tri_setup(x, y, (float)(i - i0 + 1), e - i0 + 1, h, w);
  bool slot0 = false;
#pragma unroll
  for (int k = 0; k < 4; ++k) slot0 = slot0 || (c.z0 == 0 && c.tok[k] >= 0 && c.wxy[k][0] != 0.f);
  if (threadIdx.x == 0) u_flag[u] = slot0 ? 1 : 0;
  if (slot0) return;                        // depends on the anchor frame: sampled per work item
  const int f0 = i0 + c.z0 - 1;
  const int f1 = c.z1 < 0 ? -1 : i0 + c.z1 - 1;
  sample_point(tpc, C, P, c, f0, f1, nullptr, u_norm + u, u_hi + (size_t)u * C, u_lo + (size_t)u * C);
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
  const int a = grp_frame[lo];
  const int uu = grp_item0[lo] + (j - grp_map0[lo]);
  const int slot = uu / T, i = uu - slot * T;
  const int n = qlist[(size_t)a * N + slot];
  const size_t u = (size_t)n * T + i;
  out_index[j] = (n * T + a) * T + i;
  const int r0 = grp_row0[lo];
  arow[j] = r0 < n_unique ? r0 + (j - grp_map0[lo]) : chunk_row0 + j;
  if (u_flag[u]) return;   // sampled per work item: gather_anchor_kernel writes the norm and eps
  dnorm[j] = u_norm[u];
  if (with_eps) desc_eps[j] = xw_eps_s8(u_rho[u], rho_f[a], eps_slack);
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
  const int a = grp_frame[lo];
  const int uu = grp_item0[lo] + (j - grp_map0[lo]);
  const int slot = uu / T, i = uu - slot * T;
  const int n = qlist[(size_t)a * N + slot];
  const size_t u = (size_t)n * T + i;
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
  const int i0 = (i / frame_batch) * frame_batch, e = min(i0 + frame_batch, T);
  const float* pt = traj + u * 3;
  float x = __fadd_rn(__fmul_rn(pa.aw, pt[0]), pa.bw);
  float y = __fadd_rn(__fmul_rn(pa.ah, pt[1]), pa.bh);
  TriCorners c = tri_setup(x, y, (float)(i - i0 + 1), e - i0 + 1, h, w);
  int f0 = c.z0 == 0 ? a : i0 + c.z0 - 1;
  int f1 = c.z1 < 0 ? -1 : (c.z1 == 0 ? a : i0 + c.z1 - 1);
  sample_point(tpc, C, P, c, f0, f1, nullptr, dnorm + j, desc_hi + (size_t)j * C, desc_lo + (size_t)j * C);
  if (desc_q8) {
    const float r = quant_desc(desc_hi + (size_t)j * C, desc_lo + (size_t)j * C, C, dnorm + j, desc_q8 + (size_t)j * C, desc_fac + j);
    if (threadIdx.x == 0) desc_eps[j] = xw_eps_s8(r, rho_f[a], eps_slack);
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

// auxiliary stream + events of the phase-C pipeline (one set per process; DTK_OVERLAP=0 disables the overlap)
struct InferAsync {
  int mode;                 // 1: sampling overlapped with the GEMMs (default); 2: sampling and the head fast path
  cudaStream_t aux, aux2;   // head stream, sampling stream
  cudaEvent_t fork, join, sample[2], gemm[2], head[2];
  int head_ctas_per_sm;
};
static int g_overlap_mode = -1;   // -1: DTK_OVERLAP or the default (1); see dinotrk_infer_set_overlap
struct InferAsyncSlot { InferAsync ia; int state; };   // state 0: not created, 1: ready, -1: creation failed
static InferAsync* infer_async() {
  static PerDev<InferAsyncSlot> slots;   // streams and events belong to the device they were created on
  InferAsyncSlot& slot = slots.get();
  InferAsync& ia = slot.ia;
  int& state = slot.state;
  int mode = g_overlap_mode;
  if (mode < 0) {
    const char* e = getenv("DTK_OVERLAP");
    mode = e ? atoi(e) : 1;
  }
  if (mode <= 0) return nullptr;
  if (state == 0) {
    state = -1;
    const char* hc = getenv("DTK_HEAD_OVERLAP_CTAS");
    ia.head_ctas_per_sm = hc ? atoi(hc) : 2;
    if (cudaStreamCreateWithFlags(&ia.aux, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    if (cudaStreamCreateWithFlags(&ia.aux2, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    cudaEvent_t* evs[] = {&ia.fork, &ia.join, &ia.sample[0], &ia.sample[1], &ia.gemm[0], &ia.gemm[1], &ia.head[0], &ia.head[1]};
    for (cudaEvent_t* ev : evs)
      if (cudaEventCreateWithFlags(ev, cudaEventDisableTiming) != cudaSuccess) return nullptr;
    state = 1;
  }
  if (state != 1) return nullptr;
  ia.mode = mode;
  return &ia;
}

// events, pinned counters and selection of the exact-window pipeline (one set per device)
constexpr int XW_RING = 4;
constexpr int XW_PROBE_MAPS = 4096;   // size of the probe chunk (automatic pipeline choice)
struct XwAsync {
  int state;                                   // 0: not created, 1: ready, -1: failed
  cudaEvent_t sample[XW_RING], done[XW_RING], freed[XW_RING];
  int* host_cnt;                               // pinned: [XW_RING][2] queue totals / uncertified + [16] phase-A uncertified counts
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
    if (cudaHostAlloc(&xa.host_cnt, (2 * XW_RING + 16 + 4) * sizeof(int), cudaHostAllocDefault) != cudaSuccess) return nullptr;
    xa.state = 1;
  }
  return xa.state == 1 ? &xa : nullptr;
}
static int g_xw_path = -1;                     // -1: automatic (DTK_XW or on), 0: full-map path only, 1: exact-window path
static int g_xw_coarse = -1;                   // -1: automatic, 0: fp16 coarse pass, 1: int8 coarse pass
// anchor-phase maps | on the exact-window path | queued | path used | queued by the certificate | tensor-core contraction |
// int8 coarse pass | bits of the largest per-frame int8 residual | exact-window maps whose descriptor was read in place from
// the unique table | those gathered into the chunk's rows
constexpr int INFER_STATS = 10;
static long long g_infer_stats[INFER_STATS] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
// the probe chunk queues more than this fraction of its maps on the int8 coarse pass: the rest of the phase runs the fp16
// pass.  A queued map costs a full-map split-precision GEMM, ~3 fp16 coarse passes, while the int8 pass saves about half
// of one per map: int8 loses above ~1/6 extra queued maps.  1/16 leaves a wide margin.
constexpr int XW_S8_PROBE_QUEUE_DIV = 16;

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
  for (int i = 0; i < (n < INFER_STATS ? n : INFER_STATS); ++i) out[i] = g_infer_stats[i];
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
  DTK_CHECK_ARG(mode >= -1 && mode <= 2, "infer_set_overlap: mode must be -1 (default / DTK_OVERLAP), 0, 1 or 2");
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
  const float* tpc = feat->tpc;
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
  cudaStream_t st = (cudaStream_t)stream;
  const int P = g->h * g->w, ms = dinotrk_map_stride(g);
  const int ch = infer_chunk_eff(chunk_maps, T);
  const int fb = frame_batch > 0 ? (frame_batch < T ? frame_batch : T) : T;
  const int gcap = infer_gcap(T, ch);
  const PointAffine pa = make_point_affine(*g);

  const size_t max_chunks = infer_max_chunks(T, N, (size_t)ch);
  Arena ar(workspace);
  InferWs ws(ar, T, C, N, P, ms, ch, gcap, max_chunks);
  const int n_unique = N * T;
  DTK_CHECK_ARG(ws.xw_rows <= 0x7fffffffu, "infer: %zu descriptor rows exceed the row index", ws.xw_rows);
  const bool tensor = fv.tensor();   // tensor-core GEMM: tile keys for the head, fp16 split fused into the samplers
  FeatView fv_split = fv;            // the full-map pipeline's sampler writes the separate halves: F16X3 there
  fv_split.hilo = nullptr;

  // The chunks of a phase are planned on the host in one go and their group arrays uploaded with ONE copy, so the
  // per-chunk launches below never block the host (a pageable cudaMemcpyAsync per chunk would).
  std::vector<ChunkMeta> metas;
  std::vector<int> plan_host;
  auto upload_plan = [&]() -> int {
    DTK_CHECK_ARG(metas.size() <= max_chunks, "infer: chunk plan exceeds its bound (%zu > %zu)", metas.size(), max_chunks);
    if (!plan_host.empty())
      DTK_CUDA(cudaMemcpyAsync(ws.d_groups, plan_host.data(), plan_host.size() * sizeof(int), cudaMemcpyHostToDevice, st));
    return DINOTRK_OK;
  };
  struct Grp { const int *f, *r, *m, *map0, *item; };
  auto grp_of = [&](size_t k) {
    const int* b = ws.d_groups + k * 5 * gcap;
    return Grp{b, b + gcap, b + 2 * gcap, b + 3 * gcap, b + 4 * gcap};
  };

  int n_chunks_A = 0;
  long long maps_A = 0;
  // ---- phase A: trajectories -------------------------------------------------------------------
  if (start_phase <= 0) {
    NvtxRange nv("dinotrk.infer.A.trajectories");
    {
      ProfRange pr(PROF_SAMPLE, st);
      sample_query_kernel<<<N, SAMPLE_THREADS, 0, st>>>(tpc, T, C, P, g->h, g->w, pa, query_points, ws.descA, ws.normA);
      DTK_LAUNCHED();
    }
    if (tensor) {   // the query descriptors are reused by every chunk: split them once (layout of desc_rows = N)
      for (int k = 0; k < 2; ++k) {
        const DescSplit a(ws.cb[k].split, N, C);
        int rc = corr_hilo(fv) ? launch_split_hilo(ws.descA, a.hi, N, C, st)
                               : launch_split_f16(ws.descA, a.hi, a.lo, (size_t)N * C, st);
        if (rc) return rc;
      }
    }
    plan_chunks(0, T, N, nullptr, ch, gcap, metas, plan_host);
    int rc = upload_plan();
    if (rc) return rc;
    for (size_t k = 0; k < metas.size(); ++k) {
      const ChunkMeta& cm = metas[k];
      const ChunkBufs& b = ws.cb[k & 1];
      const Grp gp = grp_of(k);
      {
        ProfRange pr(PROF_MISC, st);
        index_traj_kernel<<<cdiv(cm.used, 256), 256, 0, st>>>(gp.f, gp.r, gp.map0, cm.n_groups, cm.used, T, ws.out_index_ring[k & 3], traj);
        DTK_LAUNCHED();
      }
      CorrAssist as;
      as.tkeys = tensor ? b.tkeys : nullptr; as.zero_word = b.hscratch; as.split_ready = tensor; as.no_thin = cm.no_thin;
      rc = launch_corr_maps(fv, ws.descA, N, ws.normA, gp.f, gp.r, gp.m, gp.map0, cm.n_groups, cm.used, cm.maxm, b.maps, ms, b.plan,
                            b.split, st, as);
      if (rc) return rc;
      rc = launch_head(b.maps, cm.used, ms, *g, *hw, ws.out_index_ring[k & 3], traj, 3, 0, nullptr, b.hscratch, st, as.tkeys, true);
      if (rc) return rc;
      if (k < 16)   // uncertified maps of this chunk: the anchor phase chooses its pipeline from their share
        DTK_CUDA(cudaMemcpyAsync(ws.d_cntA + k, b.hscratch, sizeof(int), cudaMemcpyDeviceToDevice, st));
    }
    n_chunks_A = (int)std::min<size_t>(metas.size(), 16);
    maps_A = (long long)N * T;
  }
  if (stop_after < 1) return DINOTRK_OK;

  // ---- phase B: cosine similarities along the trajectories --------------------------------------
  if (start_phase <= 1) {
    NvtxRange nv("dinotrk.infer.B.cos_sims");
    int rc = dinotrk_traj_cos_sims(tpc, T, C, g, traj, query_points, N, cos_sims, nullptr, 0, stream);
    if (rc) return rc;
  }
  if (stop_after < 2) return DINOTRK_OK;

  // ---- phase C: anchor re-tracking ---------------------------------------------------------------
  // Three streams: the caller's stream runs the correlation GEMMs back to back; one auxiliary stream samples the
  // descriptors of chunk k+1, another runs the head of chunk k, both while the GEMM of chunk k+1 owns the tensor cores
  // (the head kernel is then launched with one CTA per SM so that it fits next to the GEMM's ~200 KB of shared memory;
  // the rare full-map head launches cannot co-reside and simply wait for the GEMM's CTAs to retire).
  if (start_phase <= 2) {
    NvtxRange nv("dinotrk.infer.C.anchors");
    {
      ProfRange pr(PROF_ANCHOR_LIST, st);
      anchor_lists_kernel<<<T, ANCHOR_LIST_THREADS, 0, st>>>(cos_sims, N, T, anchor_th, ws.d_cnt, ws.d_qlist);
      DTK_LAUNCHED();
    }
    std::vector<int> cnt(T);
    // pipeline of the anchor phase: coarse pass + exact window (xwin.cuh) on the tensor path, unless disabled
    bool use_xw = tensor && disc_fits_box(*g);
    int pathsel = g_xw_path;
    if (pathsel < 0) { const char* e = getenv("DTK_XW"); if (e) pathsel = atoi(e) != 0 ? 1 : 0; }
    if (pathsel == 0) use_xw = false;
    XwAsync* xa = use_xw ? xw_async() : nullptr;
    if (!xa) use_xw = false;
    if (xa) {   // reciprocal token norms for the coarse epilogue + the smallest norm of the video (the host reads it below)
      int rcn = launch_xw_rnorms(fv, ws.d_rnorms, ws.d_minnorm, st);
      if (rcn) return rcn;
      DTK_CUDA(cudaMemcpyAsync(xa->host_cnt + 2 * XW_RING + 16, ws.d_minnorm, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    }
    if (xa && n_chunks_A > 0)
      DTK_CUDA(cudaMemcpyAsync(xa->host_cnt + 2 * XW_RING, ws.d_cntA, (size_t)n_chunks_A * sizeof(int), cudaMemcpyDeviceToHost, st));
    DTK_CUDA(cudaMemcpyAsync(cnt.data(), ws.d_cnt, (size_t)T * sizeof(int), cudaMemcpyDeviceToHost, st));
    std::vector<float> rho_f(fv.s8() ? T : 0);
    if (fv.s8()) DTK_CUDA(cudaMemcpyAsync(rho_f.data(), fv.q_rho, (size_t)T * sizeof(float), cudaMemcpyDeviceToHost, st));
    std::vector<int> qlist_h, uflag_h;
    if (use_xw) {
      // every (query, source frame) descriptor once, before the host waits (it depends on the trajectories only); with the
      // int8 rows whenever the int8 coarse pass can still be chosen.  The planner needs the anchor lists and the flags.
      const bool q8 = fv.s8() && g_xw_coarse != 0 && C % 16 == 0 && C <= XW_S8_MAX_C;
      {
        ProfRange pr(PROF_SAMPLE, st);
        sample_unique_kernel<<<N * T, SAMPLE_THREADS, 0, st>>>(tpc, T, C, P, g->h, g->w, pa, traj, fb, ws.u_hi, ws.u_lo, ws.u_norm, ws.u_flag,
                                                               q8 ? ws.u_q8 : nullptr, ws.u_fac, ws.u_rho);
        DTK_LAUNCHED();
      }
      qlist_h.resize((size_t)T * N); uflag_h.resize((size_t)N * T);
      DTK_CUDA(cudaMemcpyAsync(qlist_h.data(), ws.d_qlist, qlist_h.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
      DTK_CUDA(cudaMemcpyAsync(uflag_h.data(), ws.u_flag, uflag_h.size() * sizeof(int), cudaMemcpyDeviceToHost, st));
    }
    DTK_CUDA(cudaStreamSynchronize(st));  // the one host sync: the anchor work lists
    if (use_xw) {   // a token below the split's faithful range (a zero one included) voids the coarse pass's error bound
      float mn;
      memcpy(&mn, xa->host_cnt + 2 * XW_RING + 16, sizeof(float));
      if (!(mn >= split_min_norm(C))) use_xw = false;
    }
    if (use_xw && pathsel < 0 && n_chunks_A > 0) {
      // head weights the certificate cannot handle send (almost) every map to the full-map kernels anyway: the trajectory
      // phase just showed it; skip the exact-window attempt then.  (Depends on the weights and the video only.)
      long long unc = 0;
      for (int k = 0; k < n_chunks_A; ++k) unc += xa->host_cnt[2 * XW_RING + k];
      if (unc * 4 > maps_A) use_xw = false;
    }
    long long maps_C = 0;
    for (int a = 0; a < T; ++a) maps_C += (long long)cnt[a] * T;
    g_infer_stats[0] = maps_C; g_infer_stats[1] = 0; g_infer_stats[2] = 0; g_infer_stats[3] = use_xw ? 1 : 0; g_infer_stats[4] = 0;
    g_infer_stats[5] = tensor ? 1 : 0; g_infer_stats[8] = 0; g_infer_stats[9] = 0;
    // coarse pass of the exact-window pipeline (decided once use_xw is final): int8 when the features carry their int8
    // operands (forced: required), unless a frame's residual makes the bound too loose (automatic mode; below: or the probe
    // chunk queues too many maps)
    DTK_CHECK_ARG(g_xw_coarse != 1 || !use_xw || fv.s8(), "infer: int8 coarse pass forced without the int8 features");
    bool s8 = use_xw && fv.s8() && g_xw_coarse != 0;
    DTK_CHECK_ARG(!s8 || (C % 16 == 0 && C <= XW_S8_MAX_C), "infer: int8 coarse pass needs C %% 16 == 0 and C <= %d", XW_S8_MAX_C);
    {
      float rho_max = 0.f;
      for (float r : rho_f) rho_max = std::max(rho_max, r);
      if (g_xw_coarse < 0 && !(rho_max <= XW_S8_RHO_MAX)) s8 = false;
      unsigned bits;
      memcpy(&bits, &rho_max, sizeof(bits));
      g_infer_stats[6] = s8 ? 1 : 0; g_infer_stats[7] = bits;
    }
    size_t k0 = 0;            // first chunk of the full-map pipeline (> 0 after an exact-window probe)
    bool planned = false;
    if (use_xw) {
      // automatic mode: the first chunk is a small probe; if the head's certificate sends more than a quarter of it to the
      // full-map queue (refiner weights whose outside-the-box logit bound needs the exact map), the rest of the phase runs
      // the full-map pipeline directly.  The probe is the same set of work items for every chunk size >= XW_PROBE_MAPS.
      const bool probing = pathsel < 0;
      const int probe_cap = std::max(T, (XW_PROBE_MAPS / T) * T);
      std::vector<unsigned char> qflag(N, 0);   // a query with a flagged source frame is never read in place
      for (size_t u = 0; u < uflag_h.size(); ++u)
        if (uflag_h[u]) qflag[u / T] = 1;
      const AnchorRows rows{qlist_h.data(), qflag.data(), n_unique, XW_RING, ch};
      DTK_CHECK_ARG(plan_chunks(1, T, N, cnt.data(), ch, gcap, metas, plan_host, T, probing ? probe_cap : 0, &rows),
                    "infer: a chunk of the anchor phase has more than %d groups", gcap);
      int rc = upload_plan();
      if (rc) return rc;
      planned = true;
      CellPlan cp;
      plan_cells(T, gcap, metas, plan_host, cp);
      DTK_CHECK_ARG(cp.first.back() * 5 <= (size_t)N * T * ws.cell_nb * 5 + 16, "infer: cell plan exceeds its bound");
      if (!cp.v.empty()) DTK_CUDA(cudaMemcpyAsync(ws.d_cells, cp.v.data(), cp.v.size() * sizeof(int), cudaMemcpyHostToDevice, st));
      if (!cp.tiles.empty()) DTK_CUDA(cudaMemcpyAsync(ws.d_tiles, cp.tiles.data(), cp.tiles.size() * sizeof(int), cudaMemcpyHostToDevice, st));
      InferAsync* ia = infer_async();
      const bool ovl = ia != nullptr && metas.size() > 1;
      cudaStream_t sb = ovl ? ia->aux2 : st;   // sampling stream
      if (ovl) {
        DTK_CUDA(cudaEventRecord(ia->fork, st));
        DTK_CUDA(cudaStreamWaitEvent(sb, ia->fork, 0));
      }
      auto cells_of = [&](size_t k) {
        XwCells c;
        const int n = (int)(cp.first[k + 1] - cp.first[k]);
        const int* base = ws.d_cells + 5 * cp.first[k];
        c.row0 = base; c.m = base + n; c.frame = base + 2 * n; c.group = base + 3 * n; c.arow = base + 4 * n;
        c.n_cells = n; c.max_m = cp.max_m;
        return c;
      };
      auto enqueue_sample_x = [&](size_t k) -> int {
        const ChunkMeta& cm = metas[k];
        const XwSet& x = ws.xr[k % XW_RING];
        const Grp gp = grp_of(k);
        if (ovl && k >= XW_RING) DTK_CUDA(cudaStreamWaitEvent(sb, xa->freed[k % XW_RING], 0));   // chunk k - 4 is through
        {
          ProfRange pr(PROF_SAMPLE, sb);
          anchor_scalars_kernel<<<cdiv(cm.used, 256), 256, 0, sb>>>(T, ws.d_qlist, N, gp.f, gp.r, gp.map0, gp.item, cm.n_groups, cm.used,
                                                                   n_unique, x.row0, ws.u_norm, ws.u_flag, ws.u_rho, fv.q_rho, xw_s8_slack(C), s8, x.out_index,
                                                                   x.arow, x.norm, x.eps);
          DTK_LAUNCHED();
          if (cm.n_gathered > 0) {
            const size_t r0 = (size_t)x.row0;
            gather_anchor_kernel<<<cm.gather_hi - cm.gather_lo, SAMPLE_THREADS, 0, sb>>>(
                tpc, T, C, P, g->h, g->w, pa, traj, ws.d_qlist, N, gp.f, gp.r, gp.map0, gp.item, cm.n_groups, n_unique, cm.gather_lo, fb, ws.u_hi, ws.u_lo, ws.u_flag,
                                                                    x.norm, ws.u_hi + r0 * C, ws.u_lo + r0 * C, ws.u_q8, ws.u_fac, fv.q_rho, xw_s8_slack(C),
                                                                    s8 ? ws.u_q8 + r0 * C : nullptr, ws.u_fac + r0, x.eps);
            DTK_LAUNCHED();
          }
        }
        if (ovl) DTK_CUDA(cudaEventRecord(xa->sample[k % XW_RING], sb));
        return DINOTRK_OK;
      };
      // Full-map queue.  The queued maps of chunk j (the host knows how many once the chunk's head has run) are appended to
      // ONE compact descriptor array (buffer set ws.cb[0]); the queue is worked off -- split-precision GEMM over all tokens on
      // 128-row tiles + the head kernels of head.cu -- when it is full and at the end of the phase.
      int q_rows = 0, q_groups = 0;
      auto flush = [&]() -> int {
        if (q_rows == 0) return DINOTRK_OK;
        const ChunkBufs& b = ws.cb[0];
        CorrAssist as;
        as.tkeys = b.tkeys; as.zero_word = b.hscratch; as.split_ready = true; as.no_thin = true; as.all_wide = true; as.small_tiles = true;
        int rc2 = launch_corr_maps(fv, nullptr, ch, b.norm, ws.d_cgrp, ws.d_cgrp + ws.sg_cap, ws.d_cgrp + 2 * ws.sg_cap, ws.d_cgrp + 3 * ws.sg_cap, q_groups,
                                   q_rows, q_rows, b.maps, ms, ws.d_splan, b.split, st, as);
        if (rc2) return rc2;
        rc2 = launch_head(b.maps, q_rows, ms, *g, *hw, ws.out_index_ring[0], anchors, 2, 0, nullptr, b.hscratch, st, b.tkeys, true);
        q_rows = q_groups = 0;
        return rc2;
      };
      auto finish = [&](size_t j) -> int {
        DTK_CUDA(cudaEventSynchronize(xa->done[j % XW_RING]));
        const int n_slow = xa->host_cnt[2 * (j % XW_RING)];
        g_infer_stats[4] += xa->host_cnt[2 * (j % XW_RING) + 1];
        const ChunkMeta& cm = metas[j];
        const XwSet& x = ws.xr[j % XW_RING];
        const Grp gp = grp_of(j);
        DTK_CHECK_ARG(n_slow >= 0 && n_slow <= cm.used, "infer: corrupt full-map queue (%d of %d)", n_slow, cm.used);
        g_infer_stats[1] += cm.used - n_slow; g_infer_stats[2] += n_slow;
        if (n_slow > 0) {
          if (q_rows + n_slow > ch || q_groups + cm.n_groups > ws.sg_cap) {
            int rc2 = flush();
            if (rc2) return rc2;
          }
          const ChunkBufs& b = ws.cb[0];
          const DescSplit c(b.split, ch, C);   // layout of a descriptor array of `ch` rows
          int rc2 = launch_xw_compact(nullptr, ws.u_hi, ws.u_lo, x.arow, x.norm, x.out_index, C, gp.f, gp.map0, cm.n_groups,
                                      n_slow, x.xc, nullptr, c.hi, c.lo, b.norm, ws.out_index_ring[0], ws.d_cgrp, ws.sg_cap, st, q_rows, q_groups,
                                      corr_hilo(fv));
          if (rc2) return rc2;
          q_rows += n_slow; q_groups += cm.n_groups;
        }
        DTK_CUDA(cudaEventRecord(xa->freed[j % XW_RING], st));
        return DINOTRK_OK;
      };
      if (!metas.empty() && (rc = enqueue_sample_x(0))) return rc;
      size_t n_finished = 0, k_end = metas.size();
      for (size_t k = 0; k < metas.size(); ++k) {
        const ChunkMeta& cm = metas[k];
        const XwSet& x = ws.xr[k % XW_RING];
        const Grp gp = grp_of(k);
        const XwCells cells = cells_of(k);
        if (ovl) DTK_CUDA(cudaStreamWaitEvent(st, xa->sample[k % XW_RING], 0));
        const float* eps = s8 ? x.eps : nullptr;   // (nullptr: the fp16 pass's XW_EPS)
        g_infer_stats[8] += cm.used - cm.n_gathered; g_infer_stats[9] += cm.n_gathered;
        if ((rc = launch_xw_coarse(fv, ws.u_hi, (int)ws.xw_rows, ws.u_norm, gp.f, gp.r, gp.m, gp.map0, ws.d_tiles + k * (gcap + 1),
                                   cm.n_groups, cm.used / TC2_BM_ROWS + cm.n_groups, x.xc, st, ws.d_rnorms, s8 ? ws.u_q8 : nullptr,
                                   ws.u_fac))) return rc;
        if ((rc = launch_xw_plan(cells, x.norm, cm.n_groups, *g, x.xc, st, cm.used, split_min_norm(C), eps))) return rc;
        if ((rc = launch_xw_gemm(fv, *g, ws.u_hi, ws.u_lo, (int)ws.xw_rows, cells, x.xc, st))) return rc;
        if ((rc = launch_xw_head(fv, *g, *hw, cells, x.norm, gp.map0, cm.used, x.out_index, anchors, 2, 0, x.xc, st, cm.n_groups,
                                 eps)))
          return rc;
        DTK_CUDA(cudaMemcpyAsync(xa->host_cnt + 2 * (k % XW_RING), x.xc.slow_cnt + cm.n_groups, 2 * sizeof(int), cudaMemcpyDeviceToHost, st));
        DTK_CUDA(cudaEventRecord(xa->done[k % XW_RING], st));
        if (k == 0 && probing && metas.size() > 1) {   // the probe: wait for it, look at the certificate's verdicts
          if ((rc = finish(0))) return rc;
          n_finished = 1;
          if (g_infer_stats[4] * 4 > (long long)cm.used) { k_end = 1; break; }
          if (s8 && g_xw_coarse < 0 && g_infer_stats[2] * XW_S8_PROBE_QUEUE_DIV > (long long)cm.used) {
            s8 = false;                   // the rest of the phase on the fp16 coarse pass
            g_infer_stats[6] = 0;
          }
        }
        if (k + 1 < metas.size() && (rc = enqueue_sample_x(k + 1))) return rc;
        while (n_finished + 2 <= k)
          if ((rc = finish(n_finished++))) return rc;
      }
      while (n_finished < k_end)
        if ((rc = finish(n_finished++))) return rc;
      if ((rc = flush())) return rc;
      if (ovl) {
        DTK_CUDA(cudaEventRecord(ia->join, sb));
        DTK_CUDA(cudaStreamWaitEvent(st, ia->join, 0));
      }
      if (k_end == metas.size()) {
        if (stop_after < 3) return DINOTRK_OK;
        NvtxRange nvd("dinotrk.infer.D.occlusion");
        return dinotrk_occlusion(traj, cos_sims, anchors, N, T, anchor_th, cos_th, occ, stream);
      }
      // switched: chunks k0.. on the full-map pipeline below.  The same chunks, their rows per chunk again.  (Everything
      // that read the plan is in the caller's stream by now, so the upload is ordered behind it.)
      k0 = k_end;
      g_infer_stats[3] = 0;
      g_infer_stats[6] = 0;
      plan_chunks(1, T, N, cnt.data(), ch, gcap, metas, plan_host, T, probing ? probe_cap : 0);
      if ((rc = upload_plan())) return rc;
    }
    if (!planned) {
      plan_chunks(1, T, N, cnt.data(), ch, gcap, metas, plan_host);
      int rc0 = upload_plan();
      if (rc0) return rc0;
    }
    int rc = DINOTRK_OK;
    InferAsync* ia = infer_async();
    const bool ovl = ia != nullptr && metas.size() > k0 + 1;
    cudaStream_t sa = (ovl && ia->mode >= 2) ? ia->aux : st;    // head stream
    cudaStream_t sb = ovl ? ia->aux2 : st;   // sampling stream
    if (ovl) {
      DTK_CUDA(cudaEventRecord(ia->fork, st));
      DTK_CUDA(cudaStreamWaitEvent(sa, ia->fork, 0));
      DTK_CUDA(cudaStreamWaitEvent(sb, ia->fork, 0));
    }
    auto enqueue_sample = [&](size_t k) -> int {   // descriptors of chunk k (buffer set k & 1)
      const ChunkMeta& cm = metas[k];
      const ChunkBufs& b = ws.cb[k & 1];
      const Grp gp = grp_of(k);
      if (ovl && k >= k0 + 2) DTK_CUDA(cudaStreamWaitEvent(sb, ia->gemm[k & 1], 0));   // GEMM k-2 read the descriptors of this set
      {
        ProfRange pr(PROF_SAMPLE, sb);
        // the split layout of launch_corr_gemm_tc for desc_rows = used
        const DescSplit c(b.split, cm.used, C);
        __half* c_hi = tensor ? reinterpret_cast<__half*>(c.hi) : nullptr;
        __half* c_lo = tensor ? reinterpret_cast<__half*>(c.lo) : nullptr;
        sample_anchor_kernel<<<cm.used, SAMPLE_THREADS, 0, sb>>>(tpc, T, C, P, g->h, g->w, pa, traj, ws.d_qlist, N, gp.f, gp.map0,
                                                                gp.item, cm.n_groups, fb, b.desc, b.norm, ws.out_index_ring[k & 3], c_hi, c_lo);
        DTK_LAUNCHED();
      }
      if (ovl) DTK_CUDA(cudaEventRecord(ia->sample[k & 1], sb));
      return DINOTRK_OK;
    };
    // the full-map head of chunk j (usually an empty list) runs on the GEMM stream between two GEMMs: it needs ~70 KB of
    // shared memory per CTA and could not co-reside with a GEMM anyway
    auto head_full = [&](size_t j) -> int {
      const ChunkBufs& b = ws.cb[j & 1];
      if (ovl) DTK_CUDA(cudaStreamWaitEvent(st, ia->head[j & 1], 0));   // fast head of chunk j (its list is complete)
      return launch_head(b.maps, metas[j].used, ms, *g, *hw, ws.out_index_ring[j & 3], anchors, 2, 0, nullptr, b.hscratch, st,
                         tensor ? b.tkeys : nullptr, true, 0, 2);
    };
    if (k0 < metas.size() && (rc = enqueue_sample(k0))) return rc;
    for (size_t k = k0; k < metas.size(); ++k) {
      const ChunkMeta& cm = metas[k];
      const ChunkBufs& b = ws.cb[k & 1];
      const Grp gp = grp_of(k);
      if (ovl) DTK_CUDA(cudaStreamWaitEvent(st, ia->sample[k & 1], 0));
      if (k >= k0 + 2 && (rc = head_full(k - 2))) return rc;   // last reader of maps / keys / list of this buffer set
      CorrAssist as;
      as.tkeys = tensor ? b.tkeys : nullptr; as.zero_word = b.hscratch; as.split_ready = tensor; as.no_thin = cm.no_thin;
      rc = launch_corr_maps(fv_split, b.desc, cm.used, b.norm, gp.f, gp.r, gp.m, gp.map0, cm.n_groups, cm.used, cm.maxm, b.maps, ms,
                            b.plan, b.split, st, as);
      if (rc) return rc;
      if (ovl) DTK_CUDA(cudaEventRecord(ia->gemm[k & 1], st));
      if (k + 1 < metas.size() && (rc = enqueue_sample(k + 1))) return rc;
      if (ovl) DTK_CUDA(cudaStreamWaitEvent(sa, ia->gemm[k & 1], 0));
      rc = launch_head(b.maps, cm.used, ms, *g, *hw, ws.out_index_ring[k & 3], anchors, 2, 0, nullptr, b.hscratch, sa, as.tkeys, true,
                       (ovl && ia->mode >= 2) ? ia->head_ctas_per_sm : 0, 1);
      if (rc) return rc;
      if (ovl) DTK_CUDA(cudaEventRecord(ia->head[k & 1], sa));
    }
    for (size_t j = std::max(k0, metas.size() >= 2 ? metas.size() - 2 : 0); j < metas.size(); ++j)
      if ((rc = head_full(j))) return rc;
    if (ovl) {
      DTK_CUDA(cudaEventRecord(ia->join, sa));
      DTK_CUDA(cudaStreamWaitEvent(st, ia->join, 0));
    }
  }
  if (stop_after < 3) return DINOTRK_OK;

  // ---- phase D: occlusion --------------------------------------------------------------------------
  NvtxRange nvd("dinotrk.infer.D.occlusion");
  return dinotrk_occlusion(traj, cos_sims, anchors, N, T, anchor_th, cos_th, occ, stream);
}

}  // extern "C"

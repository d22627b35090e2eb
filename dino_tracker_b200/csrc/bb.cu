// DINO best-buddies: mutual nearest neighbours between the token sets of two frames
// (preprocessing_dino_bb/extract_dino_best_buddies.py:12-54).
//
// The reference materialises the 8107 x 8107 cosine-affinity matrix per ordered pair (263 MB), divides it,
// and runs two arg-max passes over it.  Here, per ordered pair (s, t):
//   1. wgmma split-fp16 (hi/lo, 3-pass) GEMM  Fs x Ft^T  with a fused epilogue that keeps, per source token and 256-token
//      column tile, the best and second-best cosine (value + index) -- the matrix never leaves the SM;
//   2. a warp per source token merges the 32 tile partials, and re-evaluates its (one or two) candidates in
//      exact fp32 so that the arg-max and the reported cosine do not depend on tensor-core rounding;
//   3. mutual check  nn_ts[nn_st[n]] == n  on the index vectors.
#include "common.cuh"
#include "corr.cuh"
#include "tcgemm.cuh"

namespace dtk {

// order-preserving float -> uint (cosines can be negative)
__device__ __forceinline__ unsigned f2ord(float v) {
  unsigned b = __float_as_uint(v);
  return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ float ord2f(unsigned u) {
  return __uint_as_float((u & 0x80000000u) ? (u & 0x7fffffffu) : ~u);
}

struct BBPartial {   // per (pair, column tile, source token)
  unsigned long long key1;  // f2ord(best) << 32 | (0x7fffffff - index): max key = best value, ties -> first index
  float v2; int i2;         // runner-up
};

struct BBEpi {
  const float* norms;      // [T][P]
  const int* grp_src;      // [n_pairs] source frame (A rows = tokens of that frame)
  const int* grp_tgt;      // [n_pairs] target frame (B batch)
  BBPartial* part;         // [n_pairs][n_tiles][P]
  int P, n_tiles;
  struct State { unsigned long long k1; float v2; int i2; };
  __device__ __forceinline__ void tile_begin(State& s) const { s.k1 = 0ull; s.v2 = -INFINITY; s.i2 = -1; }
  __device__ __forceinline__ void operator()(State& s, int g, int r, int col0, const float (&f)[32], int ncols) const {
    const float ns = norms[(size_t)grp_src[g] * P + r];
    const float* nt = norms + (size_t)grp_tgt[g] * P + col0;
#pragma unroll
    for (int i = 0; i < 32; ++i) {
      if (i < ncols) {
        float v = corr_cos(f[i], ns, __ldg(nt + i));
        unsigned long long k = ((unsigned long long)f2ord(v) << 32) | (unsigned)(0x7fffffff - (col0 + i));
        if (k > s.k1) {
          if (s.k1 != 0ull) { s.v2 = ord2f((unsigned)(s.k1 >> 32)); s.i2 = 0x7fffffff - (int)(s.k1 & 0xffffffffu); }
          s.k1 = k;
        } else if (v > s.v2) {
          s.v2 = v; s.i2 = col0 + i;
        }
      }
    }
  }
  __device__ __forceinline__ void tile_end(State& s, int g, int r, int n_tile) const {
    BBPartial p{s.k1, s.v2, s.i2};
    part[((size_t)g * n_tiles + n_tile) * P + r] = p;
  }
};

// warp per (pair, source token): merge tile partials -> top-2, exact fp32 re-evaluation, final nn + cosine
__global__ void bb_resolve_kernel(const float* __restrict__ tpc, const float* __restrict__ norms, int C, int P,
                                  const int* __restrict__ grp_src, const int* __restrict__ grp_tgt,
                                  const BBPartial* __restrict__ part, int n_tiles, int n_pairs, float ambiguity,
                                  int* __restrict__ nn_idx, float* __restrict__ nn_cos) {
  const int lane = threadIdx.x & 31;
  const size_t wid = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (wid >= (size_t)n_pairs * P) return;
  const int g = (int)(wid / P), r = (int)(wid - (size_t)g * P);
  // top-2 as (value, first index) keys: every lane ends with the same two candidates even when values tie (the exact
  // re-evaluation below sums the lanes' partial dot products, so all lanes must evaluate the same token)
  unsigned long long k1 = 0ull, k2 = 0ull;
  auto push = [&](unsigned long long k) {
    if (k > k1) { k2 = k1; k1 = k; } else if (k > k2) { k2 = k; }
  };
  for (int t = lane; t < n_tiles; t += 32) {
    BBPartial p = part[((size_t)g * n_tiles + t) * P + r];
    push(p.key1);
    if (p.i2 >= 0) push(((unsigned long long)f2ord(p.v2) << 32) | (unsigned)(0x7fffffff - p.i2));
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {   // the two lanes of a step hold disjoint token sets: no key arrives twice
    const unsigned long long ok1 = __shfl_xor_sync(0xffffffffu, k1, o), ok2 = __shfl_xor_sync(0xffffffffu, k2, o);
    push(ok1);
    push(ok2);
  }
  int i1 = 0x7fffffff - (int)(k1 & 0xffffffffu);
  const float v1 = ord2f((unsigned)(k1 >> 32));
  const int i2 = k2 ? 0x7fffffff - (int)(k2 & 0xffffffffu) : -1;
  const float v2 = k2 ? ord2f((unsigned)(k2 >> 32)) : -INFINITY;
  const int fs = grp_src[g], ft = grp_tgt[g];
  const float4* a = reinterpret_cast<const float4*>(tpc + ((size_t)fs * P + r) * C);
  auto exact = [&](int col) {
    const float4* b = reinterpret_cast<const float4*>(tpc + ((size_t)ft * P + col) * C);
    float acc = 0.f;
    for (int i = lane; i < C / 4; i += 32) {
      float4 x = __ldg(a + i), y = __ldg(b + i);
      acc = fmaf(x.x, y.x, acc); acc = fmaf(x.y, y.y, acc); acc = fmaf(x.z, y.z, acc); acc = fmaf(x.w, y.w, acc);
    }
    acc = warp_sum(acc);
    return corr_cos(acc, norms[(size_t)fs * P + r], norms[(size_t)ft * P + col]);
  };
  float e1 = exact(i1);
  if (i2 >= 0 && v1 - v2 < ambiguity) {   // near-tie under tensor-core rounding: decide in exact fp32
    float e2 = exact(i2);
    if (e2 > e1 || (e2 == e1 && i2 < i1)) { e1 = e2; i1 = i2; }
  }
  if (lane == 0) { nn_idx[(size_t)g * P + r] = i1; nn_cos[(size_t)g * P + r] = e1; }
}

// mutual[n] = (nn_ts[nn_st[n]] == n)
__global__ void bb_mutual_kernel(const int* __restrict__ nn_st, const int* __restrict__ nn_ts, int P, size_t total,
                                 uint8_t* __restrict__ mutual) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= total) return;
  size_t g = i / P;
  int n = (int)(i - g * P);
  mutual[i] = nn_ts[g * P + nn_st[i]] == n ? 1 : 0;
}

// ---- best-buddy peak filter (preprocessing_dino_bb/compute_dino_bb_nms.py:12-66) ---------------------------------------
// Per similarity map of one source point against a target frame, the reference keeps the 400 largest values, puts a
// (2 box_size)^2 box on each, runs greedy NMS (torchvision.ops.batched_nms: descending score, a box is dropped when its
// IoU with an already KEPT box exceeds the threshold) and reports the two largest kept values and their ratio r.  Greedy
// NMS keeps the maximum first; the second kept box is therefore the highest-scoring candidate whose IoU with the
// maximum's box is <= threshold -- provided it is among the 400 largest values.  So per map: arg-max, the best value
// outside the maximum's suppression zone, and a rank test (fewer than `topk` values strictly above it).  Nothing is
// sorted.  Box arithmetic in fp32 as torchvision does it: inter / (area_a + area_b - inter) > thresh.
constexpr int NMS_THREADS = 256;
__global__ void __launch_bounds__(NMS_THREADS)
bb_nms_kernel(const float* __restrict__ maps, int n_maps, int map_stride, int P, int w, int stride_px, int half_patch,
              float box, float iou_thresh, int topk, float* __restrict__ peak_affs, float* __restrict__ r_out) {
  __shared__ unsigned long long s_key[NMS_THREADS / 32];
  __shared__ float s_f[NMS_THREADS / 32];
  __shared__ int s_i[NMS_THREADS / 32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  for (int map = blockIdx.x; map < n_maps; map += gridDim.x) {
    const float* m = maps + (size_t)map * map_stride;
    // first arg-max (values are >= 0 after the ReLU of the correlation epilogue; a negative similarity can never be one of
    // the reported peaks: the reference multiplies by the keep mask and takes a top-2 over values that include zeros)
    unsigned long long key = 0ull;
    for (int i = tid; i < P; i += NMS_THREADS) {
      const unsigned long long k = ((unsigned long long)__float_as_uint(m[i] + 0.f) << 32) | (unsigned)(0x7fffffff - i);
      key = k > key ? k : key;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, key, o); key = t > key ? t : key; }
    if (lane == 0) s_key[warp] = key;
    __syncthreads();
    unsigned long long kb = s_key[0];
#pragma unroll
    for (int k = 1; k < NMS_THREADS / 32; ++k) kb = s_key[k] > kb ? s_key[k] : kb;
    const int amax = 0x7fffffff - (int)(kb & 0xffffffffu);
    const float vmax = __uint_as_float((unsigned)(kb >> 32));
    const float ax = (float)(half_patch + (amax % w) * stride_px), ay = (float)(half_patch + (amax / w) * stride_px);
    const float ax1 = ax - box, ax2 = ax + box, ay1 = ay - box, ay2 = ay + box;
    const float area = (ax2 - ax1) * (ay2 - ay1);
    // best value whose box survives next to the maximum's box
    float v2 = 0.f;
    for (int i = tid; i < P; i += NMS_THREADS) {
      if (i == amax) continue;
      const float x = (float)(half_patch + (i % w) * stride_px), y = (float)(half_patch + (i / w) * stride_px);
      const float iw = fmaxf(fminf(ax2, x + box) - fmaxf(ax1, x - box), 0.f);
      const float ih = fmaxf(fminf(ay2, y + box) - fmaxf(ay1, y - box), 0.f);
      const float inter = iw * ih;
      const float iou = inter / (area + area - inter);
      if (!(iou > iou_thresh)) v2 = fmaxf(v2, m[i]);
    }
    v2 = warp_max(v2);
    if (lane == 0) s_f[warp] = v2;
    __syncthreads();
    v2 = s_f[0];
#pragma unroll
    for (int k = 1; k < NMS_THREADS / 32; ++k) v2 = fmaxf(v2, s_f[k]);
    // is it among the `topk` largest values of the map?
    int above = 0;
    for (int i = tid; i < P; i += NMS_THREADS) above += m[i] > v2 ? 1 : 0;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) above += __shfl_xor_sync(0xffffffffu, above, o);
    if (lane == 0) s_i[warp] = above;
    __syncthreads();
    if (tid == 0) {
      int tot = 0;
      for (int k = 0; k < NMS_THREADS / 32; ++k) tot += s_i[k];
      const float second = tot < topk ? v2 : 0.f;
      peak_affs[2 * (size_t)map] = vmax;
      peak_affs[2 * (size_t)map + 1] = second;
      r_out[map] = __fdiv_rn(second, vmax);
    }
    __syncthreads();
  }
}

__global__ void bb_plan_kernel(int n_pairs, int P, const int* __restrict__ src, int* row0, int* m, int* tile_start) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  const int tiles = (P + TC_BM - 1) / TC_BM;
  if (i < n_pairs) { row0[i] = src[i] * P; m[i] = P; tile_start[i] = i * tiles; }
  if (i == 0) tile_start[n_pairs] = n_pairs * tiles;
}

struct BBWs {
  BBPartial* part; int* row0; int* m; int* tile_start;
  BBWs(Arena& ar, int n_pairs, int P) {
    part = ar.take<BBPartial>((size_t)n_pairs * cdiv(P, TC_BN) * P);
    row0 = ar.take<int>(n_pairs + 1);
    m = ar.take<int>(n_pairs + 1);
    tile_start = ar.take<int>(n_pairs + 1);
  }
};

}  // namespace dtk

using namespace dtk;

extern "C" {

size_t dinotrk_best_buddies_workspace_bytes(int n_pairs, int P) {
  return align_up(layout_end<BBWs>(n_pairs, P), 256) + 1024;
}

int dinotrk_best_buddies_pairs(const dinotrk_features* feat, const dinotrk_geom* g, const int* pair_src,
                               const int* pair_tgt, int n_pairs, int* nn_idx, float* nn_cos, void* workspace,
                               size_t workspace_bytes, void* stream) {
  DTK_CHECK_ARG(feat && feat->tpc && feat->norms && feat->hi && feat->lo && g && pair_src && pair_tgt && nn_idx && nn_cos,
                "best_buddies: null pointer (the TF32 split of the features is required)");
  const int P = g->h * g->w, C = feat->C, T = feat->T;
  DTK_CHECK_ARG(C % 8 == 0 && n_pairs >= 0, "best_buddies: C must be a multiple of 8");
  DTK_CHECK_ARG(workspace && workspace_bytes >= dinotrk_best_buddies_workspace_bytes(n_pairs, P), "best_buddies: workspace too small");
  if (n_pairs == 0) return DINOTRK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  const int n_tiles = cdiv(P, TC_BN);
  Arena ar(workspace);
  const BBWs ws(ar, n_pairs, P);
  {
    ProfRange pr(PROF_MISC, st);
    bb_plan_kernel<<<cdiv(n_pairs, 128), 128, 0, st>>>(n_pairs, P, pair_src, ws.row0, ws.m, ws.tile_start);
    DTK_LAUNCHED();
  }
  // A: the source frames' tokens, B: the target frames (one batch item per frame)
  const TcOperands op{feat->hi, feat->lo, (uint64_t)T * P, 0, feat->hi, feat->lo, (uint64_t)T, 0};
  const TcProblem pb{pair_tgt, ws.row0, ws.m, ws.tile_start, n_pairs, P, C};
  BBEpi epi{feat->norms, pair_src, pair_tgt, ws.part, P, n_tiles};
  if (int rc = tc_launch<TcMode::F16X3, BBEpi>(op, pb, n_pairs * cdiv(P, TC_BM), epi, st, PROF_BB)) return rc;
  {
    ProfRange pr(PROF_BB, st);
    size_t warps = (size_t)n_pairs * P;
    bb_resolve_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, st>>>(feat->tpc, feat->norms, C, P, pair_src, pair_tgt, ws.part,
                                                                  n_tiles, n_pairs, 2e-4f, nn_idx, nn_cos);
    DTK_LAUNCHED();
  }
  return DINOTRK_OK;
}

int dinotrk_bb_nms(const float* maps, int n_maps, const dinotrk_geom* g, float box_size, float iou_thresh, int topk,
                   float* peak_affs, float* r, void* stream) {
  DTK_CHECK_ARG(maps && g && peak_affs && r && n_maps >= 0 && topk > 0 && box_size > 0.f, "bb_nms: bad arguments");
  if (n_maps == 0) return DINOTRK_OK;
  const int P = g->h * g->w;
  DTK_CHECK_ARG(topk <= P, "bb_nms: topk %d exceeds the %d tokens of a map (torch.topk would fail too)", topk, P);
  int grid = n_maps < num_sms() * 8 ? n_maps : num_sms() * 8;
  ProfRange pr(PROF_BB, (cudaStream_t)stream);
  bb_nms_kernel<<<grid, NMS_THREADS, 0, (cudaStream_t)stream>>>(maps, n_maps, dinotrk_map_stride(g), P, g->w, g->stride, g->patch / 2,
                                                                box_size, iou_thresh, topk, peak_affs, r);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_bb_mutual(const int* nn_st, const int* nn_ts, int n_pairs, int P, uint8_t* mutual, void* stream) {
  DTK_CHECK_ARG(nn_st && nn_ts && mutual && n_pairs >= 0 && P > 0, "bb_mutual: bad args");
  size_t total = (size_t)n_pairs * P;
  if (total == 0) return DINOTRK_OK;
  ProfRange pr(PROF_BB, (cudaStream_t)stream);
  bb_mutual_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(nn_st, nn_ts, P, total, mutual);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // extern "C"

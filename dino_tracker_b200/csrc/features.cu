// Feature cache layout conversion, token norms and descriptor sampling.
//   reference: models/tracker.py:64-71 (cache), :77-111 (sampling), utils.py:75-101.
#include <stdarg.h>

#include <vector>

#include "common.cuh"
#include "sample.cuh"

namespace dtk {

static thread_local char g_err[512] = "";
unsigned long long g_launches = 0;

void set_error(const char* fmt, ...) {
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(g_err, sizeof(g_err), fmt, ap);
  va_end(ap);
}

bool g_prof_on = false;
struct ProfRec { cudaEvent_t a, b; int cls; };
static std::vector<ProfRec> g_prof_recs;
static std::vector<cudaEvent_t> g_prof_pool;
static cudaEvent_t prof_event() {
  if (!g_prof_pool.empty()) { cudaEvent_t e = g_prof_pool.back(); g_prof_pool.pop_back(); return e; }
  cudaEvent_t e; cudaEventCreate(&e); return e;
}
void prof_begin(int cls, cudaStream_t st) {
  ProfRec r{prof_event(), prof_event(), cls};
  cudaEventRecord(r.a, st);
  g_prof_recs.push_back(r);
}
void prof_end(cudaStream_t st) { cudaEventRecord(g_prof_recs.back().b, st); }

// ---- exclusive scan of block counts: one block per row of nb counts ---------------------------------------------
constexpr int SCAN_THREADS = 1024;
__global__ void __launch_bounds__(SCAN_THREADS)
scan_counts_kernel(const int* __restrict__ cnt, int n, int* __restrict__ off, int* __restrict__ total) {
  __shared__ int s_sum[SCAN_THREADS];
  cnt += (size_t)blockIdx.x * n;
  off += (size_t)blockIdx.x * n;
  const int per = (n + SCAN_THREADS - 1) / SCAN_THREADS, b = threadIdx.x * per, e = min(b + per, n);
  int sum = 0;
  for (int i = b; i < e; ++i) sum += cnt[i];
  s_sum[threadIdx.x] = sum;
  __syncthreads();
  for (int o = 1; o < SCAN_THREADS; o <<= 1) {   // Hillis-Steele inclusive scan
    const int v = threadIdx.x >= o ? s_sum[threadIdx.x - o] : 0;
    __syncthreads();
    s_sum[threadIdx.x] += v;
    __syncthreads();
  }
  int run = s_sum[threadIdx.x] - sum;
  for (int i = b; i < e; ++i) { off[i] = run; run += cnt[i]; }
  if (threadIdx.x == SCAN_THREADS - 1) total[blockIdx.x] = s_sum[SCAN_THREADS - 1];
}

int launch_count_scan(const int* cnt, int nb, int rows, int* off, int* total, cudaStream_t stream) {
  scan_counts_kernel<<<rows, SCAN_THREADS, 0, stream>>>(cnt, nb, off, total);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// ---- [T][C][P] <-> [T][P][C] tiled transposes -------------------------------------------------
__global__ void transpose_kernel(const float* __restrict__ in, float* __restrict__ out, int R, int S) {
  // per batch item (blockIdx.z): in [R][S] -> out [S][R]
  __shared__ float tile[32][33];
  const float* src = in + (size_t)blockIdx.z * R * S;
  float* dst = out + (size_t)blockIdx.z * R * S;
  int s0 = blockIdx.x * 32, r0 = blockIdx.y * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int r = r0 + j, s = s0 + threadIdx.x;
    tile[j][threadIdx.x] = (r < R && s < S) ? src[(size_t)r * S + s] : 0.f;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    int s = s0 + j, r = r0 + threadIdx.x;
    if (r < R && s < S) dst[(size_t)s * R + r] = tile[threadIdx.x][j];
  }
}

// one warp per token: |f|_2 over C contiguous floats
__global__ void token_norm_kernel(const float* __restrict__ tpc, float* __restrict__ norms, size_t n_tok, int C) {
  size_t tok = (size_t)blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
  if (tok >= n_tok) return;
  const float4* row = reinterpret_cast<const float4*>(tpc + tok * C);
  float acc = 0.f;
  for (int i = threadIdx.x & 31; i < C / 4; i += 32) {
    float4 v = __ldg(row + i);
    acc = fmaf(v.x, v.x, acc); acc = fmaf(v.y, v.y, acc);
    acc = fmaf(v.z, v.z, acc); acc = fmaf(v.w, v.w, acc);
  }
  acc = warp_sum(acc);
  if ((threadIdx.x & 31) == 0) norms[tok] = sqrtf(acc);
}

// generic sampler: explicit frames_set
__global__ void sample_kernel(const float* __restrict__ tpc, int C, int P, int h, int w, PointAffine pa,
                              const float* __restrict__ points, const int* __restrict__ frames_set, int N,
                              int normalized, float* __restrict__ desc, float* __restrict__ desc_norm) {
  int b = blockIdx.x;
  float x = points[b * 3 + 0], y = points[b * 3 + 1], idx = points[b * 3 + 2];
  if (!normalized) {
    x = __fadd_rn(__fmul_rn(pa.aw, x), pa.bw);
    y = __fadd_rn(__fmul_rn(pa.ah, y), pa.bh);
  }
  TriCorners c = tri_setup(x, y, idx, N, h, w);
  int f0 = frames_set[c.z0];
  int f1 = c.z1 >= 0 ? frames_set[c.z1] : -1;
  sample_point(tpc, C, P, c, f0, f1, desc + (size_t)b * C, desc_norm ? desc_norm + b : nullptr);
}

}  // namespace dtk

using namespace dtk;

extern "C" {

int dinotrk_version(void) { return DINOTRK_VERSION; }
const char* dinotrk_last_error(void) { return dtk::g_err; }
unsigned long long dinotrk_launch_count(void) { return dtk::g_launches; }

static const char* kProfNames[PROF_COUNT] = {"sample", "corr_gemm", "corr_stream", "head", "traj_cos", "anchor_lists",
                                              "occlusion", "pack", "delta_conv", "delta_blur", "delta_align", "misc",
                                              "best_buddies", "vit_gemm", "vit_attn", "vit_misc", "head_full",
                                              "xw_coarse_gemm", "xw_plan", "xw_exact_gemm", "xw_head", "train_backward",
                                              "delta_train_conv", "delta_bn", "delta_dgrad", "delta_wgrad",
                                              "fg_mask", "contrastive", "sampler", "cycle", "emb_reg"};
int dinotrk_profile_classes(void) { return PROF_COUNT; }
const char* dinotrk_profile_class_name(int cls) { return (cls >= 0 && cls < PROF_COUNT) ? kProfNames[cls] : ""; }
void dinotrk_profile_enable(int on) { dtk::g_prof_on = on != 0; }
int dinotrk_profile_collect(double* ms, unsigned long long* launches, int n) {
  DTK_CHECK_ARG(ms && launches && n >= PROF_COUNT, "profile_collect: need %d slots", (int)PROF_COUNT);
  for (int i = 0; i < n; ++i) { ms[i] = 0; launches[i] = 0; }
  for (auto& r : g_prof_recs) {
    DTK_CUDA(cudaEventSynchronize(r.b));
    float t = 0.f;
    DTK_CUDA(cudaEventElapsedTime(&t, r.a, r.b));
    ms[r.cls] += t; launches[r.cls] += 1;
    g_prof_pool.push_back(r.a); g_prof_pool.push_back(r.b);
  }
  g_prof_recs.clear();
  return DINOTRK_OK;
}

int dinotrk_make_geom(int H, int W, int patch, int stride, int radius, dinotrk_geom* g) {
  DTK_CHECK_ARG(g != nullptr, "geom: null output");
  DTK_CHECK_ARG(patch > 0 && stride > 0 && H >= patch && W >= patch && radius >= 0,
                "geom: bad sizes H=%d W=%d patch=%d stride=%d", H, W, patch, stride);
  g->H = H; g->W = W; g->patch = patch; g->stride = stride; g->radius = radius;
  g->h = 1 + (H - patch) / stride;
  g->w = 1 + (W - patch) / stride;
  return DINOTRK_OK;
}

int dinotrk_token_norms(const float* tpc, float* norms, int T, int C, int P, void* stream) {
  DTK_CHECK_ARG(tpc && norms && T > 0 && P > 0 && C > 0 && C % 4 == 0, "token_norms: bad args (C must be a multiple of 4)");
  size_t n = (size_t)T * P;
  ProfRange pr(PROF_PACK, (cudaStream_t)stream);
  token_norm_kernel<<<(unsigned)((n + 7) / 8), 256, 0, (cudaStream_t)stream>>>(tpc, norms, n, C);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_pack_features(const float* chw, float* tpc, float* norms, int T, int C, int P, void* stream) {
  DTK_CHECK_ARG(chw && tpc && T > 0 && P > 0 && C > 0 && C % 4 == 0, "pack_features: bad args (C must be a multiple of 4)");
  dim3 grid(cdiv(P, 32), cdiv(C, 32), T), block(32, 8);
  {
    ProfRange pr(PROF_PACK, (cudaStream_t)stream);
    transpose_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(chw, tpc, C, P);
    DTK_LAUNCHED();
  }
  if (norms) return dinotrk_token_norms(tpc, norms, T, C, P, stream);
  return DINOTRK_OK;
}

int dinotrk_unpack_features(const float* tpc, float* chw, int T, int C, int P, void* stream) {
  DTK_CHECK_ARG(chw && tpc && T > 0 && P > 0 && C > 0, "unpack_features: bad args");
  dim3 grid(cdiv(C, 32), cdiv(P, 32), T), block(32, 8);
  transpose_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(tpc, chw, P, C);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int dinotrk_sample_descriptors(const float* tpc, int T, int C, const dinotrk_geom* g, const float* points,
                               int B, const int* frames_set, int N, int points_normalized, float* desc,
                               float* desc_norm, void* stream) {
  DTK_CHECK_ARG(tpc && g && points && frames_set && desc, "sample_descriptors: null pointer");
  DTK_CHECK_ARG(T > 0 && C > 0 && C % 4 == 0 && N > 0 && B >= 0, "sample_descriptors: bad sizes");
  if (B == 0) return DINOTRK_OK;
  ProfRange pr(PROF_SAMPLE, (cudaStream_t)stream);
  sample_kernel<<<B, SAMPLE_THREADS, 0, (cudaStream_t)stream>>>(tpc, C, g->h * g->w, g->h, g->w,
                                                              make_point_affine(*g), points, frames_set, N,
                                                              points_normalized, desc, desc_norm);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // extern "C"

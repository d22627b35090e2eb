// Tensor-core correlation GEMM (wgmma, split-precision fp16 hi/lo) + operand splitting + TMA tensor-map helpers + the
// uniform group plan and max |x| kernels that tcgemm.cuh declares.
//
//   corr[j][p] = relu( <d_j, F[frame][p]> / max(|d_j| |F[frame][p]|, 1e-8) )     (models/tracker.py:158-173)
// (the ReLU is a template choice: the contrastive losses keep the signed cosines, contrastive.cu)
//
// The contraction runs as lo*hi + hi*lo + hi*hi on the f16 tensor pipe with fp32 accumulation in registers
// (operands pre-split into fp16 hi + fp16 lo, x = hi + lo up to 2^-22 |x|), which keeps the products
// faithful to ~2^-21; the cosine normalisation and ReLU are the epilogue on the accumulator.
#include <cuda_fp16.h>

#include "common.cuh"
#include "corr.cuh"
#include "tcgemm.cuh"
#include "xwin.cuh"

namespace dtk {

int num_sms() {
  static PerDev<int> sms_dev;
  int& sms = sms_dev.get();
  if (sms == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || sms <= 0) sms = 1;
  }
  return sms;
}

// ---- driver entry point for cuTensorMapEncodeTiled (resolved once; no link-time libcuda dependency) ----
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
static EncodeTiledFn get_encode() {
  static EncodeTiledFn fn = nullptr;
  if (!fn) {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = (EncodeTiledFn)p;
  }
  return fn;
}

static CUtensorMapSwizzle swizzle_of(int bytes) {
  return bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B;
}

// (8-bit operands travel as UINT8: TMA copies bytes, the wgmma instruction gives them their signed type)
static CUtensorMapDataType tmap_type(int elem) {
  return elem == TMAP_F32 ? CU_TENSOR_MAP_DATA_TYPE_FLOAT32 : elem == TMAP_BF16 ? CU_TENSOR_MAP_DATA_TYPE_BFLOAT16
       : elem == TMAP_S8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
}
static int elem_bytes_of(int elem) { return elem == TMAP_F32 ? 4 : elem == TMAP_S8 ? 1 : 2; }

static int encode(CUtensorMap* map, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides,
                  const cuuint32_t* box, int elem, int swizzle = 128) {
  EncodeTiledFn fn = get_encode();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return DINOTRK_ECUDA; }
  cuuint32_t estr[3] = {1, 1, 1};
  CUtensorMapDataType dt = tmap_type(elem);
  CUresult r = fn(map, dt, rank, const_cast<void*>(base), dims, strides, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_of(swizzle), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled failed (%d)", (int)r); return DINOTRK_ECUDA; }
  return DINOTRK_OK;
}

int make_tmap_2d(CUtensorMap* map, const void* base, uint64_t rows, uint64_t cols, uint32_t box_rows, uint32_t box_cols,
                 int elem, uint64_t ld, int swizzle) {
  const int elem_bytes = elem_bytes_of(elem);
  if (ld == 0) ld = cols;
  cuuint64_t dims[2] = {cols, rows};
  cuuint64_t strides[1] = {ld * (uint64_t)elem_bytes};
  cuuint32_t box[2] = {box_cols, box_rows};
  return encode(map, base, 2, dims, strides, box, elem, swizzle);
}
int make_tmap_3d(CUtensorMap* map, const void* base, uint64_t batch, uint64_t rows, uint64_t cols, uint32_t box_rows,
                 uint32_t box_cols, int elem, uint64_t ld) {
  const int elem_bytes = elem_bytes_of(elem);
  if (ld == 0) ld = cols;
  cuuint64_t dims[3] = {cols, rows, batch};
  cuuint64_t strides[2] = {ld * (uint64_t)elem_bytes, rows * ld * (uint64_t)elem_bytes};
  cuuint32_t box[3] = {box_cols, box_rows, 1};
  return encode(map, base, 3, dims, strides, box, elem);
}

int make_tmap_4d(CUtensorMap* map, const void* base, const uint64_t dims[4], const uint64_t strides_bytes[3],
                 const uint32_t box[4], int elem, int swizzle) {
  EncodeTiledFn fn = get_encode();
  if (!fn) { set_error("cuTensorMapEncodeTiled entry point not available"); return DINOTRK_ECUDA; }
  cuuint64_t d[4] = {dims[0], dims[1], dims[2], dims[3]};
  cuuint64_t s[3] = {strides_bytes[0], strides_bytes[1], strides_bytes[2]};
  cuuint32_t b[4] = {box[0], box[1], box[2], box[3]};
  cuuint32_t estr[4] = {1, 1, 1, 1};
  CUtensorMapDataType dt = tmap_type(elem);
  CUresult r = fn(map, dt, 4, const_cast<void*>(base), d, s, b, estr, CU_TENSOR_MAP_INTERLEAVE_NONE,
                  swizzle_of(swizzle), CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) { set_error("cuTensorMapEncodeTiled (4-d) failed (%d)", (int)r); return DINOTRK_ECUDA; }
  return DINOTRK_OK;
}

// x = hi + lo (+ residual <= 2^-22 |x| in the fp16 normal range): hi = rn_fp16(x), lo = rn_fp16(x - hi)
__device__ __forceinline__ void split4(const float4& v, uint2& hi, uint2& lo) {
  __half h0 = __float2half_rn(v.x), h1 = __float2half_rn(v.y), h2 = __float2half_rn(v.z), h3 = __float2half_rn(v.w);
  __half l0 = __float2half_rn(v.x - __half2float(h0)), l1 = __float2half_rn(v.y - __half2float(h1));
  __half l2 = __float2half_rn(v.z - __half2float(h2)), l3 = __float2half_rn(v.w - __half2float(h3));
  __half2 a = __halves2half2(h0, h1), b2 = __halves2half2(h2, h3), c = __halves2half2(l0, l1), d = __halves2half2(l2, l3);
  hi = make_uint2(*reinterpret_cast<unsigned*>(&a), *reinterpret_cast<unsigned*>(&b2));
  lo = make_uint2(*reinterpret_cast<unsigned*>(&c), *reinterpret_cast<unsigned*>(&d));
}

__global__ void split_f16_kernel(const float4* __restrict__ x, uint2* __restrict__ hi, uint2* __restrict__ lo, size_t n4) {
  size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (; i < n4; i += stride) split4(__ldg(x + i), hi[i], lo[i]);
}

// the split interleaved per 32 channels (dinotrk_split_hilo): thread = 4 channels of a row; in a 32-channel block, hi of
// channels 4 q .. 4 q + 3 goes to the block's 8-byte word q and lo to word 8 + q
__global__ void split_hilo_kernel(const float* __restrict__ x, uint2* __restrict__ hilo, size_t rows, int C) {
  const int nb = (C + 31) / 32;
  const size_t n = rows * nb * 8;
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const size_t rb = i >> 3, row = rb / nb;
    const int q = (int)(i & 7), c = 32 * (int)(rb - row * nb) + 4 * q;
    const float4 v = c < C ? __ldg(reinterpret_cast<const float4*>(x + row * C + c)) : make_float4(0.f, 0.f, 0.f, 0.f);
    split4(v, hilo[16 * rb + q], hilo[16 * rb + 8 + q]);
  }
}

int launch_split_hilo(const float* x, void* hilo, size_t rows, int C, cudaStream_t st) {
  DTK_CHECK_ARG(C > 0 && C % 4 == 0, "split_hilo: C must be a positive multiple of 4");
  const size_t n = rows * ((C + 31) / 32) * 8;
  if (n == 0) return DINOTRK_OK;
  unsigned grid = (unsigned)((n + 255) / 256);
  if (grid > (unsigned)num_sms() * 16) grid = num_sms() * 16;
  ProfRange pr(PROF_MISC, st);
  split_hilo_kernel<<<grid, 256, 0, st>>>(x, reinterpret_cast<uint2*>(hilo), rows, C);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

int launch_split_f16(const float* x, void* hi, void* lo, size_t n, cudaStream_t st) {
  if (n == 0) return DINOTRK_OK;
  DTK_CHECK_ARG(n % 4 == 0, "split_fp16: length must be a multiple of 4");
  size_t n4 = n / 4;
  unsigned grid = (unsigned)((n4 + 255) / 256);
  if (grid > (unsigned)num_sms() * 16) grid = num_sms() * 16;
  ProfRange pr(PROF_MISC, st);
  split_f16_kernel<<<grid, 256, 0, st>>>(reinterpret_cast<const float4*>(x), reinterpret_cast<uint2*>(hi),
                                         reinterpret_cast<uint2*>(lo), n4);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// uniform group tables of the wgmma GEMM (tcgemm.cuh, launch_tc_plan)
__global__ void tc_plan_kernel(int* batch, int* row0, int* m, int* tile_start, int n_groups, int rows, int row_stride,
                               int row_base, int batch_base, int tile_rows) {
  if (threadIdx.x == 0 && blockIdx.x == 0) {
    int acc = 0;
    for (int g = 0; g < n_groups; ++g) {
      batch[g] = batch_base + g; row0[g] = row_base + g * row_stride; m[g] = rows; tile_start[g] = acc;
      acc += (rows + tile_rows - 1) / tile_rows;
    }
    tile_start[n_groups] = acc;
  }
}

int launch_tc_plan(const TcPlan& pl, int n_groups, int rows, int row_stride, int row_base, int batch_base, int tile_rows,
                   cudaStream_t st) {
  tc_plan_kernel<<<1, 32, 0, st>>>(pl.batch, pl.row0, pl.m, pl.tile_start, n_groups, rows, row_stride, row_base, batch_base,
                                   tile_rows);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// max |g| as the bits of a non-negative float (integer order = float order; the max does not depend on the order)
__global__ void amax_kernel(const float* __restrict__ g, size_t n, unsigned* __restrict__ amax) {
  unsigned m = 0;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (size_t)gridDim.x * blockDim.x)
    m = max(m, __float_as_uint(fabsf(g[i])));
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) m = max(m, __shfl_xor_sync(0xffffffffu, m, o));
  if ((threadIdx.x & 31) == 0) atomicMax(amax, m);
}

int launch_amax(const float* x, size_t n, unsigned* amax, unsigned grid, cudaStream_t st) {
  amax_kernel<<<grid, 256, 0, st>>>(x, n, amax);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

// int8 operands of the coarse pass (xw_quant_row): one warp per row; rho_max[row / rows_per_group] = largest rho of the
// group (float bits: non-negative floats order like their bits; zeroed by the caller)
__global__ void __launch_bounds__(256)
quant_s8_kernel(const float* __restrict__ x, const float* __restrict__ norms, size_t rows, int C, int rows_per_group,
                int8_t* __restrict__ q, float* __restrict__ fac, float* __restrict__ rho, unsigned* __restrict__ rho_max) {
  const size_t nw = (size_t)gridDim.x * 8;
  for (size_t r = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5); r < rows; r += nw) {
    const float* xr = x + r * C;
    const float v = xw_quant_row([&](int k) { return __ldg(reinterpret_cast<const float4*>(xr + k)); }, C, norms[r],
                                 q + r * C, fac + r);
    if ((threadIdx.x & 31) == 0) {
      if (rho) rho[r] = v;
      if (rho_max) atomicMax(rho_max + r / rows_per_group, __float_as_uint(v));
    }
  }
}

// range[0] = max |x| (NaN counts as above every bound), range[1] = smallest non-zero norm; both as float bits, which order like
// the values for non-negative floats.  range[1] stays 0x7f7f7f7f (3.4e38) when every norm is zero.
__global__ void split_range_kernel(const float* __restrict__ x, size_t n, const float* __restrict__ norms, size_t n_tok,
                                   unsigned* __restrict__ range) {
  const size_t stride = (size_t)gridDim.x * blockDim.x;
  unsigned mx = 0u, mn = 0x7f7f7f7fu;
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    const unsigned b = __float_as_uint(x[i]) & 0x7fffffffu;
    mx = b > mx ? b : mx;
  }
  for (size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x; i < n_tok; i += stride) {
    const float v = norms[i];
    if (v > 0.f && __float_as_uint(v) < mn) mn = __float_as_uint(v);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    mx = max(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    mn = min(mn, __shfl_xor_sync(0xffffffffu, mn, o));
  }
  if ((threadIdx.x & 31) == 0) { atomicMax(range, mx); atomicMin(range + 1, mn); }
}

template <bool kRelu>
struct CorrEpi {
  const float* norms;      // [T][P]
  const float* desc_norm;  // [rows]
  const int* grp_frame;
  const int* grp_row0;
  const int* grp_map0;
  float* maps;
  int map_stride, P;
  unsigned long long* tkeys;   // optional [maps][n_tiles]: (tile maximum, first token holding it) keys for the head (corr.cuh)
  int n_tiles;
  const float* clamp = nullptr;   // optional [desc rows]: per-row replacement of the norm product's 1e-8 (scaled operands)
  struct State { float mx; int tok; };
  __device__ __forceinline__ void tile_begin(State& s) const { s.mx = -1.f; s.tok = 0; }   // map values are >= 0 (ReLU)
  __device__ __forceinline__ static float act(float v) { return kRelu ? fmaxf(v, 0.f) : v; }
  __device__ __forceinline__ void tile_end(State& s, int g, int r, int nt) const {
    if (tkeys)   // + 0.f: never the bit pattern of -0
      tkeys[(size_t)(grp_map0[g] + r) * n_tiles + nt] =
          ((unsigned long long)__float_as_uint(s.mx + 0.f) << 32) | (unsigned)(0x7fffffff - s.tok);
  }
  __device__ __forceinline__ void operator()(State& s, int g, int r, int col0, const float (&f)[32], int ncols) const {
    const float dn = desc_norm[grp_row0[g] + r];
    const float eps = clamp ? clamp[grp_row0[g] + r] : 1e-8f;
    const float* fn = norms + (size_t)grp_frame[g] * P + col0;
    float* out = maps + (size_t)(grp_map0[g] + r) * map_stride + col0;
    if (ncols == 32) {
#pragma unroll
      for (int i = 0; i < 32; i += 4) {
        // norms rows are only 4-byte aligned (P is odd): scalar broadcast loads
        float4 n4 = make_float4(__ldg(fn + i), __ldg(fn + i + 1), __ldg(fn + i + 2), __ldg(fn + i + 3));
        float4 o;
        o.x = act(corr_cos(f[i + 0], dn, n4.x, eps));
        o.y = act(corr_cos(f[i + 1], dn, n4.y, eps));
        o.z = act(corr_cos(f[i + 2], dn, n4.z, eps));
        o.w = act(corr_cos(f[i + 3], dn, n4.w, eps));
        *reinterpret_cast<float4*>(out + i) = o;
        // strict >: the first token of the tile holding the maximum (columns are visited in increasing order)
        if (o.x > s.mx) { s.mx = o.x; s.tok = col0 + i; }
        if (o.y > s.mx) { s.mx = o.y; s.tok = col0 + i + 1; }
        if (o.z > s.mx) { s.mx = o.z; s.tok = col0 + i + 2; }
        if (o.w > s.mx) { s.mx = o.w; s.tok = col0 + i + 3; }
      }
    } else {
#pragma unroll
      for (int i = 0; i < 32; ++i)
        if (i < ncols) {
          const float o = act(corr_cos(f[i], dn, fn[i], eps));
          out[i] = o;
          if (o > s.mx) { s.mx = o; s.tok = col0 + i; }
        }
    }
  }
};

size_t corr_tc_workspace_bytes(int total_rows, int C) { return 2 * align_up((size_t)total_rows * C * 2, 256); }

// wide groups on tensor cores; tile_start must already hold the plan (corr_plan_kernel).
int launch_corr_gemm_tc(const void* tpc_hi, const void* tpc_lo, const float* norms, int T, int C, int P,
                        const float* desc, int desc_rows, const float* desc_norm, const int* grp_frame,
                        const int* grp_row0, const int* grp_m, const int* grp_map0, const int* tile_start, int n_groups,
                        int max_tiles, float* maps, int map_stride, float* desc_split_ws, cudaStream_t st,
                        unsigned long long* tkeys, bool split_ready, int tile_rows, bool relu, const float* clamp,
                        const void* tpc_hilo) {
  static_assert(TC_BN == CORR_TILE, "the tile maxima are per GEMM N tile");
  DTK_CHECK_ARG(C % 8 == 0, "corr (tensor path): C must be a multiple of 8");
  DTK_CHECK_ARG(relu || tkeys == nullptr, "corr (tensor path): tile keys need the ReLU maps");
  DTK_CHECK_ARG(!tpc_hilo || (relu && C % 32 == 0), "corr (tensor path): interleaved operands need C %% 32 == 0 and ReLU maps");
  const bool pairs = tile_rows == TC2_BM;   // tile_start was planned with this M tile
  const TcProblem pb{grp_frame, grp_row0, grp_m, tile_start, n_groups, P, C};
  if (tpc_hilo) {   // descriptors interleaved like the features: [desc_rows][2 C] at the start of the workspace
    int rc = split_ready ? DINOTRK_OK : launch_split_hilo(desc, desc_split_ws, desc_rows, C, st);
    if (rc) return rc;
    const TcOperands op{desc_split_ws, nullptr, (uint64_t)desc_rows, 0, tpc_hilo, nullptr, (uint64_t)T, 0};
    using Epi = CorrEpi<true>;
    const Epi epi{norms, desc_norm, grp_frame, grp_row0, grp_map0, maps, map_stride, P, tkeys, cdiv(P, CORR_TILE)};
    return pairs ? tc_launch<TcMode::F16X3I, Epi, TC_BN, true>(op, pb, max_tiles, epi, st, PROF_CORR_GEMM)
                 : tc_launch<TcMode::F16X3I, Epi>(op, pb, max_tiles, epi, st, PROF_CORR_GEMM);
  }
  const DescSplit d(desc_split_ws, desc_rows, C);
  int rc = split_ready ? DINOTRK_OK : launch_split_f16(desc, d.hi, d.lo, (size_t)desc_rows * C, st);
  if (rc) return rc;
  const TcOperands op{d.hi, d.lo, (uint64_t)desc_rows, 0, tpc_hi, tpc_lo, (uint64_t)T, 0};
  auto run = [&](const auto& epi) {
    using Epi = std::decay_t<decltype(epi)>;
    return pairs ? tc_launch<TcMode::F16X3, Epi, TC_BN, true>(op, pb, max_tiles, epi, st, PROF_CORR_GEMM)
                 : tc_launch<TcMode::F16X3, Epi>(op, pb, max_tiles, epi, st, PROF_CORR_GEMM);
  };
  if (relu)
    return run(CorrEpi<true>{norms, desc_norm, grp_frame, grp_row0, grp_map0, maps, map_stride, P, tkeys, cdiv(P, CORR_TILE)});
  return run(CorrEpi<false>{norms, desc_norm, grp_frame, grp_row0, grp_map0, maps, map_stride, P, nullptr, cdiv(P, CORR_TILE),
                            clamp});
}

}  // namespace dtk

using namespace dtk;

extern "C" int dinotrk_split_fp16(const float* x, void* hi, void* lo, size_t n, void* stream) {
  DTK_CHECK_ARG(x && hi && lo, "split_fp16: null pointer");
  return launch_split_f16(x, hi, lo, n, (cudaStream_t)stream);
}

extern "C" int dinotrk_split_hilo(const float* x, void* hilo, size_t rows, int C, void* stream) {
  DTK_CHECK_ARG(x && hilo, "split_hilo: null pointer");
  return launch_split_hilo(x, hilo, rows, C, (cudaStream_t)stream);
}

extern "C" int dinotrk_split_range(const float* x, size_t n, const float* norms, size_t n_tok, float* range, void* stream) {
  DTK_CHECK_ARG(x && norms && range, "split_range: null pointer");
  cudaStream_t st = (cudaStream_t)stream;
  unsigned* r = reinterpret_cast<unsigned*>(range);
  DTK_CUDA(cudaMemsetAsync(r, 0, sizeof(unsigned), st));
  DTK_CUDA(cudaMemsetAsync(r + 1, 0x7f, sizeof(unsigned), st));
  size_t m = n > n_tok ? n : n_tok;
  unsigned grid = (unsigned)((m + 255) / 256);
  if (grid > (unsigned)num_sms() * 8) grid = num_sms() * 8;
  if (grid == 0) return DINOTRK_OK;
  ProfRange pr(PROF_MISC, st);
  split_range_kernel<<<grid, 256, 0, st>>>(x, n, norms, n_tok, r);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

extern "C" int dinotrk_split_faithful(float max_abs, float min_norm, int C) {
  return (max_abs <= SPLIT_MAX_ABS && min_norm >= split_min_norm(C)) ? 1 : 0;
}

extern "C" int dinotrk_quantise_s8(const float* x, const float* norms, size_t rows, int C, int rows_per_group, void* q, float* fac,
                                   float* rho, float* rho_max, void* stream) {
  DTK_CHECK_ARG(x && norms && q && fac, "quantise_s8: null pointer");
  DTK_CHECK_ARG(C > 0 && C % 16 == 0 && rows_per_group > 0, "quantise_s8: C must be a positive multiple of 16");
  if (rows == 0) return DINOTRK_OK;
  cudaStream_t st = (cudaStream_t)stream;
  if (rho_max) DTK_CUDA(cudaMemsetAsync(rho_max, 0, ((rows + rows_per_group - 1) / rows_per_group) * sizeof(float), st));
  size_t grid = (rows + 7) / 8;
  if (grid > (size_t)num_sms() * 16) grid = (size_t)num_sms() * 16;
  ProfRange pr(PROF_MISC, st);
  quant_s8_kernel<<<(unsigned)grid, 256, 0, st>>>(x, norms, rows, C, rows_per_group, reinterpret_cast<int8_t*>(q), fac, rho,
                                                  reinterpret_cast<unsigned*>(rho_max));
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

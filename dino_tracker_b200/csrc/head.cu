// Tracker head: arg-max, 2-layer normalised-conv refiner, spatial softmax, disc-masked soft-argmax
// with the numerical-stability fallback (models/networks/tracker_head.py:107-121, :68-98, :100-105;
// conv_norm.py:34-46; data/dataset.py:21-53).
//
// Two kernels:
//  * head_window_kernel (fast path, every map): arg-max, then the EXACT refiner only on the 11x11 box around
//    the arg-max (hidden layer on 13x13, input window 15x15).  The soft-argmax needs nothing else as long as
//    the numerical-stability branch (disc mass < 1e-8 of the whole softmax) does not fire; that is certified
//    with a rigorous, monotone upper bound on every logit outside the box (from the largest map value outside
//    the 7x7 core and the positive parts of the normalised weights).  Maps that cannot be certified are
//    queued for
//  * head_kernel (full map): the complete refiner + softmax, exactly as the reference evaluates it.
//
// head_kernel: one persistent CTA per SM; one warp per 4-row band of the map, one lane per 4x4-pixel tile
// (band = 32 tiles = 128 columns >= w).  Per hidden channel a lane computes its 16 hidden values from
// the 6x6 input window it keeps in registers, publishes its top/bottom rows to shared memory (the only
// cross-warp traffic), takes the side/corner halo from its lane neighbours by shuffle and
// accumulates the second convolution into 16 registers.  The next map is prefetched with cp.async
// while the current one is being refined.
//
// Grids wider or taller than 128 tokens take head_big_kernel for the full map instead (thread = 4x4 tile recomputing its
// hidden halo, one map buffer); both fast-path kernels work on any grid of the envelope.
#include <algorithm>

#include "common.cuh"
#include "corr.cuh"
#include "head.cuh"

namespace dtk {

constexpr int HEAD_MAX_W = 128, HEAD_MAX_H = 128;

__device__ __forceinline__ void cp_async16_head(void* smem, const void* gmem) {
  unsigned s = (unsigned)__cvta_generic_to_shared(smem);
  asm volatile("cp.async.cg.shared.global [%0], [%1], 16;\n" ::"r"(s), "l"(gmem));
}

template <typename T>
__device__ __forceinline__ T block_bcast_reduce(T v, T* red, int warp, int lane, int nwarps, T (*op)(T, T)) {
  // warp-level then cross-warp; every thread returns the result
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v = op(v, __shfl_xor_sync(0xffffffffu, v, o));
  __syncthreads();
  if (lane == 0) red[warp] = v;
  __syncthreads();
  T r = red[0];
  for (int k = 1; k < nwarps; ++k) r = op(r, red[k]);
  return r;
}
__device__ __forceinline__ float opmax(float a, float b) { return fmaxf(a, b); }
__device__ __forceinline__ float opadd(float a, float b) { return a + b; }
// arg-max key: larger value wins, ties -> smaller index (torch.argmax returns the first maximum).
// Values are >= 0 (ReLU'd), so the float bit pattern orders like the value.
__device__ __forceinline__ unsigned long long opkey(unsigned long long a, unsigned long long b) { return a > b ? a : b; }

// online-softmax pair (max, sum of exp relative to max)
struct MS { float m, s; };
__device__ __forceinline__ MS ms_merge(MS a, MS b) {
  float m = fmaxf(a.m, b.m);
  float sa = a.m == -INFINITY ? 0.f : a.s * __expf(a.m - m);
  float sb = b.m == -INFINITY ? 0.f : b.s * __expf(b.m - m);
  return MS{m, sa + sb};
}
struct F3 { float a, b, c; };

// kWrap: the band's last lane (tile 31) lies completely outside the map (w <= 124), so the side halo can be
// taken with rotating shuffles (lane 0 reads the all-zero tile 31) -- no edge selects in the hot loop.
template <int MAXT, bool kWrap>
__global__ void __launch_bounds__(MAXT, 1)
head_kernel(const float* __restrict__ maps, int n_maps_arg, const int* __restrict__ map_list,
            const int* __restrict__ list_count, HeadParams hp, dinotrk_head_weights wts,
            const int* __restrict__ out_index, float* __restrict__ out, int* __restrict__ aux) {
  extern __shared__ __align__(16) float smem[];
  // with a list: process map_list[0 .. *list_count) (maps the window kernel could not certify)
  const int n_maps = map_list ? *list_count : n_maps_arg;
  auto map_of = [&](int k) { return map_list ? map_list[k] : k; };
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
  const int h = hp.h, w = hp.w, P = hp.P;
  const int lin_elems = (hp.map_stride + 3) & ~3;
  float* sm_lin[2] = {smem, smem + lin_elems};
  float* sm_hid = smem + 2 * lin_elems;                   // [2 buffers][nwarps][2 rows][128]
  float* sm_red = sm_hid + 2 * nwarps * 2 * 128;          // [3 * 32] floats
  unsigned long long* sm_red64 = reinterpret_cast<unsigned long long*>(sm_red + 96);  // [32]

  const int r0 = warp * 4, c0 = lane * 4;  // this lane's tile
  const int nchunks = hp.map_stride / 4;
  constexpr float kNeg = -1e30f;
  // additive masks: hidden activations of pixels outside the map must be exactly 0 (zero padding of the
  // second convolution); bias + kNeg makes the ReLU do that without per-pixel selects.
  float rmask[4], cmask[4];
#pragma unroll
  for (int i = 0; i < 4; ++i) { rmask[i] = (r0 + i < h) ? 0.f : kNeg; cmask[i] = (c0 + i < w) ? 0.f : kNeg; }
  const int lane_l = (lane + 31) & 31, lane_r = (lane + 1) & 31;

  int mk = blockIdx.x;
  if (mk < n_maps) {
    const float4* src = reinterpret_cast<const float4*>(maps + (size_t)map_of(mk) * hp.map_stride);
    for (int i = threadIdx.x; i < nchunks; i += blockDim.x) cp_async16_head(sm_lin[0] + 4 * i, src + i);
  }
  asm volatile("cp.async.commit_group;\n" ::);

  for (int it = 0; mk < n_maps; mk += gridDim.x, ++it) {
    const int map = map_of(mk);
    const float* lin = sm_lin[it & 1];
    {  // prefetch the next map into the other buffer
      int nmk = mk + gridDim.x;
      if (nmk < n_maps) {
        const float4* src = reinterpret_cast<const float4*>(maps + (size_t)map_of(nmk) * hp.map_stride);
        float* dst = sm_lin[(it + 1) & 1];
        for (int i = threadIdx.x; i < nchunks; i += blockDim.x) cp_async16_head(dst + 4 * i, src + i);
      }
      asm volatile("cp.async.commit_group;\n" ::);
      asm volatile("cp.async.wait_group 1;\n" ::);
    }
    __syncthreads();

    // ---- arg-max of the (already ReLU'd) map: first maximal index ----------------------------
    unsigned long long key = 0ull;
    for (int i = threadIdx.x; i < P; i += blockDim.x) {
      float v = lin[i] + 0.f;  // -0.0 -> +0.0 so that the bit pattern orders like the value
      unsigned long long k = ((unsigned long long)__float_as_uint(v) << 32) | (unsigned)(0x7fffffff - i);
      key = k > key ? k : key;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, key, o); key = t > key ? t : key; }
    if (lane == 0) sm_red64[warp] = key;

    // ---- 6x6 input window (zero outside the map = conv zero padding) -------------------------
    float m[6][6];
#pragma unroll
    for (int i = 0; i < 6; ++i) {
      int r = r0 - 1 + i;
#pragma unroll
      for (int j = 0; j < 6; ++j) {
        int c = c0 - 1 + j;
        m[i][j] = (r >= 0 && r < h && c >= 0 && c < w) ? lin[r * w + c] : 0.f;
      }
    }

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j) acc[i][j] = wts.b2;

    float hid[6][6];  // [1..4][1..4] own values, ring = halo
    auto conv1 = [&](int o) {
      float w1[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) w1[k] = wts.w1[o][k];
      const float b1 = wts.b1[o];
#pragma unroll
      for (int i = 0; i < 4; ++i) {
        const float br = b1 + rmask[i];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float a = br + cmask[j];
#pragma unroll
          for (int ki = 0; ki < 3; ++ki)
#pragma unroll
            for (int kj = 0; kj < 3; ++kj) a = fmaf(w1[ki * 3 + kj], m[i + ki][j + kj], a);
          hid[i + 1][j + 1] = fmaxf(a, 0.f);
        }
      }
      float* hb = sm_hid + ((o & 1) * nwarps + warp) * 2 * 128;
      *reinterpret_cast<float4*>(hb + c0) = make_float4(hid[1][1], hid[1][2], hid[1][3], hid[1][4]);
      *reinterpret_cast<float4*>(hb + 128 + c0) = make_float4(hid[4][1], hid[4][2], hid[4][3], hid[4][4]);
    };

    conv1(0);
    __syncthreads();  // also publishes sm_red64 (arg-max partials)
#pragma unroll 1
    for (int o = 0; o < 16; ++o) {
      float w2[9];
#pragma unroll
      for (int k = 0; k < 9; ++k) w2[k] = wts.w2[o][k];
      // halo rows of channel o were published before the previous barrier
      float4 top = make_float4(0.f, 0.f, 0.f, 0.f), bot = top;
      if (warp > 0) top = *reinterpret_cast<const float4*>(sm_hid + ((o & 1) * nwarps + warp - 1) * 2 * 128 + 128 + c0);
      if (warp + 1 < nwarps) bot = *reinterpret_cast<const float4*>(sm_hid + ((o & 1) * nwarps + warp + 1) * 2 * 128 + c0);
      hid[0][1] = top.x; hid[0][2] = top.y; hid[0][3] = top.z; hid[0][4] = top.w;
      hid[5][1] = bot.x; hid[5][2] = bot.y; hid[5][3] = bot.z; hid[5][4] = bot.w;
#pragma unroll
      for (int i = 0; i < 6; ++i) {
        if (kWrap) {
          hid[i][0] = __shfl_sync(0xffffffffu, hid[i][4], lane_l);
          hid[i][5] = __shfl_sync(0xffffffffu, hid[i][1], lane_r);
        } else {
          float l = __shfl_up_sync(0xffffffffu, hid[i][4], 1);
          float r = __shfl_down_sync(0xffffffffu, hid[i][1], 1);
          hid[i][0] = lane > 0 ? l : 0.f;
          hid[i][5] = lane < 31 ? r : 0.f;
        }
      }
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          float a = acc[i][j];
#pragma unroll
          for (int ki = 0; ki < 3; ++ki)
#pragma unroll
            for (int kj = 0; kj < 3; ++kj) a = fmaf(w2[ki * 3 + kj], hid[i + ki][j + kj], a);
          acc[i][j] = a;
        }
      if (o + 1 < 16) conv1(o + 1);   // next channel's hidden layer; published by the barrier below
      __syncthreads();
    }

    // ---- arg-max result (partials were published before the first barrier) ---------------------
    unsigned long long kbest = sm_red64[0];
    for (int k = 1; k < nwarps; ++k) { unsigned long long t = sm_red64[k]; kbest = t > kbest ? t : kbest; }
    const int amax = 0x7fffffff - (int)(kbest & 0xffffffffu);
    const int arow = amax / w, acol = amax - arow * w;

    // ---- softmax statistics over the whole map: one online (max, sum) reduction --------------------
    MS ms{-INFINITY, 0.f};
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (r0 + i < h && c0 + j < w) ms.m = fmaxf(ms.m, acc[i][j]);
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
      for (int j = 0; j < 4; ++j)
        if (r0 + i < h && c0 + j < w) ms.s += __expf(acc[i][j] - ms.m);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      MS t{__shfl_xor_sync(0xffffffffu, ms.m, o), __shfl_xor_sync(0xffffffffu, ms.s, o)};
      ms = ms_merge(ms, t);
    }
    if (lane == 0) { sm_red[warp] = ms.m; sm_red[32 + warp] = ms.s; }
    __syncthreads();
    float zmax = -INFINITY;
    for (int k = 0; k < nwarps; ++k) zmax = fmaxf(zmax, sm_red[k]);

    // ---- disc-masked soft-argmax (mask: |token centre - argmax centre| <= radius px) ----------
    // Only the few threads whose tile meets the disc do any work; exact expf / division here.
    float s = 0.f, sx = 0.f, sy = 0.f, gx = 0.f, gy = 0.f, cnt = 0.f, ssum_part = 0.f;
    {
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const bool disc = in_disc(hp, r0 + i, c0 + j, arow, acol);
          if (r0 + i < h && c0 + j < w && disc) {
            float e = expf(acc[i][j] - zmax);
            float x = token_px(hp, c0 + j), y = token_px(hp, r0 + i);
            s += e; sx = fmaf(x, e, sx); sy = fmaf(y, e, sy);
            gx += x; gy += y; cnt += 1.f;
          }
        }
    }
    // global sum of exp(z - zmax) from the per-warp (max, sum) pairs
    for (int k = 0; k < nwarps; ++k) {
      float mk = sm_red[k];
      if (mk != -INFINITY) ssum_part += sm_red[32 + k] * expf(mk - zmax);
    }
    const float ssum = ssum_part;
    // reduce (s, sx, sy, gx, gy, cnt) in one pass
    float vals[6] = {s, sx, sy, gx, gy, cnt};
#pragma unroll
    for (int q = 0; q < 6; ++q)
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) vals[q] += __shfl_xor_sync(0xffffffffu, vals[q], o);
    __syncthreads();  // everyone has read sm_red (max/sum pairs) -> reuse it
    if (lane == 0) {
#pragma unroll
      for (int q = 0; q < 6; ++q) sm_red[q * 32 + warp] = vals[q];
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      float tot[6];
      for (int q = 0; q < 6; ++q) { float t = 0.f; for (int k = 0; k < nwarps; ++k) t += sm_red[q * 32 + k]; tot[q] = t; }
      head_full_finish(hp, tot, ssum, map, amax, out_index, out, aux);
    }
    __syncthreads();  // lin / sm_hid / sm_red are reused by the next iteration
  }
  asm volatile("cp.async.wait_group 0;\n" ::);
}


// ------------------------------------------------------------------------------------------------------
// Fast path: exact refiner on the 11x11 box around the arg-max + certified absence of the fallback branch.
constexpr int WIN_THREADS = 128;

__global__ void __launch_bounds__(WIN_THREADS)
head_window_kernel(const float* __restrict__ maps, int n_maps, HeadParams hp, dinotrk_head_weights wts,
                   const int* __restrict__ out_index, float* __restrict__ out, int* __restrict__ aux,
                   int* __restrict__ slow_list, int* __restrict__ slow_count) {
  extern __shared__ __align__(16) float smem[];
  const int lin_elems = (hp.map_stride + 3) & ~3;
  float* lin = smem;                           // one map (several CTAs per SM hide the load latency)
  float* sm_m = smem + lin_elems;              // [WM][WM] input window, zero outside the map
  float* sm_h = sm_m + WM * WM + 3;            // [16][WH][WH] hidden window, zero outside the map
  float* sm_red = sm_h + 16 * WH * WH;         // partials
  unsigned long long* sm_key = reinterpret_cast<unsigned long long*>(sm_red + 32);  // [4]
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int h = hp.h, w = hp.w, P = hp.P;
  const int nchunks = hp.map_stride / 4;       // float4 chunks; the tail of the last chunk (>= P) is masked below

  for (int map = blockIdx.x; map < n_maps; map += gridDim.x) {
    {
      const float4* src = reinterpret_cast<const float4*>(maps + (size_t)map * hp.map_stride);
      for (int i = tid; i < nchunks; i += WIN_THREADS) cp_async16_head(lin + 4 * i, src + i);
      asm volatile("cp.async.commit_group;\n" ::);
      asm volatile("cp.async.wait_group 0;\n" ::);
    }
    __syncthreads();

    // ---- arg-max (first maximal index): chunk-wise maxima, then the first chunk / element holding the max ----
    float best = -1.f;
    int bchunk = 0;
    for (int i = tid; i < nchunks; i += WIN_THREADS) {
      float4 v = *reinterpret_cast<const float4*>(lin + 4 * i);
      const int base = 4 * i;
      float m4 = v.x;                                          // element base always < P
      if (base + 1 < P) m4 = fmaxf(m4, v.y);
      if (base + 2 < P) m4 = fmaxf(m4, v.z);
      if (base + 3 < P) m4 = fmaxf(m4, v.w);
      if (m4 > best) { best = m4; bchunk = i; }                // strict: keeps the first chunk of this thread
    }
    // threads without a chunk (tiny maps) must not win: key 0 (values are >= 0, so real keys order like floats)
    unsigned long long key = best < 0.f ? 0ull
        : (((unsigned long long)__float_as_uint(best + 0.f) << 32) | (unsigned)(0x7fffffff - bchunk));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, key, o); key = t > key ? t : key; }
    if (lane == 0) sm_key[warp] = key;
    __syncthreads();
    unsigned long long kb = sm_key[0];
#pragma unroll
    for (int k = 1; k < WIN_THREADS / 32; ++k) { unsigned long long t = sm_key[k]; kb = t > kb ? t : kb; }
    const int wchunk = 0x7fffffff - (int)(kb & 0xffffffffu);
    const float vmax = __uint_as_float((unsigned)(kb >> 32));
    int amax = 4 * wchunk;
    {
      const float* q = lin + 4 * wchunk;
      amax += (q[0] + 0.f == vmax) ? 0 : (q[1] + 0.f == vmax) ? 1 : (q[2] + 0.f == vmax) ? 2 : 3;
    }
    const int arow = amax / w, acol = amax - arow * w;

    // ---- input window (15 x 15, zero outside the map) ---------------------------------------------
    for (int i = tid; i < WM * WM; i += WIN_THREADS) {
      int y = i / WM, x = i - y * WM;
      int r = arow - 7 + y, c = acol - 7 + x;
      sm_m[i] = (r >= 0 && r < h && c >= 0 && c < w) ? lin[r * w + c] : 0.f;
    }
    __syncthreads();
    // ---- largest map value outside the 7x7 core: blank the core in the private copy, then a plain max ----
    if (tid < 49) {
      int r = arow - 3 + tid / 7, c = acol - 3 + tid % 7;
      if (r >= 0 && r < h && c >= 0 && c < w) lin[r * w + c] = 0.f;
    }
    // ---- hidden layer on the 13 x 13 window (zero outside the map: padding of the second conv) -----
    for (int i = tid; i < WH * WH; i += WIN_THREADS) {
      int y = i / WH, x = i - y * WH;
      int r = arow - 6 + y, c = acol - 6 + x;
      const bool inside = r >= 0 && r < h && c >= 0 && c < w;
      float mw[9];
#pragma unroll
      for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) mw[ky * 3 + kx] = sm_m[(y + ky) * WM + x + kx];
#pragma unroll 4
      for (int o = 0; o < 16; ++o) {
        float a = wts.b1[o];
#pragma unroll
        for (int k = 0; k < 9; ++k) a = fmaf(wts.w1[o][k], mw[k], a);
        sm_h[o * WH * WH + i] = inside ? fmaxf(a, 0.f) : 0.f;
      }
    }
    __syncthreads();
    float mout = 0.f;
    for (int i = tid; i < nchunks; i += WIN_THREADS) {
      float4 v = *reinterpret_cast<const float4*>(lin + 4 * i);
      const int base = 4 * i;
      float m4 = v.x;
      if (base + 1 < P) m4 = fmaxf(m4, v.y);
      if (base + 2 < P) m4 = fmaxf(m4, v.z);
      if (base + 3 < P) m4 = fmaxf(m4, v.w);
      mout = fmaxf(mout, m4);
    }
    mout = warp_max(mout);

    // ---- logits on the 11 x 11 box; thread = box pixel ----------------------------------------------
    float z = -INFINITY;
    bool valid = false, indisc = false;
    float px = 0.f, py = 0.f;
    if (tid < WB * WB) {
      int y = tid / WB, x = tid - y * WB;
      int r = arow - 5 + y, c = acol - 5 + x;
      valid = r >= 0 && r < h && c >= 0 && c < w;
      if (valid) {
        float a = wts.b2;
#pragma unroll 4
        for (int o = 0; o < 16; ++o) {
          const float* hb = sm_h + o * WH * WH + y * WH + x;
#pragma unroll
          for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) a = fmaf(wts.w2[o][ky * 3 + kx], hb[ky * WH + kx], a);
        }
        z = a;
        indisc = in_disc(hp, r, c, arow, acol);
        px = token_px(hp, c);
        py = token_px(hp, r);
      }
    }
    float zmax = warp_max(z);
    if (lane == 0) { sm_red[warp] = mout; sm_red[8 + warp] = zmax; }
    __syncthreads();
    mout = fmaxf(fmaxf(sm_red[0], sm_red[1]), fmaxf(sm_red[2], sm_red[3]));
    zmax = fmaxf(fmaxf(sm_red[8], sm_red[9]), fmaxf(sm_red[10], sm_red[11]));
    const float e = valid ? expf(z - zmax) : 0.f;
    float v5[5] = {e, indisc ? e : 0.f, indisc ? px * e : 0.f, indisc ? py * e : 0.f, valid ? 1.f : 0.f};
#pragma unroll
    for (int q = 0; q < 5; ++q) v5[q] = warp_sum(v5[q]);
    if (lane == 0) {
#pragma unroll
      for (int q = 0; q < 5; ++q) sm_red[12 + q * 4 + warp] = v5[q];
    }
    __syncthreads();
    if (tid == 0) {
      float tot[5];
#pragma unroll
      for (int q = 0; q < 5; ++q) tot[q] = sm_red[12 + q * 4] + sm_red[13 + q * 4] + sm_red[14 + q * 4] + sm_red[15 + q * 4];
      if (head_certified(hp, wts, mout, zmax, tot)) {
        head_store_point(hp, __fdiv_rn(tot[2], tot[1]), __fdiv_rn(tot[3], tot[1]), out_index, out, map);
        if (aux) { aux[2 * map] = amax; aux[2 * map + 1] = 0; }
      } else {
        slow_list[atomicAdd(slow_count, 1)] = map;
      }
    }
    __syncthreads();  // lin / windows are reused by the next iteration
  }
}

// ------------------------------------------------------------------------------------------------------
// Fast path on the tensor-core pipeline: the correlation GEMM epilogue leaves, per map and 256-token tile, one 64-bit key
// (value bits << 32 | 0x7fffffff - first token holding it; corr.cuh), so the arg-max is a 32-key reduction and the largest
// value outside the 7x7 core needs only the ~1 k tokens of the tiles that touch the core rows.  The map itself is touched
// for the 15x15 window and those tokens only.  Same certificate and same per-value arithmetic as head_window_kernel;
// the work is laid out so that the refiner weights sit in registers (hidden layer: thread = channel x row, weights of
// that channel loaded once per kernel) or shared memory (output layer), not in constant-bank operands.
constexpr int TMK_THREADS = 128;
constexpr int WMP = 16;   // pitch of the input window rows (15 used): float4 loads
constexpr int WHC = 20;   // hidden window [position][16 channels], 20-float pitch: float4 reads of consecutive positions
                          // fall into distinct bank groups

__global__ void __launch_bounds__(TMK_THREADS, 12)   // 40 registers: 12 CTAs per SM hide the per-map latency chain
head_tm_kernel(const float* __restrict__ maps, const unsigned long long* __restrict__ tkeys, int n_tiles, int n_maps,
               HeadParams hp, dinotrk_head_weights wts, const int* __restrict__ out_index, float* __restrict__ out,
               int* __restrict__ aux, int* __restrict__ slow_list, int* __restrict__ slow_count) {
  __shared__ __align__(16) float sm_m[WM * WMP];          // input window, zero outside the map
  __shared__ __align__(16) float sm_h[WH * WH * WHC];     // hidden window, zero outside the map
  __shared__ __align__(16) float sm_w2[4 * 9 * 4];        // output-layer weights [channel / 4][tap][channel % 4]
  __shared__ float sm_red[32];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int h = hp.h, w = hp.w, P = hp.P;
  const int ch = tid & 15, rg = tid >> 4;                 // hidden layer: channel, row group
  float w1r[9];
#pragma unroll
  for (int k = 0; k < 9; ++k) w1r[k] = wts.w1[ch][k];
  const float b1r = wts.b1[ch];
  for (int i = tid; i < 4 * 9 * 4; i += TMK_THREADS) { const int o4 = i / 36, k = (i / 4) % 9, j = i & 3; sm_w2[i] = wts.w2[o4 * 4 + j][k]; }
  __syncthreads();

  int map = blockIdx.x;
  unsigned long long knext = (map < n_maps && lane < n_tiles) ? __ldg(tkeys + (size_t)map * n_tiles + lane) : 0ull;
  for (; map < n_maps; map += gridDim.x) {
    const float* src = maps + (size_t)map * hp.map_stride;
    const unsigned long long* tk = tkeys + (size_t)map * n_tiles;
    // ---- arg-max from the tile keys (every warp redundantly; keys of the next map are already in flight) ----
    unsigned long long kown = knext, key = knext;
    {
      const int nm = map + gridDim.x;
      knext = (nm < n_maps && lane < n_tiles) ? __ldg(tkeys + (size_t)nm * n_tiles + lane) : 0ull;
    }
    for (int t = lane + 32; t < n_tiles; t += 32) { unsigned long long k = __ldg(tk + t); key = k > key ? k : key; }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, key, o); key = t > key ? t : key; }
    if (key == ~0ull) {   // thin group (streaming kernel): no tile keys -> full-map kernel
      if (tid == 0) slow_list[atomicAdd(slow_count, 1)] = map;
      continue;
    }
    const int amax = 0x7fffffff - (int)(key & 0xffffffffu);
    const int arow = amax / w, acol = amax - arow * w;
    // ---- largest map value outside the 7x7 core: whole tiles from the keys, the tiles touching the core rows token-wise
    const int t_lo = (max(arow - 3, 0) * w + max(acol - 3, 0)) / CORR_TILE;
    const int t_hi = (min(arow + 3, h - 1) * w + min(acol + 3, w - 1)) / CORR_TILE;
    float mout = 0.f;
    if (lane < n_tiles && (lane < t_lo || lane > t_hi)) mout = __uint_as_float((unsigned)(kown >> 32));
    for (int t = lane + 32; t < n_tiles; t += 32)
      if (t < t_lo || t > t_hi) mout = fmaxf(mout, __uint_as_float((unsigned)(__ldg(tk + t) >> 32)));
    if (warp != 0) mout = 0.f;   // the keys are counted once
    // All global loads of this map (window + the tokens of the tiles touching the core rows) are issued before any is
    // consumed: one DRAM round trip per map instead of one per row.
    constexpr int WROUNDS = (WM * WMP + TMK_THREADS - 1) / TMK_THREADS;
    float wv[WROUNDS];
#pragma unroll
    for (int q = 0; q < WROUNDS; ++q) {
      const int i = tid + q * TMK_THREADS;
      const int y = i >> 4, x = i & 15;
      const int r = arow - 7 + y, c = acol - 7 + x;
      wv[q] = (i < WM * WMP && x < WM && r >= 0 && r < h && c >= 0 && c < w) ? __ldg(src + r * w + c) : 0.f;
    }
    {
      const int tok_lo = t_lo * CORR_TILE, tok_hi = min((t_hi + 1) * CORR_TILE, P);   // [tok_lo, tok_hi)
      const int r_lo = tok_lo / w, r_hi = (tok_hi - 1) / w;
      constexpr int RB = 12;   // rows per batch of loads (4 tiles of 256 tokens span <= 10 rows at w = 121)
      for (int c = tid; c < w; c += TMK_THREADS)
        for (int rb = r_lo; rb <= r_hi; rb += RB) {
          float tv[RB];
#pragma unroll
          for (int j = 0; j < RB; ++j) {
            const int r = rb + j, p = r * w + c;
            const bool ok = r <= r_hi && p >= tok_lo && p < tok_hi && !(abs(r - arow) <= 3 && abs(c - acol) <= 3);
            tv[j] = ok ? __ldg(src + p) : 0.f;
          }
#pragma unroll
          for (int j = 0; j < RB; ++j) mout = fmaxf(mout, tv[j]);
        }
    }
    // ---- input window (15 x 15, zero outside the map) ---------------------------------------------
#pragma unroll
    for (int q = 0; q < WROUNDS; ++q) {
      const int i = tid + q * TMK_THREADS;
      if (i < WM * WMP) sm_m[i] = wv[q];
    }
    __syncthreads();
    // ---- hidden layer on the 13 x 13 window: thread = (channel, row); taps in (ky, kx) order as everywhere else ----
    for (int y = rg; y < WH; y += TMK_THREADS / 16) {
      const int r = arow - 6 + y;
      const bool row_in = r >= 0 && r < h;
      // 3 x 3 input window sliding along the row: three new values per output (broadcast loads: the 16 channel
      // threads of a row read the same addresses), few live registers -> 12 CTAs per SM
      const float* m0 = sm_m + y * WMP;
      float i00 = m0[0], i01 = m0[1], i10 = m0[WMP], i11 = m0[WMP + 1], i20 = m0[2 * WMP], i21 = m0[2 * WMP + 1];
#pragma unroll
      for (int x = 0; x < WH; ++x) {
        const float i02 = m0[x + 2], i12 = m0[WMP + x + 2], i22 = m0[2 * WMP + x + 2];
        float a = b1r;
        a = fmaf(w1r[0], i00, a); a = fmaf(w1r[1], i01, a); a = fmaf(w1r[2], i02, a);
        a = fmaf(w1r[3], i10, a); a = fmaf(w1r[4], i11, a); a = fmaf(w1r[5], i12, a);
        a = fmaf(w1r[6], i20, a); a = fmaf(w1r[7], i21, a); a = fmaf(w1r[8], i22, a);
        const int c = acol - 6 + x;
        sm_h[(y * WH + x) * WHC + ch] = (row_in && c >= 0 && c < w) ? fmaxf(a, 0.f) : 0.f;
        i00 = i01; i01 = i02; i10 = i11; i11 = i12; i20 = i21; i21 = i22;
      }
    }
    __syncthreads();
    mout = warp_max(mout);

    // ---- logits on the 11 x 11 box; thread = box pixel ----
    float z = -INFINITY;
    bool valid = false, indisc = false;
    float px = 0.f, py = 0.f;
    if (tid < WB * WB) {
      const int y = tid / WB, x = tid - y * WB;
      const int r = arow - 5 + y, c = acol - 5 + x;
      valid = r >= 0 && r < h && c >= 0 && c < w;
      if (valid) {
        float a = wts.b2;
#pragma unroll
        for (int o4 = 0; o4 < 4; ++o4)
#pragma unroll
          for (int ky = 0; ky < 3; ++ky)
#pragma unroll
            for (int kx = 0; kx < 3; ++kx) {   // one float4 of hidden values (4 channels) x one float4 of weights per tap
              const float4 hv = *reinterpret_cast<const float4*>(sm_h + ((y + ky) * WH + x + kx) * WHC + o4 * 4);
              const float4 wv4 = *reinterpret_cast<const float4*>(sm_w2 + (o4 * 9 + ky * 3 + kx) * 4);
              a = fmaf(wv4.x, hv.x, a); a = fmaf(wv4.y, hv.y, a); a = fmaf(wv4.z, hv.z, a); a = fmaf(wv4.w, hv.w, a);
            }
        z = a;
        indisc = in_disc(hp, r, c, arow, acol);
        px = token_px(hp, c);
        py = token_px(hp, r);
      }
    }
    float zmax = warp_max(z);
    if (lane == 0) { sm_red[warp] = mout; sm_red[4 + warp] = zmax; }
    __syncthreads();
    mout = fmaxf(fmaxf(sm_red[0], sm_red[1]), fmaxf(sm_red[2], sm_red[3]));
    zmax = fmaxf(fmaxf(sm_red[4], sm_red[5]), fmaxf(sm_red[6], sm_red[7]));
    const float e = valid ? expf(z - zmax) : 0.f;
    float v5[5] = {e, indisc ? e : 0.f, indisc ? px * e : 0.f, indisc ? py * e : 0.f, valid ? 1.f : 0.f};
#pragma unroll
    for (int q = 0; q < 5; ++q) v5[q] = warp_sum(v5[q]);
    if (lane == 0) {
#pragma unroll
      for (int q = 0; q < 5; ++q) sm_red[8 + q * 4 + warp] = v5[q];
    }
    __syncthreads();
    if (tid == 0) {
      float tot[5];
#pragma unroll
      for (int q = 0; q < 5; ++q) tot[q] = sm_red[8 + q * 4] + sm_red[9 + q * 4] + sm_red[10 + q * 4] + sm_red[11 + q * 4];
      if (head_certified(hp, wts, mout, zmax, tot)) {
        head_store_point(hp, __fdiv_rn(tot[2], tot[1]), __fdiv_rn(tot[3], tot[1]), out_index, out, map);
        if (aux) { aux[2 * map] = amax; aux[2 * map + 1] = 0; }
      } else {
        slow_list[atomicAdd(slow_count, 1)] = map;
      }
    }
    // no barrier here: the next iteration writes sm_m before its 1st barrier (last read before this iteration's 2nd),
    // sm_h after its 1st (last read before this iteration's 3rd), sm_red[0..7] after its 2nd (read between the 3rd and
    // 4th) and sm_red[8..] after its 3rd -- which tid 0, the only reader after the 4th, has to reach first.
  }
}

// ------------------------------------------------------------------------------------------------------
// Full map on grids beyond head_kernel's band layout (w > 128 or h > 128, up to the DTK_GRID_MAX_* envelope): one CTA per
// map with the map once in shared memory (32,768 tokens = 128 KiB leave no room for a second buffer; several CTAs per SM
// hide the load instead).  Thread = 4 x 4 output tile.  Per hidden channel it recomputes its 6 x 6 hidden window from the
// 8 x 8 input window it keeps in registers, so no halo crosses threads and any grid shape works.  Every hidden value and
// logit is formed by the same operation sequence as in head_kernel (b1 then the 9 taps in (ky, kx) order; b2 then the
// channels).  The logits of the (2 box_r + 1)^2 box around the arg-max are kept for the disc soft-argmax.
constexpr int HB_THREADS = 256;
constexpr int HB_WARPS = HB_THREADS / 32;

__global__ void __launch_bounds__(HB_THREADS, 2)
head_big_kernel(const float* __restrict__ maps, int n_maps_arg, const int* __restrict__ map_list,
                const int* __restrict__ list_count, HeadParams hp, dinotrk_head_weights wts, int box_r,
                const int* __restrict__ out_index, float* __restrict__ out, int* __restrict__ aux) {
  extern __shared__ __align__(16) float smem[];
  const int n_maps = map_list ? *list_count : n_maps_arg;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int h = hp.h, w = hp.w, P = hp.P;
  const int lin_elems = (hp.map_stride + 3) & ~3;
  const int box_s = 2 * box_r + 1;
  float* lin = smem;
  float* sm_box = smem + lin_elems;                        // [box_s][box_s] logits around the arg-max
  float* sm_red = sm_box + ((box_s * box_s + 3) & ~3);     // [6][HB_WARPS]
  unsigned long long* sm_red64 = reinterpret_cast<unsigned long long*>(sm_red + 6 * HB_WARPS);  // [HB_WARPS]
  const int nchunks = hp.map_stride / 4;
  const int tiles_x = (w + 3) >> 2, n_tiles = tiles_x * ((h + 3) >> 2);

  for (int mk = blockIdx.x; mk < n_maps; mk += gridDim.x) {
    const int map = map_list ? map_list[mk] : mk;
    {
      const float4* src = reinterpret_cast<const float4*>(maps + (size_t)map * hp.map_stride);
      for (int i = tid; i < nchunks; i += HB_THREADS) cp_async16_head(lin + 4 * i, src + i);
      asm volatile("cp.async.commit_group;\n" ::);
      asm volatile("cp.async.wait_group 0;\n" ::);
    }
    __syncthreads();

    // ---- arg-max of the (already ReLU'd) map: first maximal index ----
    unsigned long long key = 0ull;
    for (int i = tid; i < P; i += HB_THREADS) {
      float v = lin[i] + 0.f;
      unsigned long long k = ((unsigned long long)__float_as_uint(v) << 32) | (unsigned)(0x7fffffff - i);
      key = k > key ? k : key;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { unsigned long long t = __shfl_xor_sync(0xffffffffu, key, o); key = t > key ? t : key; }
    if (lane == 0) sm_red64[warp] = key;
    __syncthreads();
    unsigned long long kbest = sm_red64[0];
#pragma unroll
    for (int k = 1; k < HB_WARPS; ++k) { unsigned long long t = sm_red64[k]; kbest = t > kbest ? t : kbest; }
    const int amax = 0x7fffffff - (int)(kbest & 0xffffffffu);
    const int arow = amax / w, acol = amax - arow * w;

    // ---- refiner, tile by tile; online (max, sum) of the softmax over the whole map ----
    MS ms{-INFINITY, 0.f};
    for (int t = tid; t < n_tiles; t += HB_THREADS) {
      const int r0 = (t / tiles_x) * 4, c0 = (t - (t / tiles_x) * tiles_x) * 4;
      float m[8][8];
#pragma unroll
      for (int i = 0; i < 8; ++i) {
        const int r = r0 - 2 + i;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
          const int c = c0 - 2 + j;
          m[i][j] = (r >= 0 && r < h && c >= 0 && c < w) ? lin[r * w + c] : 0.f;
        }
      }
      bool hin[6][6];   // hidden position inside the map (outside: 0, the zero padding of the second convolution)
#pragma unroll
      for (int i = 0; i < 6; ++i)
#pragma unroll
        for (int j = 0; j < 6; ++j) hin[i][j] = r0 - 1 + i >= 0 && r0 - 1 + i < h && c0 - 1 + j >= 0 && c0 - 1 + j < w;
      float acc[4][4];
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = wts.b2;
#pragma unroll 1
      for (int o = 0; o < 16; ++o) {
        float hid[6][6];
#pragma unroll
        for (int i = 0; i < 6; ++i)
#pragma unroll
          for (int j = 0; j < 6; ++j) {
            float a = wts.b1[o];
#pragma unroll
            for (int ki = 0; ki < 3; ++ki)
#pragma unroll
              for (int kj = 0; kj < 3; ++kj) a = fmaf(wts.w1[o][ki * 3 + kj], m[i + ki][j + kj], a);
            hid[i][j] = hin[i][j] ? fmaxf(a, 0.f) : 0.f;
          }
#pragma unroll
        for (int i = 0; i < 4; ++i)
#pragma unroll
          for (int j = 0; j < 4; ++j) {
            float a = acc[i][j];
#pragma unroll
            for (int ki = 0; ki < 3; ++ki)
#pragma unroll
              for (int kj = 0; kj < 3; ++kj) a = fmaf(wts.w2[o][ki * 3 + kj], hid[i + ki][j + kj], a);
            acc[i][j] = a;
          }
      }
      MS tm{-INFINITY, 0.f};
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j)
          if (r0 + i < h && c0 + j < w) tm.m = fmaxf(tm.m, acc[i][j]);
#pragma unroll
      for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) {
          const int r = r0 + i, c = c0 + j;
          if (r < h && c < w) {
            tm.s += __expf(acc[i][j] - tm.m);
            if (abs(r - arow) <= box_r && abs(c - acol) <= box_r) sm_box[(r - arow + box_r) * box_s + c - acol + box_r] = acc[i][j];
          }
        }
      ms = ms_merge(ms, tm);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
      MS t{__shfl_xor_sync(0xffffffffu, ms.m, o), __shfl_xor_sync(0xffffffffu, ms.s, o)};
      ms = ms_merge(ms, t);
    }
    if (lane == 0) { sm_red[warp] = ms.m; sm_red[HB_WARPS + warp] = ms.s; }
    __syncthreads();   // also publishes sm_box

    // ---- disc-masked soft-argmax (warp 0) with the stability branch, as head_kernel ----
    if (warp == 0) {
      float zmax = -INFINITY;
#pragma unroll
      for (int k = 0; k < HB_WARPS; ++k) zmax = fmaxf(zmax, sm_red[k]);
      float s = 0.f, sx = 0.f, sy = 0.f, gx = 0.f, gy = 0.f, cnt = 0.f;
      for (int q = lane; q < box_s * box_s; q += 32) {
        const int r = arow - box_r + q / box_s, c = acol - box_r + q % box_s;
        const bool disc = in_disc(hp, r, c, arow, acol);
        if (r >= 0 && r < h && c >= 0 && c < w && disc) {
          const float e = expf(sm_box[q] - zmax);
          const float x = token_px(hp, c), y = token_px(hp, r);
          s += e; sx = fmaf(x, e, sx); sy = fmaf(y, e, sy);
          gx += x; gy += y; cnt += 1.f;
        }
      }
      float vals[6] = {s, sx, sy, gx, gy, cnt};
#pragma unroll
      for (int q = 0; q < 6; ++q) vals[q] = warp_sum(vals[q]);
      if (lane == 0) {
        float ssum = 0.f;
#pragma unroll
        for (int k = 0; k < HB_WARPS; ++k) {
          const float mk_ = sm_red[k];
          if (mk_ != -INFINITY) ssum += sm_red[HB_WARPS + k] * expf(mk_ - zmax);
        }
        head_full_finish(hp, vals, ssum, map, amax, out_index, out, aux);
      }
    }
    __syncthreads();  // lin / sm_box / sm_red are reused by the next map
  }
}

__global__ void zero_int_kernel(int* p) { *p = 0; }

int launch_head(const float* maps, int n_maps, int map_stride, const dinotrk_geom& g,
                const dinotrk_head_weights& hw, const int* out_index, float* out, int out_stride, int out_mode,
                int* aux, int* scratch, cudaStream_t st, const unsigned long long* tkeys, bool counter_zeroed,
                int parts) {
  if (n_maps <= 0) return DINOTRK_OK;
  DTK_CHECK_GRID(g, "head");
  const HeadParams hp = make_head_params(g, hw, map_stride, out_stride, out_mode);
  const int sms = num_sms();
  const int lin_elems = (map_stride + 3) & ~3;
  // the window fast path needs the disc inside the 11 x 11 box and a scratch list for the uncertified maps
  const bool window_ok = scratch != nullptr && disc_fits_box(g);
  int* slow_count = scratch;
  int* slow_list = scratch ? scratch + 1 : nullptr;
  if (window_ok && (parts & 1)) {
    if (!counter_zeroed) {
      ProfRange pr(PROF_MISC, st);
      zero_int_kernel<<<1, 1, 0, st>>>(slow_count);
      DTK_LAUNCHED();
    }
    if (tkeys != nullptr) {
      static PerDev<int> per_sm_dev;
      int& per_sm_tm = per_sm_dev.get();
      if (per_sm_tm == 0) {
        DTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_tm, head_tm_kernel, TMK_THREADS, 0));
        if (per_sm_tm < 1) per_sm_tm = 1;
      }
      int grid = n_maps < sms * per_sm_tm ? n_maps : sms * per_sm_tm;
      ProfRange pr(PROF_HEAD, st);
      head_tm_kernel<<<grid, TMK_THREADS, 0, st>>>(maps, tkeys, cdiv(hp.P, CORR_TILE), n_maps, hp, hw, out_index, out, aux,
                                                   slow_list, slow_count);
      DTK_LAUNCHED();
    } else {
      size_t smem = (size_t)(lin_elems + WM * WM + 3 + 16 * WH * WH + 32) * sizeof(float) + 4 * sizeof(unsigned long long);
      static PerDev<size_t> attr_w_dev;
      size_t& attr_w = attr_w_dev.get();
      if (smem > attr_w) {
        DTK_CUDA(cudaFuncSetAttribute(head_window_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        attr_w = smem;
      }
      int per_sm = (int)((220 * 1024) / (smem + 1024));
      if (per_sm < 1) per_sm = 1;
      if (per_sm > 8) per_sm = 8;
      int grid = n_maps < sms * per_sm ? n_maps : sms * per_sm;
      ProfRange pr(PROF_HEAD, st);
      head_window_kernel<<<grid, WIN_THREADS, smem, st>>>(maps, n_maps, hp, hw, out_index, out, aux, slow_list, slow_count);
      DTK_LAUNCHED();
    }
  }
  if (!(parts & 2)) return DINOTRK_OK;
  // full-map kernel: every map (no scratch) or only the maps the window kernel could not certify
  if (g.w > HEAD_MAX_W || g.h > HEAD_MAX_H) {
    const int box_r = std::min(g.radius / g.stride, std::max(g.h, g.w));   // the disc lies in the box around the arg-max
    const int box_s = 2 * box_r + 1;
    const size_t smem = (size_t)(lin_elems + ((box_s * box_s + 3) & ~3) + 6 * HB_WARPS) * sizeof(float) +
                        HB_WARPS * sizeof(unsigned long long);
    DTK_CHECK_ARG(smem <= 227 * 1024, "head: disc radius %d px at stride %d does not fit the full-map kernel", g.radius, g.stride);
    static PerDev<size_t> attr_big_dev;
    static PerDev<int> per_sm_big_dev;   // occupancy at the smem of attr_big_dev
    size_t& attr_big = attr_big_dev.get();
    int& per_sm_big = per_sm_big_dev.get();
    if (smem != attr_big) {
      DTK_CUDA(cudaFuncSetAttribute(head_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
      DTK_CUDA(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm_big, head_big_kernel, HB_THREADS, smem));
      if (per_sm_big < 1) per_sm_big = 1;
      attr_big = smem;
    }
    const int grid = n_maps < sms * per_sm_big ? n_maps : sms * per_sm_big;
    ProfRange pr(PROF_HEAD_FULL, st);
    head_big_kernel<<<grid, HB_THREADS, smem, st>>>(maps, n_maps, window_ok ? slow_list : nullptr, window_ok ? slow_count : nullptr,
                                                   hp, hw, box_r, out_index, out, aux);
    DTK_LAUNCHED();
    return DINOTRK_OK;
  }
  const int nwarps = cdiv(g.h, 4);
  const int threads = nwarps * 32;
  size_t smem = (size_t)(2 * lin_elems + 2 * nwarps * 2 * 128 + 6 * 32) * sizeof(float) + 32 * sizeof(unsigned long long);
  static PerDev<size_t[4]> attr_smem_dev;
  size_t (&attr_smem)[4] = attr_smem_dev.get();
  const bool wrap = g.w <= 124;                 // tile 31 of every band lies outside the map
  const int variant = (threads <= 576 ? 0 : 2) + (wrap ? 0 : 1);  // <= 576 threads: 112 registers/thread; else 64
  auto kern = variant == 0 ? head_kernel<576, true> : variant == 1 ? head_kernel<576, false>
            : variant == 2 ? head_kernel<1024, true> : head_kernel<1024, false>;
  if (smem > attr_smem[variant]) {
    DTK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    attr_smem[variant] = smem;
  }
  int grid = n_maps < sms ? n_maps : sms;
  ProfRange pr(PROF_HEAD_FULL, st);
  kern<<<grid, threads, smem, st>>>(maps, n_maps, window_ok ? slow_list : nullptr, window_ok ? slow_count : nullptr, hp,
                                    hw, out_index, out, aux);
  DTK_LAUNCHED();
  return DINOTRK_OK;
}

}  // namespace dtk

using namespace dtk;

extern "C" int dinotrk_head(const float* maps, int n_maps, const dinotrk_geom* g, const dinotrk_head_weights* hw,
                            const int* out_index, float* out, int out_stride, int out_mode, int* aux, int* scratch,
                            void* stream) {
  DTK_CHECK_ARG(maps && g && hw && out, "head: null pointer");
  DTK_CHECK_ARG(out_stride >= 2 && (out_mode == 0 || out_mode == 1), "head: bad out_stride/out_mode");
  return launch_head(maps, n_maps, dinotrk_map_stride(g), *g, *hw, out_index, out, out_stride, out_mode, aux, scratch,
                     (cudaStream_t)stream);
}

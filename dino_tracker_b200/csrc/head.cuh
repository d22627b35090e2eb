// The tracker head's per-map rules, written once for every kernel that evaluates them: the full-map and window heads
// (head.cu), the exact-window head (xwin.cu) and the training step's reverse pass (train.cu).  The exact-window path is
// right only because its certificate and its output are the full-map head's, so they live here and nowhere else.
#pragma once
#include "common.cuh"

namespace dtk {

// Windows around the arg-max (side lengths): the box holding the disc, the hidden window its logits read and the input
// window that hidden window reads.
constexpr int HEAD_BOX_R = 5;   // box half-width in tokens
constexpr int WB = 2 * HEAD_BOX_R + 1, WH = WB + 2, WM = WB + 4;

struct HeadParams {
  int h, w, P, map_stride;
  int stride_px, half_patch, radius2;  // pixel geometry: centre = half_patch + stride * index
  float normW, normH;                  // W - 1, H - 1
  int out_stride, out_mode;
  float P1[16], P2[16];                // sums of the positive parts of the normalised 3x3 kernels (logit bound)
};

inline HeadParams make_head_params(const dinotrk_geom& g, const dinotrk_head_weights& hw, int map_stride, int out_stride,
                                   int out_mode) {
  HeadParams hp;
  hp.h = g.h; hp.w = g.w; hp.P = g.h * g.w; hp.map_stride = map_stride;
  hp.stride_px = g.stride; hp.half_patch = g.patch / 2; hp.radius2 = g.radius * g.radius;
  hp.normW = (float)(g.W - 1); hp.normH = (float)(g.H - 1);
  hp.out_stride = out_stride; hp.out_mode = out_mode;
  for (int o = 0; o < 16; ++o) {
    float p1 = 0.f, p2 = 0.f;
    for (int k = 0; k < 9; ++k) { p1 += hw.w1[o][k] > 0.f ? hw.w1[o][k] : 0.f; p2 += hw.w2[o][k] > 0.f ? hw.w2[o][k] : 0.f; }
    hp.P1[o] = p1 * (1.f + 1e-6f); hp.P2[o] = p2 * (1.f + 1e-6f);   // rounded up: the bound must stay a bound
  }
  return hp;
}

// The disc lies inside the box around the arg-max, so the window heads and the reverse pass need nothing outside it.
inline bool disc_fits_box(const dinotrk_geom& g) { return g.radius <= HEAD_BOX_R * g.stride; }

// pixel coordinate of the centre of token row / column i
__device__ __forceinline__ float token_px(const HeadParams& hp, int i) { return (float)(hp.half_patch + i * hp.stride_px); }

// token (r, c) lies in the disc: |token centre - arg-max centre| <= radius px
__device__ __forceinline__ bool in_disc(const HeadParams& hp, int r, int c, int arow, int acol) {
  const int dr = (r - arow) * hp.stride_px, dc = (c - acol) * hp.stride_px;
  return dr * dr + dc * dc <= hp.radius2;
}

// Certificate of a window head from its box sums tot = {sum e, disc sum e, disc sum x e, disc sum y e, box tokens},
// e = exp(z - zmax), and m_out >= every map value outside the 7 x 7 core.  Every logit outside the box is at most
// b2 + sum_o P2_o * relu(b1_o + P1_o * mout) (all terms monotone in m >= 0).  Certified: the disc mass is >= 2e-8 of (an
// upper bound of) the whole softmax, so the reference does not take the stability branch and its result is
// sum(x e) / sum(e) over the disc (the normaliser cancels).
__device__ __forceinline__ bool head_certified(const HeadParams& hp, const dinotrk_head_weights& wts, float mout, float zmax,
                                               const float (&tot)[5]) {
  float F = wts.b2;
#pragma unroll
  for (int o = 0; o < 16; ++o) F = fmaf(hp.P2[o], fmaxf(fmaf(hp.P1[o], mout, wts.b1[o]), 0.f), F);
  const float rest = ((float)hp.P - tot[4]) * expf(fminf(F - zmax, 80.f));
  return tot[1] >= 2e-8f * (tot[0] + rest) && tot[1] > 0.f && isfinite(rest);
}

// Stores the point (px, py) of map `map` at out[out_index[map] * out_stride]: RangeNormalizer((W, H)) dst=(-1,1)
// x / (W-1); * 2; + (-1) (data/dataset.py:33-35), and for out_mode 0 back through unnormalize(src=(-1,1)):
// (v - (-1)) / 2 * (W-1) (data/dataset.py:50-52).
__device__ __forceinline__ void head_store_point(const HeadParams& hp, float px, float py, const int* __restrict__ out_index,
                                                 float* __restrict__ out, int map) {
  float nx = __fadd_rn(__fmul_rn(2.f, __fdiv_rn(px, hp.normW)), -1.f);
  float ny = __fadd_rn(__fmul_rn(2.f, __fdiv_rn(py, hp.normH)), -1.f);
  if (hp.out_mode == 0) {
    nx = __fmul_rn(__fdiv_rn(__fadd_rn(nx, 1.f), 2.f), hp.normW);
    ny = __fmul_rn(__fdiv_rn(__fadd_rn(ny, 1.f), 2.f), hp.normH);
  }
  const size_t oi = (size_t)(out_index ? out_index[map] : map) * hp.out_stride;
  out[oi] = nx; out[oi + 1] = ny;
}

// Finish of a full-map head from the disc sums t = {sum e, sum x e, sum y e, sum x, sum y, disc tokens} and ssum = the sum
// of e over the whole map: p_i = e_i / ssum, the stability fallback when the disc mass is below 1e-8, the point, and
// aux = (arg-max, fallback taken).
__device__ __forceinline__ void head_full_finish(const HeadParams& hp, const float (&t)[6], float ssum, int map, int amax,
                                                 const int* __restrict__ out_index, float* __restrict__ out, int* __restrict__ aux) {
  // p_i = e_i / S_all; s = sum p_i over the disc   (softmax then mask, tracker_head.py:84-86)
  float sp = __fdiv_rn(t[0], ssum), spx = __fdiv_rn(t[1], ssum), spy = __fdiv_rn(t[2], ssum);
  const bool fallback = sp < 1e-8f;
  if (fallback) {  // heatmap <- (heatmap + 1/|mask|) * mask  (tracker_head.py:87-94)
    float u = __fdiv_rn(1.f, t[5]);
    sp = fmaf(t[5], u, sp); spx = fmaf(t[3], u, spx); spy = fmaf(t[4], u, spy);
  }
  head_store_point(hp, __fdiv_rn(spx, sp), __fdiv_rn(spy, sp), out_index, out, map);
  if (aux) { aux[2 * map] = amax; aux[2 * map + 1] = fallback ? 1 : 0; }
}

}  // namespace dtk

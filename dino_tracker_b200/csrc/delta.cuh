// Delta-DINO pieces shared by the inference stack (delta.cu) and the training node (delta_train.cu).
#pragma once
#include <cuda_fp16.h>

#include "common.cuh"

namespace dtk {

struct ConvShape {
  int B, H, W, Cin, Cout, dil;  // Cin is the padded (multiple of 4) channel count of the NHWC input
  int relu;
};

// reflect padding of one coordinate (pad < n)
__device__ __forceinline__ int reflect(int v, int n) {
  v = v < 0 ? -v : v;
  return v >= n ? 2 * (n - 1) - v : v;
}

constexpr size_t CONV_TC_ROWS = 32768;   // im2col rows per GEMM pass (bounds the fp16 scratch)

// largest K (25 * C_in_pad, rounded up to 8) over the four convolutions: the fp16 im2col scratch holds
// CONV_TC_ROWS rows of it per half
size_t delta_conv_kmax(const int* channels);

// one conv layer on tensor cores (explicit im2col with the fp16 hi/lo split + F16X3 wgmma GEMM), NHWC fp32 in / out;
// launches are timed under profile class `prof`
int launch_conv_tc(const float* in, const __half* w_hi, const __half* w_lo, const float* bias, float* out, ConvShape cs,
                   int Kp, __half* col_hi, __half* col_lo, int* plan, cudaStream_t st, int prof = PROF_CONV);

// RGB frames [B][3][H][W] -> NHWC with a zero 4th channel
int launch_rgb_to_nhwc4(const float* frames, float* out, int B, int HW, cudaStream_t st);

}  // namespace dtk

// CaffeNet's cross-channel local response norm (models/alexnet.lua's norm1 / norm2: local_size 5, alpha 1e-4, beta 0.75,
// k 1), in one fixed fp32 arithmetic so that a restatement can pin the device bit for bit:
//   q_j = x_j * x_j
//   S_c = q_j for j = c - 2 .. c + 2 inside [0, C), added in ascending j, starting from the first term (no sliding window)
//   s   = 1 + a * S_c               a = (float)(1e-4 / 5): a multiply, then an add
//   d   = sqrt(s) * sqrt(sqrt(s))   s^0.75; sqrt is correctly rounded on the host and the device
//   y   = x_c / d
// Every step is one rounded fp32 operation: *_rn intrinsics on the device, and the host build (tests through
// csrc/lrn_host.cpp) is compiled with -ffp-contract=off. Torch's and cudnn's LRN compute pow(scale, -beta) instead (as
// recalled, parity unpinned), a few ulp away.
//
// __host__ __device__ so that the CPU suite runs the very arithmetic lrn_split_kernel (elementwise.cu) runs.
#pragma once
#include <math.h>

#if defined(__CUDACC__)
#define MPN_LRN_HD __host__ __device__ __forceinline__
#else
#define MPN_LRN_HD inline
#endif

namespace mpn_lrn {

constexpr int kSize = 5, kHalf = 2;
constexpr float kAlphaOverSize = (float)(1e-4 / 5);

MPN_LRN_HD float mul(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fmul_rn(a, b);
#else
  return a * b;
#endif
}
MPN_LRN_HD float add(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fadd_rn(a, b);
#else
  return a + b;
#endif
}
MPN_LRN_HD float div(float a, float b) {
#if defined(__CUDA_ARCH__)
  return __fdiv_rn(a, b);
#else
  return a / b;
#endif
}
MPN_LRN_HD float sqrt_rn(float a) {
#if defined(__CUDA_ARCH__)
  return __fsqrt_rn(a);
#else
  return sqrtf(a);
#endif
}

// y_c of channel c of a C-channel pixel; x(j) returns channel j's input (only j in [c - 2, c + 2] inside [0, C) is read).
// S starts at 0: 0 + q_j is q_j exactly (q_j >= 0), so this is the sum from the first term. The fixed trip count lets
// the kernel index its registers with constants.
template <class X>
MPN_LRN_HD float lrn_channel(const X &x, int c, int C) {
  float S = 0.0f;
#pragma unroll
  for (int d = -kHalf; d <= kHalf; ++d) {
    const int j = c + d;
    if (j < 0 || j >= C) continue;
    const float xj = x(j);
    S = add(S, mul(xj, xj));
  }
  const float s = add(1.0f, mul(kAlphaOverSize, S));
  const float r = sqrt_rn(s);
  return div(x(c), mul(r, sqrt_rn(r)));
}

}  // namespace mpn_lrn

// Host build of the LRN arithmetic (csrc/lrn_rule.cuh), for the CPU suite: the very function lrn_split_kernel runs per
// channel, compiled with -ffp-contract=off (the device side uses *_rn intrinsics). Not linked into libmpn_b200.so.
#include <stdint.h>
#include "lrn_rule.cuh"

// x: pixels x ld fp32, the first C channels the layer's input; y: pixels x C
extern "C" void hd_lrn(const float *x, int64_t pixels, int C, int64_t ld, float *y) {
  for (int64_t p = 0; p < pixels; ++p) {
    const float *xp = x + p * ld;
    auto at = [xp](int j) { return xp[j]; };
    for (int c = 0; c < C; ++c) y[p * C + c] = mpn_lrn::lrn_channel(at, c, C);
  }
}

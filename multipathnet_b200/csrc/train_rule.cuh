// train_rule.cuh — the element rules of the per-ROI training step (train.cu), compiled for the device and, through the
// host-only views mpn_debug_dropout / mpn_debug_criteria / mpn_debug_sgd, for the host, where the CPU suite restates them.
#pragma once
#include <stdint.h>
#include <math.h>
#if defined(__CUDACC__)
#define MPN_HD __host__ __device__ __forceinline__
#else
#define MPN_HD inline
#endif

// ---- nn.Dropout (v2, train mode): out = in * keep / (1 - p). The keep bits come from Philox4x32-10 (Salmon et al.,
// SC'11; the Random123 round function and key schedule) with key = (seed lo, seed hi) and counter =
// (element / 4, step, tower << 16 | layer, 0): word element % 4 of the output, u = word >> 8, keep iff u >= floor(p * 2^24).
// `layer` is the index of the Linear within its tower's layer list. It does not try to match Torch's generator.
MPN_HD void mpn_philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1, uint32_t out[4]) {
  for (int i = 0; i < 10; ++i) {
    if (i > 0) { k0 += 0x9E3779B9u; k1 += 0xBB67AE85u; }
    const uint64_t p0 = (uint64_t)0xD2511F53u * c0, p1 = (uint64_t)0xCD9E8D57u * c2;
    const uint32_t hi0 = (uint32_t)(p0 >> 32), lo0 = (uint32_t)p0, hi1 = (uint32_t)(p1 >> 32), lo1 = (uint32_t)p1;
    c0 = hi1 ^ c1 ^ k0; c1 = lo1; c2 = hi0 ^ c3 ^ k1; c3 = lo0;
  }
  out[0] = c0; out[1] = c1; out[2] = c2; out[3] = c3;
}
MPN_HD uint32_t mpn_dropout_threshold(float p) { return (uint32_t)((double)p * 16777216.0); }
MPN_HD int mpn_dropout_keep(uint64_t seed, uint32_t step, int tower, int layer, uint64_t elem, uint32_t thr) {
  uint32_t o[4];
  const uint64_t q = elem >> 2;
  mpn_philox4x32_10((uint32_t)q, (uint32_t)(q >> 32), step, ((uint32_t)tower << 16) | (uint32_t)layer, (uint32_t)seed,
                    (uint32_t)(seed >> 32), o);
  return (o[elem & 3] >> 8) >= thr;
}

// ---- nn.ParallelCriterion{CrossEntropy, BBoxRegression x w} for one row r of R (BBoxRegressionCriterion.lua:11-41).
// x: C logits, d: 4C raw deltas, t: 4C targets, label in 1..C (1 = background). Returns the row's cross entropy and its
// SmoothL1 sum (both un-normalised); writes d loss / d x (divided by R) and w * d bbox / d d (divided by R). The SmoothL1
// gradient is taken on the masked buffer and is not masked again, as the reference does.
MPN_HD void mpn_criteria_row(const float *x, const float *d, const float *t, int label, int C, double inv_R, double bbox_w,
                             float *gx, float *gd, double *ce, double *sl1) {
  const int lab = label - 1;
  double m = x[0];
  for (int j = 1; j < C; ++j) m = x[j] > m ? (double)x[j] : m;
  double s = 0.0;
  for (int j = 0; j < C; ++j) s += exp((double)x[j] - m);
  *ce = m + log(s) - (double)x[lab];
  for (int j = 0; j < C; ++j) gx[j] = (float)((exp((double)x[j] - m) / s - (j == lab ? 1.0 : 0.0)) * inv_R);
  double acc = 0.0;
  for (int j = 0; j < 4 * C; ++j) {
    const double in = (lab > 0 && j / 4 == lab) ? (double)d[j] : 0.0;
    const double diff = in - (double)t[j], ad = fabs(diff);
    acc += ad < 1.0 ? 0.5 * diff * diff : ad - 0.5;
    const double g = diff < -1.0 ? -1.0 : (diff > 1.0 ? 1.0 : diff);
    gd[j] = (float)(g * inv_R * bbox_w);
  }
  *sl1 = acc;
}

// ---- optim.sgd for one element (as recalled: the package is not in the reference tree). Weight decay is added to the
// gradient first (0 for biases, Optim.lua:50-51); the first step copies the gradient into the momentum buffer, later
// steps take buf = m * buf + (1 - dampening) * g; then w -= lr * buf. momentum 0 skips the buffer. Every multiply-add is
// one explicit fma, so the host view and the device round alike.
MPN_HD void mpn_sgd_elem(float &w, float g, float &buf, float lr, float momentum, float dampening, float wd, int first) {
  float gg = wd != 0.f ? fmaf(wd, w, g) : g;
  if (momentum != 0.f) {
    buf = first ? gg : fmaf(momentum, buf, (1.f - dampening) * gg);
    gg = buf;
  }
  w = fmaf(-lr, gg, w);
}

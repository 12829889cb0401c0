// train_rule.cuh — the element rules of the per-ROI training step (train.cu), compiled for the device and, through the
// host-only views mpn_debug_dropout / mpn_debug_criteria / mpn_debug_sgd / mpn_debug_optim, for the host, where the CPU
// suite restates them.
#pragma once
#include <stdint.h>
#include <math.h>
#include "../../include/mpn_abi.h"   // mpn_train_optim, MPN_OPTIM_*
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

// ---- train.lua's other optim methods for one element (mpn_train_optim; as recalled like optim.sgd, parity unpinned).
// Each Torch tensor call is one fp32 rounding and a scalar * tensor + tensor is one fmaf. g is the gradient with weight
// decay added first, gg = wd != 0 ? fmaf(wd, w, g) : g (wd 0 for biases); then, with b1 = beta1, c1 = 1 - beta1, ...:
//   adam     m = fmaf(c1, gg, b1 * m); v = fmaf(c2, gg * gg, b2 * v); q = m / (sqrtf(v) + eps)
//   adamax   m = fmaf(c1, gg, b1 * m); u = fmaxf(b2 * u, fabsf(gg) + eps); q = m / u     (eps 1e-38 is subnormal: the
//            code is compiled without flushing, so g = u = 0 gives u = 1e-38 exactly and q = 0)
//   adagrad  s = fmaf(gg, gg, s); q = gg / (sqrtf(s) + 1e-10f)
//   rmsprop  m = fmaf(c2, gg * gg, b2 * m) with b2 = alpha, c2 = 1 - alpha; q = gg / (sqrtf(m) + eps)
// and w = fmaf(-lr, q, w), lr the method's step factor of mpn_optim_scalars. The no-gradient variant (an idle class head)
// is the same rule with g = 0: under adam such a head keeps moving. sgd keeps mpn_sgd_elem with lr = clr.
struct mpn_optim_step {
  float lr;              // sgd, adagrad: clr; adam: s = clr * sqrt(1 - b2^T) / (1 - b1^T); adamax: lr / (1 - b1^T); rmsprop: lr
  float b1, c1, b2, c2;  // beta1, 1 - beta1, beta2, 1 - beta2 (rmsprop: alpha, 1 - alpha in b2, c2)
  float eps, wd;
};

// the per-step scalars, computed in double as Lua does, from the fp32 rate in force, and rounded once to fp32. t: the
// steps done before this one, the same for every tensor (Optim.lua steps every module every step); T = t + 1;
// clr = lr / (1 + t * lrd). adamax and rmsprop ignore lr_decay, as optim does.
inline mpn_optim_step mpn_optim_scalars(const mpn_train_optim &o, float lr, float wd, int64_t t) {
  mpn_optim_step h = {};
  const double T = (double)t + 1.0, clr = (double)lr / (1.0 + (double)t * o.lr_decay);
  h.lr = (float)clr; h.wd = wd;
  h.b1 = (float)o.beta1; h.c1 = (float)(1.0 - o.beta1); h.b2 = (float)o.beta2; h.c2 = (float)(1.0 - o.beta2); h.eps = (float)o.epsilon;
  if (o.method == MPN_OPTIM_ADAM) h.lr = (float)(clr * sqrt(1.0 - pow(o.beta2, T)) / (1.0 - pow(o.beta1, T)));
  else if (o.method == MPN_OPTIM_ADAMAX) h.lr = (float)((double)lr / (1.0 - pow(o.beta1, T)));
  else if (o.method == MPN_OPTIM_ADAGRAD) h.eps = 1e-10f;
  else if (o.method == MPN_OPTIM_RMSPROP) { h.lr = lr; h.b2 = (float)o.alpha; h.c2 = (float)(1.0 - o.alpha); }
  return h;
}

// the state update and the step direction q of one element (w -= lr * q), g with weight decay included
template <int M>
MPN_HD float mpn_optim_dir(float g, float &s1, float &s2, const mpn_optim_step &h) {
  if (M == MPN_OPTIM_ADAM) {
    s1 = fmaf(h.c1, g, h.b1 * s1);
    s2 = fmaf(h.c2, g * g, h.b2 * s2);
    return s1 / (sqrtf(s2) + h.eps);
  }
  if (M == MPN_OPTIM_ADAMAX) {
    s1 = fmaf(h.c1, g, h.b1 * s1);
    s2 = fmaxf(h.b2 * s2, fabsf(g) + h.eps);
    return s1 / s2;
  }
  if (M == MPN_OPTIM_ADAGRAD) s1 = fmaf(g, g, s1);
  else s1 = fmaf(h.c2, g * g, h.b2 * s1);
  return g / (sqrtf(s1) + h.eps);
}

template <int M>
MPN_HD void mpn_optim_elem(float &w, float g, float &s1, float &s2, const mpn_optim_step &h) {
  const float gg = h.wd != 0.f ? fmaf(h.wd, w, g) : g;
  w = fmaf(-h.lr, mpn_optim_dir<M>(gg, s1, s2, h), w);
}

// a fixed-batch-norm weight (mpn_train_spec.n_fixed) under the methods other than sgd: the state lives in the space of
// the reference's W. The device keeps W' = fl(a W) and g' = dL/dW'; the rule takes gW = a * g' and, for the weight
// decay term, W = W' / a (one rounding each), forms the step d = lr * q in W space and applies W' = fmaf(-a, d, W'):
// exact in real arithmetic. a != 0 (mpn_model_train_begin refuses a zero scale), of either sign.
template <int M>
MPN_HD void mpn_optim_elem_fixed(float &w, float g, float a, float &s1, float &s2, const mpn_optim_step &h) {
  const float gw = a * g;
  const float gg = h.wd != 0.f ? fmaf(h.wd, w / a, gw) : gw;
  const float d = h.lr * mpn_optim_dir<M>(gg, s1, s2, h);
  w = fmaf(-a, d, w);
}

// host-only: the checks of an mpn_train_optim (mpn_train_check_optim); null: valid
inline const char *mpn_optim_refusal(const mpn_train_optim &o) {
  if (o.method < MPN_OPTIM_SGD || o.method > MPN_OPTIM_RMSPROP) return "optim: method out of range (0 sgd, 1 adam, 2 adamax, 3 adagrad, 4 rmsprop)";
  if (!(o.beta1 >= 0.0 && o.beta1 < 1.0) || !(o.beta2 >= 0.0 && o.beta2 < 1.0)) return "optim: beta1 and beta2 must lie in [0, 1)";
  if (!(o.alpha >= 0.0 && o.alpha <= 1.0)) return "optim: alpha must lie in [0, 1]";
  if (!(o.epsilon >= 0.0) || !isfinite(o.epsilon)) return "optim: epsilon must be finite and >= 0";
  if (!(o.lr_decay >= 0.0) || !isfinite(o.lr_decay)) return "optim: lr_decay must be finite and >= 0";
  return nullptr;
}

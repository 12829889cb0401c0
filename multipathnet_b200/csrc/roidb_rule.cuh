// roidb_rule.cuh — the per-row rules of the training feed (roidb.cu): DataSetJSON's ground truth and attachProposals,
// BatchProviderROI's draws, boxes and regression targets. Compiled for the device and, through the host-only views
// mpn_debug_attach_proposals / mpn_sample_plan / mpn_train_images_size / mpn_debug_sample_rows, for the host, where
// the CPU suite restates them (tests/_batch_provider_ref.py).
//
// Torch tensor arithmetic on FloatTensors is fp32, one rounding per operation, never fused (roidb.cu is compiled with
// -fmad=false and the fp32 steps below use explicit *_rn intrinsics on the device); Lua numbers are doubles. A Lua number
// that meets a FloatTensor operation (`t + x`, `t:ge(x)`) is rounded to fp32 first.
#pragma once
#include <stdint.h>
#include <math.h>
#include "image_scale.cuh"    // mpn_img::fadd / fsub / fmul / fdiv
#include "train_rule.cuh"     // mpn_philox4x32_10

namespace mpn_feed {
using mpn_img::fadd;
using mpn_img::fdiv;
using mpn_img::fmul;
using mpn_img::fsub;

// ---- DataSetJSON:getAnnotation (DataSetJSON.lua:101-112): bbox:clone():float(), then x2 = w + x + 1, y2 = h + y + 1 in fp32
MPN_HD void gt_box(const double xywh[4], float out[4]) {
  const float x = (float)xywh[0], y = (float)xywh[1], w = (float)xywh[2], h = (float)xywh[3];
  out[0] = x; out[1] = y;
  out[2] = fadd(fadd(w, x), 1.f);
  out[3] = fadd(fadd(h, y), 1.f);
}

// ---- utils.boxoverlap (utils.lua:104-128) of box a with one GT box b: clamps, +1 widths and the products in fp32; barea in
// double (Lua numbers), rounded once when it is added to the fp32 aarea; 0 where w < 0 or h < 0
MPN_HD float boxoverlap(const float a[4], const float b[4]) {
  const float x1 = a[0] < b[0] ? b[0] : a[0], y1 = a[1] < b[1] ? b[1] : a[1];
  const float x2 = a[2] > b[2] ? b[2] : a[2], y2 = a[3] > b[3] ? b[3] : a[3];
  const float w = fadd(fsub(x2, x1), 1.f), h = fadd(fsub(y2, y1), 1.f);
  const float inter = fmul(w, h);
  const float aarea = fmul(fadd(fsub(a[2], a[0]), 1.f), fadd(fsub(a[3], a[1]), 1.f));
  const double barea = ((double)b[2] - (double)b[0] + 1.0) * ((double)b[3] - (double)b[1] + 1.0);
  const float o = fdiv(inter, fsub(fadd(aarea, (float)barea), inter));
  return (w < 0.f || h < 0.f) ? 0.f : o;
}

// ---- utils.intersection (utils.lua:131-148): inter / area of a. Negative widths are NOT zeroed: a box with both w < 0 and
// h < 0 against the crowd box gets a positive value
MPN_HD float intersection(const float a[4], const float b[4]) {
  const float x1 = a[0] < b[0] ? b[0] : a[0], y1 = a[1] < b[1] ? b[1] : a[1];
  const float x2 = a[2] > b[2] ? b[2] : a[2], y2 = a[3] > b[3] ? b[3] : a[3];
  const float inter = fmul(fadd(fsub(x2, x1), 1.f), fadd(fsub(y2, y1), 1.f));
  const float aarea = fmul(fadd(fsub(a[2], a[0]), 1.f), fadd(fsub(a[3], a[1]), 1.f));
  return fdiv(inter, aarea);
}

// ---- attachProposals (DataSetJSON.lua:280-390) for one row a of all_boxes (the G GT rows first, then the proposals):
// overlap = max IoU over the GT rows (the first maximum: torch.max), correspondance = its 1-based GT index, 0 where the
// overlap is 0, label = that GT's class id; then the crowd mask: overlap = -1 where some crowd's intersection is > 0.7
// (fp32), GT rows exempt. correspondance and label survive the mask.
MPN_HD void attach_row(const float a[4], int is_gt, const float *gt, const int32_t *gt_cls, int G, const float *crowd, int NC,
                       float *overlap, int32_t *corr, int32_t *label) {
  float best = 0.f;
  int bi = 0;
  for (int g = 0; g < G; ++g) {
    const float o = boxoverlap(a, gt + 4 * g);
    if (g == 0 || !(o <= best)) { best = o; bi = g + 1; if (o != o) break; }   // TH's max: first maximum, NaN wins
  }
  if (best == 0.f) bi = 0;
  *corr = bi;
  *label = bi > 0 ? gt_cls[bi - 1] : 0;
  if (!is_gt)
    for (int c = 0; c < NC; ++c)
      if (intersection(a, crowd + 4 * c) > 0.7f) { best = -1.f; break; }
  *overlap = best;
}

// ---- BatchProviderROI:setupOne (BatchProviderROI.lua:39-50): thresholds are Lua numbers rounded to fp32 by ge / lt
MPN_HD bool is_fg(float o, float fg) { return o >= fg; }
MPN_HD bool is_bg(float o, float lo, float hi) { return o >= lo && o < hi; }

// ---- utils.convertTo, 2-D branch (utils.lua:185-198): FloatTensor ops, log of an fp32 tensor = C log on the value, rounded
MPN_HD void convert_to_f32(const float b[4], const float t[4], float out[4]) {
  const float xc = fmul(fadd(b[0], b[2]), 0.5f), yc = fmul(fadd(b[1], b[3]), 0.5f);
  const float w = fsub(b[2], b[0]), h = fsub(b[3], b[1]);
  const float xtc = fmul(fadd(t[0], t[2]), 0.5f), ytc = fmul(fadd(t[1], t[3]), 0.5f);
  const float wt = fsub(t[2], t[0]), ht = fsub(t[3], t[1]);
  out[0] = fdiv(fsub(xtc, xc), w);
  out[1] = fdiv(fsub(ytc, yc), h);
  out[2] = (float)log((double)fdiv(wt, w));
  out[3] = (float)log((double)fdiv(ht, h));
}

// ---- utils.convertTo, 1-D branch (utils.lua:172-184): Lua numbers (double) and math.log, stored once into the fp32 row
MPN_HD void convert_to_f64(const float b[4], const float t[4], float out[4]) {
  const double xc = ((double)b[0] + (double)b[2]) * 0.5, yc = ((double)b[1] + (double)b[3]) * 0.5;
  const double w = (double)b[2] - (double)b[0], h = (double)b[3] - (double)b[1];
  const double xtc = ((double)t[0] + (double)t[2]) * 0.5, ytc = ((double)t[1] + (double)t[3]) * 0.5;
  const double wt = (double)t[2] - (double)t[0], ht = (double)t[3] - (double)t[1];
  out[0] = (float)((xtc - xc) / w);
  out[1] = (float)((ytc - yc) / h);
  out[2] = (float)log(wt / w);
  out[3] = (float)log(ht / h);
}

// ---- BatchProviderROI:sample (BatchProviderROI.lua:123-131): the label's block of a fg row, (t - mean) / std in fp32
MPN_HD void target_block(const float roi[4], const float gt[4], const float mean[4], const float std_[4], float out[4]) {
  float t[4];
  convert_to_f64(roi, gt, t);
  for (int k = 0; k < 4; ++k) out[k] = fdiv(fsub(t[k], mean[k]), std_[k]);
}

// ---- selectBBoxesOne's preprocess_bbox (BatchProviderBase.lua:85-92): (b - 1) * float(im_scale) + 1 in fp32; the flip
// against `width` (getImages' IntTensor im_sizes: the resized image's width) in double, rounded once
MPN_HD void train_box(const float b[4], float scale, int width, int flip, float out[4]) {
  float d[4];
  for (int k = 0; k < 4; ++k) d[k] = fadd(fmul(fsub(b[k], 1.f), scale), 1.f);
  if (flip) {
    const float t = d[0];
    d[0] = (float)((double)width - (double)d[2] + 1.0);
    d[2] = (float)((double)width - (double)t + 1.0);
  }
  for (int k = 0; k < 4; ++k) out[k] = d[k];
}

// ---- BatchProviderBase:getImages' size rule (BatchProviderBase.lua:23-41, jitter 0): im_scale = scale / min side,
// im_s = size * im_scale; per dim in order, im_s and im_scale are divided by im_s[dim] / max_size where im_s[dim] > max_size;
// image.scale receives im_s and allocates trunc(im_s)
MPN_HD void train_size(int H0, int W0, double scale, double max_size, int *h, int *w, double *im_scale) {
  double s = scale / (double)(H0 < W0 ? H0 : W0);
  double im_s[2] = {(double)H0 * s, (double)W0 * s};
  for (int dim = 0; dim < 2; ++dim)
    if (im_s[dim] > max_size) {
      const double rat = im_s[dim] / max_size;
      im_s[0] = im_s[0] / rat; im_s[1] = im_s[1] / rat;
      s = s / rat;
    }
  *h = (int)(long)im_s[0];
  *w = (int)(long)im_s[1];
  *im_scale = s;
}

// ---- draws: Philox4x32-10 (train_rule.cuh) with key (seed lo, seed hi) and counter (draw, step, slot, set << 8 | purpose),
// word 0; torch.random(n) is restated as 1 + floor(u * n / 2^32). Dropout's counters have word 3 = 0, these never do.
// DRAW_INTEGRAL: the threshold set (= class head) of an integral model's step, drawn at slot 0, set 0, draw 0
// (train.lua's `loaders[torch.random(#loaders)]`).
enum { DRAW_IMAGE = 1, DRAW_FLIP = 2, DRAW_BG = 3, DRAW_FG = 4, DRAW_INTEGRAL = 5 };
MPN_HD uint32_t draw_u32(uint64_t seed, uint32_t step, int slot, int set, int purpose, uint32_t draw) {
  uint32_t o[4];
  mpn_philox4x32_10(draw, step, (uint32_t)slot, ((uint32_t)set << 8) | (uint32_t)purpose, (uint32_t)seed, (uint32_t)(seed >> 32), o);
  return o[0];
}
MPN_HD int64_t rand_int(uint32_t u, int64_t n) { return 1 + (int64_t)(((uint64_t)u * (uint64_t)n) >> 32); }

}  // namespace mpn_feed

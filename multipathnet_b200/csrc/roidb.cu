// roidb.cu — the training feed on the device: DataSetJSON:attachProposals once per image at construction, setupData's
// regression statistics, and BatchProviderROI:sample's ROIs, labels and targets per step. The per-row rules live in
// roidb_rule.cuh (shared with the host views at the end of this file).
//
//   roidb_match_kernel    one CTA per image: overlap / correspondance / label per row, then the fg / bg counts of every
//                         threshold set (warp ballots, no atomics)
//   scan_exclusive        coco_eval.cu's one-CTA scan over all (set, kind, image) counts: each list's start in one buffer
//   roidb_compact_kernel  one CTA per image: the fg / bg row lists of every set in row order (ballot + CTA prefix)
//   roidb_stats_rows / roidb_stats_reduce   setupData: convertTo's 2-D branch per fg row, then a fixed-order double
//                         reduction per coordinate (one CTA each, strided partial sums, tree)
//   roidb_sample_kernel   one warp per output row of a step
#include "common.cuh"
#include "roidb_rule.cuh"
#include <algorithm>
#include <cmath>

int mpn_scan_exclusive_launch(mpn_ctx *ctx, int *a, int m);                 // coco_eval.cu
int mpn_get_images_u8_flip_launch(mpn_ctx *, const uint8_t *, int32_t, int32_t, const mpn_image_transform *, int32_t, int32_t,
                                  int32_t, float *);                          // preproc.cu
int mpn_model_n_cls_heads(const mpn_model *m);                                // model.cu

namespace {
constexpr int kMT = 256;                 // threads per image in the match / compact kernels
constexpr int kMaxSets = 16;
constexpr int kMaxSlots = 32;

template <class T>
struct DBuf {
  T *p = nullptr;
  size_t n = 0;
  int alloc(mpn_ctx *ctx, size_t count) {
    if (count <= n) return MPN_OK;
    if (p) { cudaFree(p); p = nullptr; n = 0; }
    MPN_CUDA(ctx, cudaMalloc((void **)&p, sizeof(T) * std::max<size_t>(count, 1)));
    n = count;
    return MPN_OK;
  }
  void release() { if (p) cudaFree(p); p = nullptr; n = 0; }
};
struct Thresholds { float fg[kMaxSets], lo[kMaxSets], hi[kMaxSets]; int n; };
}  // namespace

struct mpn_roidb {
  mpn_ctx *ctx = nullptr;
  int32_t n_images = 0, n_sets = 0, num_classes = 0;
  std::vector<int64_t> row_off, gt_off, crowd_off;   // per image, n_images + 1 (host)
  std::vector<int32_t> n_gt;                          // GT rows per image
  std::vector<int32_t> list_off;                      // (n_sets * 2 * n_images + 1): list start of (set, kind 0 bg / 1 fg, image)
  Thresholds thr{};
  DBuf<float> boxes, overlap, gt_box, crowd_box;      // all_boxes (rows x 4), overlap per row, GT / crowd boxes
  DBuf<int32_t> corr, label, gt_cls, lists, offs;     // offs: list_off on the device (counts before the scan)
  DBuf<int64_t> row_off_dev, gt_off_dev, crowd_off_dev;
  DBuf<float> stats_tmp;
  DBuf<double> stats_out;
  // the last mpn_roidb_sample's batch
  std::vector<DBuf<uint8_t>> raw;
  std::vector<DBuf<float>> images;
  std::vector<int32_t> batch_hw, batch_rois;
  DBuf<float> b_boxes, b_targets, b_losses;
  DBuf<int32_t> b_labels;
  int64_t b_R = 0;
  int32_t b_C = 0, b_slots = 0, b_set = 0;            // b_set: the threshold set the batch was drawn from
};

// ------------------------------------------------------------------------------------------------------------- matching
__global__ void __launch_bounds__(kMT) roidb_match_kernel(const float *__restrict__ boxes, const int64_t *__restrict__ row_off,
                                                          const int64_t *__restrict__ gt_off, const float *__restrict__ gt_box,
                                                          const int32_t *__restrict__ gt_cls, const int64_t *__restrict__ crowd_off,
                                                          const float *__restrict__ crowd_box, int n_images, Thresholds thr,
                                                          float *__restrict__ overlap, int32_t *__restrict__ corr,
                                                          int32_t *__restrict__ label, int32_t *__restrict__ counts) {
  __shared__ int s_cnt[kMT / 32][2 * kMaxSets];
  const int img = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = row_off[img], n = row_off[img + 1] - r0;
  const int64_t g0 = gt_off[img], c0 = crowd_off[img];
  const int G = (int)(gt_off[img + 1] - g0), NC = (int)(crowd_off[img + 1] - c0);
  int cnt[2 * kMaxSets];
  for (int k = 0; k < 2 * kMaxSets; ++k) cnt[k] = 0;
  for (int64_t base = 0; base < n; base += kMT) {
    const int64_t i = base + threadIdx.x;
    float o = 0.f;
    const bool in = i < n;
    if (in) {
      const float4 b = reinterpret_cast<const float4 *>(boxes)[r0 + i];
      const float a[4] = {b.x, b.y, b.z, b.w};
      int32_t c, l;
      mpn_feed::attach_row(a, i < G, gt_box + 4 * g0, gt_cls + g0, G, crowd_box + 4 * c0, NC, &o, &c, &l);
      overlap[r0 + i] = o; corr[r0 + i] = c; label[r0 + i] = l;
    }
    for (int s = 0; s < thr.n; ++s) {                 // lane 0 of each warp keeps its warp's counts
      cnt[2 * s] += __popc(__ballot_sync(~0u, in && mpn_feed::is_bg(o, thr.lo[s], thr.hi[s])));
      cnt[2 * s + 1] += __popc(__ballot_sync(~0u, in && mpn_feed::is_fg(o, thr.fg[s])));
    }
  }
  if (lane == 0)
    for (int k = 0; k < 2 * thr.n; ++k) s_cnt[warp][k] = cnt[k];
  __syncthreads();
  if (threadIdx.x < 2 * thr.n) {
    int t = 0;
    for (int w = 0; w < kMT / 32; ++w) t += s_cnt[w][threadIdx.x];
    const int s = threadIdx.x >> 1, kind = threadIdx.x & 1;
    counts[((int64_t)s * 2 + kind) * n_images + img] = t;
  }
}

// the fg / bg lists of every set in row order: per chunk of kMT rows, a warp ballot gives each row its rank in its warp and
// the CTA adds the counts of the warps before it
__global__ void __launch_bounds__(kMT) roidb_compact_kernel(const float *__restrict__ overlap, const int64_t *__restrict__ row_off,
                                                            int n_images, Thresholds thr, const int32_t *__restrict__ list_off,
                                                            int32_t *__restrict__ lists) {
  __shared__ int s_w[kMT / 32];
  const int img = blockIdx.x, lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  const int64_t r0 = row_off[img], n = row_off[img + 1] - r0;
  for (int s = 0; s < thr.n; ++s)
    for (int kind = 0; kind < 2; ++kind) {
      int32_t *out = lists + list_off[((int64_t)s * 2 + kind) * n_images + img];
      int carry = 0;
      for (int64_t base = 0; base < n; base += kMT) {
        const int64_t i = base + threadIdx.x;
        bool p = false;
        if (i < n) {
          const float o = overlap[r0 + i];
          p = kind ? mpn_feed::is_fg(o, thr.fg[s]) : mpn_feed::is_bg(o, thr.lo[s], thr.hi[s]);
        }
        const unsigned m = __ballot_sync(~0u, p);
        if (lane == 0) s_w[warp] = __popc(m);
        __syncthreads();
        int before = carry, total = 0;
        for (int w = 0; w < kMT / 32; ++w) { if (w < warp) before += s_w[w]; total += s_w[w]; }
        if (p) out[before + __popc(m & ((1u << lane) - 1u))] = (int32_t)(r0 + i);
        carry += total;
        __syncthreads();
      }
    }
}

// ------------------------------------------------------------------------------------------------------------- setupData
// row j of the fg list range [a, a + n): convertTo(rois, gtboxes) (2-D branch) into tmp[4 * j .. 4 * j + 3]
__global__ void roidb_stats_rows_kernel(const int32_t *__restrict__ lists, int64_t a, int64_t n, const float *__restrict__ boxes,
                                        const int32_t *__restrict__ corr, const int64_t *__restrict__ row_off, int n_images,
                                        float *__restrict__ tmp) {
  const int64_t j = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= n) return;
  const int32_t row = lists[a + j];
  int lo = 0, hi = n_images - 1;                       // the image whose rows hold `row`
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (row_off[mid] <= row) lo = mid; else hi = mid - 1; }
  const float4 b = reinterpret_cast<const float4 *>(boxes)[row];
  const float4 g = reinterpret_cast<const float4 *>(boxes)[row_off[lo] + corr[row] - 1];
  const float bb[4] = {b.x, b.y, b.z, b.w}, gg[4] = {g.x, g.y, g.z, g.w};
  float o[4];
  mpn_feed::convert_to_f32(bb, gg, o);
  for (int k = 0; k < 4; ++k) tmp[4 * j + k] = o[k];
}

// one CTA per coordinate k: the mean, then the unbiased std from the sum of squared deviations; each thread sums the rows
// t, t + 1024, ... in order, then a fixed tree. out[k] = mean, out[4 + k] = std
__global__ void __launch_bounds__(1024) roidb_stats_reduce_kernel(const float *__restrict__ tmp, int64_t n, double *__restrict__ out) {
  __shared__ double sh[1024];
  const int k = blockIdx.x, t = threadIdx.x;
  double acc = 0.0;
  for (int64_t j = t; j < n; j += 1024) acc += (double)tmp[4 * j + k];
  sh[t] = acc;
  __syncthreads();
  for (int s = 512; s > 0; s >>= 1) { if (t < s) sh[t] += sh[t + s]; __syncthreads(); }
  const double mean = sh[0] / (double)n;
  __syncthreads();
  acc = 0.0;
  for (int64_t j = t; j < n; j += 1024) { const double d = (double)tmp[4 * j + k] - mean; acc += d * d; }
  sh[t] = acc;
  __syncthreads();
  for (int s = 512; s > 0; s >>= 1) { if (t < s) sh[t] += sh[t + s]; __syncthreads(); }
  if (t == 0) { out[k] = mean; out[4 + k] = sqrt(sh[0] / (double)(n - 1)); }
}

// ------------------------------------------------------------------------------------------------------------- sampling
struct SampleSlot {
  int32_t n_bg_src, n_fg_src;         // list sizes of the bg / fg source images (the draws' n)
  int32_t nb, nf;                     // draws: min(bg_each, n_bg_src), min(fg_each, n_fg_src)
  int32_t bg_list, fg_list;           // list starts
  int32_t fg_src, row0;               // fg source image; first output row of the slot
  int32_t width, flip;
  float scale;                        // float(im_scale)
};
struct SamplePlan {
  SampleSlot s[kMaxSlots];
  int32_t n_slots, set, C;
  uint32_t step;
  uint64_t seed;
  float mean[4], std_[4];
};

// one warp per output row: bg rows of slot k first, then its fg rows; every lane computes the row, lanes write the 4C targets
__global__ void __launch_bounds__(256) roidb_sample_kernel(SamplePlan P, int64_t R, const int32_t *__restrict__ lists,
                                                           const float *__restrict__ boxes, const int32_t *__restrict__ corr,
                                                           const int32_t *__restrict__ label, const int64_t *__restrict__ row_off,
                                                           float *__restrict__ out_boxes, int32_t *__restrict__ out_labels,
                                                           float *__restrict__ out_targets) {
  const int64_t r = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const int lane = threadIdx.x & 31;
  if (r >= R) return;
  int k = 0;
  while (k + 1 < P.n_slots && P.s[k + 1].row0 <= r) ++k;
  const SampleSlot &S = P.s[k];
  const int d = (int)(r - S.row0);
  const bool fg = d >= S.nb;
  const uint32_t u = mpn_feed::draw_u32(P.seed, P.step, k, P.set, fg ? mpn_feed::DRAW_FG : mpn_feed::DRAW_BG,
                                         (uint32_t)(fg ? d - S.nb : d));
  const int32_t pos = (int32_t)mpn_feed::rand_int(u, fg ? S.n_fg_src : S.n_bg_src) - 1;
  const int32_t row = lists[(fg ? S.fg_list : S.bg_list) + pos];
  const float4 b = reinterpret_cast<const float4 *>(boxes)[row];
  const float bb[4] = {b.x, b.y, b.z, b.w};
  float roi[4], t[4] = {0.f, 0.f, 0.f, 0.f};
  mpn_feed::train_box(bb, S.scale, S.width, S.flip, roi);
  int lab = 1;
  if (fg) {
    lab = 1 + label[row];
    const float4 g = reinterpret_cast<const float4 *>(boxes)[row_off[S.fg_src] + corr[row] - 1];
    const float gg[4] = {g.x, g.y, g.z, g.w};
    float gt[4];
    mpn_feed::train_box(gg, S.scale, S.width, S.flip, gt);
    if (lab > 1) mpn_feed::target_block(roi, gt, P.mean, P.std_, t);
  }
  if (lane < 4) out_boxes[4 * r + lane] = roi[lane];
  if (lane == 0) out_labels[r] = lab;
  for (int c = lane; c < 4 * P.C; c += 32) {
    const int q = c & 3;
    const float v = q == 0 ? t[0] : (q == 1 ? t[1] : (q == 2 ? t[2] : t[3]));
    out_targets[r * 4 * P.C + c] = (c >> 2) == lab - 1 && lab > 1 ? v : 0.f;
  }
}

// ------------------------------------------------------------------------------------------------------------- host side
namespace {
// getAnnotation + getGTBoxes + the crowd list of one image, and the proposals after filterArea / filterScore
struct ImageRows {
  std::vector<float> gt, crowd, props;
  std::vector<int32_t> cls;
};
const char *image_rows(int64_t n_ann, const double *xywh, const double *area, const int32_t *cls, const int32_t *flags, double min_area,
                       int64_t n_prop, const float *prop_box, const float *prop_score, int32_t best_number, double min_prop_area,
                       int32_t num_classes, ImageRows &R) {
  R.gt.clear(); R.crowd.clear(); R.props.clear(); R.cls.clear();
  for (int64_t j = 0; j < n_ann; ++j) {
    if (!(area[j] > min_area)) continue;
    for (int k = 0; k < 4; ++k) if (!std::isfinite(xywh[4 * j + k])) return "an annotation box is not finite";
    float b[4];
    mpn_feed::gt_box(xywh + 4 * j, b);
    const bool crowd = flags[j] & 1, difficult = flags[j] & 2;
    if (crowd) R.crowd.insert(R.crowd.end(), b, b + 4);
    if (!difficult && !crowd) {
      if (cls[j] < 1 || cls[j] > num_classes) return "a class id is outside 1..num_classes";
      R.gt.insert(R.gt.end(), b, b + 4);
      R.cls.push_back(cls[j]);
    }
  }
  std::vector<int64_t> keep;
  for (int64_t p = 0; p < n_prop; ++p) {
    const float *b = prop_box + 4 * p;
    for (int k = 0; k < 4; ++k) if (!std::isfinite(b[k])) return "a proposal box is not finite";
    if (min_prop_area != 0.0 && !(mpn_img::fmul(mpn_img::fsub(b[2], b[0]), mpn_img::fsub(b[3], b[1])) > (float)min_prop_area)) continue;
    keep.push_back(p);
  }
  if (prop_score && (int64_t)keep.size() > best_number) {     // filterScore: the best_number highest, in score order
    std::stable_sort(keep.begin(), keep.end(), [&](int64_t a, int64_t b) { return prop_score[a] > prop_score[b]; });
    keep.resize(best_number);
  }
  for (int64_t p : keep) R.props.insert(R.props.end(), prop_box + 4 * p, prop_box + 4 * p + 4);
  return nullptr;
}
}  // namespace

// the matching pass over the uploaded tables: kernels, list offsets on the host, lists
static int roidb_build(mpn_roidb *db) {
  mpn_ctx *ctx = db->ctx;
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  const int n = db->n_images;
  const int64_t n_counts = (int64_t)db->n_sets * 2 * n;
  roidb_match_kernel<<<n, kMT, 0, ctx->stream>>>(db->boxes.p, db->row_off_dev.p, db->gt_off_dev.p, db->gt_box.p, db->gt_cls.p,
                                                 db->crowd_off_dev.p, db->crowd_box.p, n, db->thr, db->overlap.p, db->corr.p,
                                                 db->label.p, db->offs.p);
  MPN_LAUNCHED(ctx);
  MPN_TRY(mpn_scan_exclusive_launch(ctx, db->offs.p, (int)n_counts));
  db->list_off.resize(n_counts + 1);
  MPN_CUDA(ctx, cudaMemcpyAsync(db->list_off.data(), db->offs.p, sizeof(int32_t) * (n_counts + 1), cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  MPN_TRY(db->lists.alloc(ctx, (size_t)db->list_off.back()));
  roidb_compact_kernel<<<n, kMT, 0, ctx->stream>>>(db->overlap.p, db->row_off_dev.p, n, db->thr, db->offs.p, db->lists.p);
  MPN_LAUNCHED(ctx);
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

extern "C" {

int mpn_roidb_create(mpn_ctx *ctx, int32_t n_images, const int64_t *ann_off, const double *ann_xywh, const double *ann_area,
                     const int32_t *ann_class, const int32_t *ann_flags, double min_area, const int64_t *prop_off,
                     const float *prop_box, const float *prop_score, int32_t best_number, double min_proposal_area,
                     int32_t num_classes, int32_t n_sets, const float *thresholds, mpn_roidb **out) {
  if (!ctx || !out) return MPN_ERR_ARG;
  *out = nullptr;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, n_images >= 1 && ann_off && prop_off && thresholds && num_classes >= 1 && best_number >= 1,
                "roidb: an argument is missing or out of range");
  MPN_CHECK_ARG(ctx, n_sets >= 1 && n_sets <= kMaxSets, "roidb: 1 to 16 threshold sets");
  MPN_CHECK_ARG(ctx, ann_off[0] == 0 && prop_off[0] == 0, "roidb: offsets start at 0");
  for (int i = 0; i < n_images; ++i)
    MPN_CHECK_ARG(ctx, ann_off[i + 1] >= ann_off[i] && prop_off[i + 1] >= prop_off[i], "roidb: offsets must ascend");
  MPN_CHECK_ARG(ctx, ann_off[n_images] == 0 || (ann_xywh && ann_area && ann_class && ann_flags), "roidb: annotation arrays missing");
  MPN_CHECK_ARG(ctx, prop_off[n_images] == 0 || prop_box, "roidb: proposal boxes missing");
  Thresholds thr{};
  thr.n = n_sets;
  for (int s = 0; s < n_sets; ++s) {
    const float fg = thresholds[3 * s], lo = thresholds[3 * s + 1], hi = thresholds[3 * s + 2];
    MPN_CHECK_ARG(ctx, std::isfinite(fg) && std::isfinite(lo) && std::isfinite(hi) && fg > 0.f && lo <= hi,
                  "roidb: a threshold set must have fg > 0 and bg_lo <= bg_hi, all finite");
    thr.fg[s] = fg; thr.lo[s] = lo; thr.hi[s] = hi;
  }
  mpn_roidb *db = new mpn_roidb();
  db->ctx = ctx; db->n_images = n_images; db->n_sets = n_sets; db->num_classes = num_classes; db->thr = thr;
  auto fail = [&](int rc) { mpn_roidb_destroy(db); return rc; };
  std::vector<float> boxes, gt, crowd;
  std::vector<int32_t> cls;
  db->row_off.assign(1, 0); db->gt_off.assign(1, 0); db->crowd_off.assign(1, 0);
  ImageRows R;
  for (int i = 0; i < n_images; ++i) {
    const int64_t a0 = ann_off[i], p0 = prop_off[i];
    const char *e = image_rows(ann_off[i + 1] - a0, ann_xywh + 4 * a0, ann_area + a0, ann_class + a0, ann_flags + a0, min_area,
                               prop_off[i + 1] - p0, prop_box + 4 * p0, prop_score ? prop_score + p0 : nullptr, best_number,
                               min_proposal_area, num_classes, R);
    if (e) return fail(mpn_fail(ctx, MPN_ERR_ARG, std::string("roidb: image ") + std::to_string(i) + ": " + e));
    boxes.insert(boxes.end(), R.gt.begin(), R.gt.end());
    boxes.insert(boxes.end(), R.props.begin(), R.props.end());
    gt.insert(gt.end(), R.gt.begin(), R.gt.end());
    crowd.insert(crowd.end(), R.crowd.begin(), R.crowd.end());
    cls.insert(cls.end(), R.cls.begin(), R.cls.end());
    db->n_gt.push_back((int32_t)R.cls.size());
    db->row_off.push_back((int64_t)boxes.size() / 4);
    db->gt_off.push_back((int64_t)gt.size() / 4);
    db->crowd_off.push_back((int64_t)crowd.size() / 4);
  }
  const int64_t rows = db->row_off.back();
  const int64_t n_counts = (int64_t)n_sets * 2 * n_images;
  if (rows * n_sets >= ((int64_t)1 << 31) - 1 || n_counts >= ((int64_t)1 << 31) - 1)
    return fail(mpn_fail(ctx, MPN_ERR_ARG, "roidb: rows x threshold sets must stay below 2^31"));
  cudaStream_t st = ctx->stream;
  int rc;
  if ((rc = db->boxes.alloc(ctx, 4 * rows)) || (rc = db->overlap.alloc(ctx, rows)) || (rc = db->corr.alloc(ctx, rows)) ||
      (rc = db->label.alloc(ctx, rows)) || (rc = db->gt_box.alloc(ctx, gt.size())) || (rc = db->crowd_box.alloc(ctx, crowd.size())) ||
      (rc = db->gt_cls.alloc(ctx, cls.size())) || (rc = db->row_off_dev.alloc(ctx, n_images + 1)) ||
      (rc = db->gt_off_dev.alloc(ctx, n_images + 1)) || (rc = db->crowd_off_dev.alloc(ctx, n_images + 1)) ||
      (rc = db->offs.alloc(ctx, n_counts + 1)))
    return fail(rc);
  auto up = [&](void *dst, const void *src, size_t bytes) {
    return bytes ? cudaMemcpyAsync(dst, src, bytes, cudaMemcpyHostToDevice, st) : cudaSuccess;
  };
  cudaError_t ce = cudaSuccess;
  const size_t oi = sizeof(int64_t) * (n_images + 1);
  for (auto [d, s, b] : {std::tuple<void *, const void *, size_t>{db->boxes.p, boxes.data(), sizeof(float) * boxes.size()},
                         {db->gt_box.p, gt.data(), sizeof(float) * gt.size()}, {db->crowd_box.p, crowd.data(), sizeof(float) * crowd.size()},
                         {db->gt_cls.p, cls.data(), sizeof(int32_t) * cls.size()}, {db->row_off_dev.p, db->row_off.data(), oi},
                         {db->gt_off_dev.p, db->gt_off.data(), oi}, {db->crowd_off_dev.p, db->crowd_off.data(), oi}})
    if (ce == cudaSuccess) ce = up(d, s, b);
  if (ce != cudaSuccess) return fail(mpn_fail(ctx, MPN_ERR_CUDA, std::string("roidb upload: ") + cudaGetErrorString(ce)));
  rc = roidb_build(db);
  if (rc) return fail(rc);
  *out = db;
  return MPN_OK;
}

void mpn_roidb_destroy(mpn_roidb *db) {
  if (!db) return;
  if (db->ctx) { cudaSetDevice(db->ctx->device); cudaStreamSynchronize(db->ctx->stream); }
  for (auto *b : {&db->boxes, &db->overlap, &db->gt_box, &db->crowd_box, &db->stats_tmp, &db->b_boxes, &db->b_targets, &db->b_losses})
    b->release();
  for (auto *b : {&db->corr, &db->label, &db->gt_cls, &db->lists, &db->offs, &db->b_labels}) b->release();
  for (auto *b : {&db->row_off_dev, &db->gt_off_dev, &db->crowd_off_dev}) b->release();
  db->stats_out.release();
  for (auto &b : db->raw) b.release();
  for (auto &b : db->images) b.release();
  delete db;
}

int mpn_roidb_counts(mpn_roidb *db, int32_t *counts, int64_t *n_rows) {
  if (!db) return MPN_ERR_ARG;
  const size_t n = (size_t)db->n_sets * 2 * db->n_images;
  if (counts)
    for (size_t j = 0; j < n; ++j) counts[j] = db->list_off[j + 1] - db->list_off[j];
  if (n_rows) *n_rows = db->row_off.back();
  return MPN_OK;
}

int mpn_roidb_image_rows(mpn_roidb *db, int32_t image, float *boxes, float *overlap, int32_t *corr, int32_t *label, int64_t capacity,
                         int64_t *n_rows, int32_t *n_gt) {
  if (!db) return MPN_ERR_ARG;
  mpn_ctx *ctx = db->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, image >= 0 && image < db->n_images, "roidb: image out of range");
  const int64_t r0 = db->row_off[image], n = db->row_off[image + 1] - r0;
  if (n_rows) *n_rows = n;
  if (n_gt) *n_gt = db->n_gt[image];
  if (!boxes && !overlap && !corr && !label) return MPN_OK;
  MPN_CHECK_ARG(ctx, capacity >= n, "roidb: output buffers too small");
  cudaStream_t st = ctx->stream;
  if (n > 0) {
    if (boxes) MPN_CUDA(ctx, cudaMemcpyAsync(boxes, db->boxes.p + 4 * r0, sizeof(float) * 4 * n, cudaMemcpyDeviceToHost, st));
    if (overlap) MPN_CUDA(ctx, cudaMemcpyAsync(overlap, db->overlap.p + r0, sizeof(float) * n, cudaMemcpyDeviceToHost, st));
    if (corr) MPN_CUDA(ctx, cudaMemcpyAsync(corr, db->corr.p + r0, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
    if (label) MPN_CUDA(ctx, cudaMemcpyAsync(label, db->label.p + r0, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, st));
  }
  MPN_CUDA(ctx, cudaStreamSynchronize(st));
  return MPN_OK;
}

int mpn_roidb_list(mpn_roidb *db, int32_t set, int32_t kind, int32_t image, int32_t *rows, int64_t capacity, int64_t *n_out) {
  if (!db) return MPN_ERR_ARG;
  mpn_ctx *ctx = db->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, set >= 0 && set < db->n_sets && (kind == 0 || kind == 1) && image >= 0 && image < db->n_images,
                "roidb: set, kind (0 bg, 1 fg) or image out of range");
  const int64_t j = ((int64_t)set * 2 + kind) * db->n_images + image;
  const int64_t a = db->list_off[j], n = db->list_off[j + 1] - a;
  if (n_out) *n_out = n;
  if (!rows) return MPN_OK;
  MPN_CHECK_ARG(ctx, capacity >= n, "roidb: output buffer too small");
  if (n > 0) MPN_CUDA(ctx, cudaMemcpyAsync(rows, db->lists.p + a, sizeof(int32_t) * n, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  const int64_t r0 = db->row_off[image];
  for (int64_t k = 0; k < n; ++k) rows[k] -= (int32_t)r0;      // rows local to the image
  return MPN_OK;
}

int mpn_roidb_regression_stats(mpn_roidb *db, int32_t set, int32_t n_first, float *mean, float *std_) {
  if (!db) return MPN_ERR_ARG;
  mpn_ctx *ctx = db->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, mean && std_ && set >= 0 && set < db->n_sets && n_first >= 1, "roidb stats: bad arguments");
  const int m = std::min(n_first, db->n_images);
  const int64_t j = ((int64_t)set * 2 + 1) * db->n_images;        // the fg lists of images 0 .. m-1 are contiguous
  const int64_t a = db->list_off[j], n = db->list_off[j + m] - a;
  MPN_CHECK_ARG(ctx, n >= 2, "roidb stats: fewer than two foreground rows in the first images");
  MPN_TRY(db->stats_tmp.alloc(ctx, 4 * n));
  MPN_TRY(db->stats_out.alloc(ctx, 8));
  {
    MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
    roidb_stats_rows_kernel<<<(unsigned)ceil_div64(n, 256), 256, 0, ctx->stream>>>(db->lists.p, a, n, db->boxes.p, db->corr.p,
                                                                                   db->row_off_dev.p, db->n_images, db->stats_tmp.p);
    MPN_LAUNCHED(ctx);
    roidb_stats_reduce_kernel<<<4, 1024, 0, ctx->stream>>>(db->stats_tmp.p, n, db->stats_out.p);
    MPN_LAUNCHED(ctx);
  }
  double o[8];
  MPN_CUDA(ctx, cudaMemcpyAsync(o, db->stats_out.p, sizeof o, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  for (int k = 0; k < 4; ++k) { mean[k] = (float)o[k]; std_[k] = (float)o[4 + k]; }
  return MPN_OK;
}

int mpn_sample_plan(const int32_t *n_bg, const int32_t *n_fg, int32_t n_images, uint64_t seed, uint32_t step, int32_t set, int32_t n_slots,
                    int32_t *image, int32_t *bg_src, int32_t *fg_src, int32_t *flip) {
  if (!n_bg || !n_fg || !image || !bg_src || !fg_src || !flip || n_images < 1 || n_slots < 1 || set < 0 || set > 255)
    return MPN_ERR_ARG;
  bool any_bg = false, any_fg = false;
  for (int i = 0; i < n_images; ++i) { any_bg |= n_bg[i] > 0; any_fg |= n_fg[i] > 0; }
  if (!any_bg || !any_fg) return MPN_ERR_STATE;                       // permuteIdx would draw forever
  for (int k = 0; k < n_slots; ++k) {
    int32_t cur = -1, bg = -1, fg = -1;
    for (uint32_t d = 0; bg < 0 || fg < 0; ++d) {                     // permuteIdx + tablex.update: a kind found stays
      cur = (int32_t)mpn_feed::rand_int(mpn_feed::draw_u32(seed, step, k, set, mpn_feed::DRAW_IMAGE, d), n_images) - 1;
      if (n_bg[cur] > 0) bg = cur;
      if (n_fg[cur] > 0) fg = cur;
    }
    image[k] = cur; bg_src[k] = bg; fg_src[k] = fg;
    flip[k] = (int32_t)mpn_feed::rand_int(mpn_feed::draw_u32(seed, step, k, set, mpn_feed::DRAW_FLIP, 0), 2) - 1;
  }
  return MPN_OK;
}

int mpn_integral_set(uint64_t seed, uint32_t step, int32_t n_sets, int32_t *set) {
  if (!set || n_sets < 1) return MPN_ERR_ARG;
  *set = (int32_t)mpn_feed::rand_int(mpn_feed::draw_u32(seed, step, 0, 0, mpn_feed::DRAW_INTEGRAL, 0), n_sets) - 1;
  return MPN_OK;
}

int mpn_train_images_size(int32_t H0, int32_t W0, double scale, double max_size, int32_t *h, int32_t *w, double *im_scale) {
  if (H0 <= 0 || W0 <= 0 || !(scale > 0) || !(max_size > 0) || !h || !w || !im_scale) return MPN_ERR_ARG;
  int hh, ww;
  mpn_feed::train_size(H0, W0, scale, max_size, &hh, &ww, im_scale);
  *h = hh; *w = ww;
  return MPN_OK;
}

int mpn_roidb_sample_dev(mpn_roidb *db, int32_t set, uint64_t seed, uint32_t step, int32_t n_slots, const int32_t *bg_src,
                         const int32_t *fg_src, const int32_t *flip, const double *im_scale, const int32_t *width, int32_t bg_each,
                         int32_t fg_each, const float *mean, const float *std_, int32_t num_classes, float *boxes_dev,
                         int32_t *labels_dev, float *targets_dev, int32_t *rois_per_image) {
  if (!db) return MPN_ERR_ARG;
  mpn_ctx *ctx = db->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, bg_src && fg_src && flip && im_scale && width && mean && std_ && boxes_dev && labels_dev && targets_dev && rois_per_image,
                "roidb sample: an argument is missing");
  MPN_CHECK_ARG(ctx, set >= 0 && set < db->n_sets && n_slots >= 1 && n_slots <= kMaxSlots && bg_each >= 0 && fg_each >= 0,
                "roidb sample: set, 1..32 images or per-image counts out of range");
  MPN_CHECK_ARG(ctx, num_classes == db->num_classes + 1, "roidb sample: num_classes must be the dataset's classes + 1 (background)");
  SamplePlan P{};
  P.n_slots = n_slots; P.set = set; P.C = num_classes; P.step = step; P.seed = seed;
  for (int k = 0; k < 4; ++k) { P.mean[k] = mean[k]; P.std_[k] = std_[k]; }
  int64_t R = 0;
  for (int k = 0; k < n_slots; ++k) {
    MPN_CHECK_ARG(ctx, bg_src[k] >= 0 && bg_src[k] < db->n_images && fg_src[k] >= 0 && fg_src[k] < db->n_images && width[k] > 0,
                  "roidb sample: a source image or width is out of range");
    const int64_t jb = ((int64_t)set * 2) * db->n_images + bg_src[k], jf = ((int64_t)set * 2 + 1) * db->n_images + fg_src[k];
    SampleSlot &S = P.s[k];
    S.bg_list = db->list_off[jb]; S.n_bg_src = db->list_off[jb + 1] - S.bg_list;
    S.fg_list = db->list_off[jf]; S.n_fg_src = db->list_off[jf + 1] - S.fg_list;
    MPN_CHECK_ARG(ctx, S.n_bg_src > 0 && S.n_fg_src > 0, "roidb sample: a bg source without bg rows or a fg source without fg rows");
    S.nb = std::min(bg_each, S.n_bg_src); S.nf = std::min(fg_each, S.n_fg_src);
    S.fg_src = fg_src[k]; S.row0 = (int32_t)R; S.width = width[k]; S.flip = flip[k] != 0; S.scale = (float)im_scale[k];
    rois_per_image[k] = S.nb + S.nf;
    R += S.nb + S.nf;
  }
  MPN_CHECK_ARG(ctx, R > 0, "roidb sample: no rows drawn");
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  roidb_sample_kernel<<<(unsigned)ceil_div64(R * 32, 256), 256, 0, ctx->stream>>>(P, R, db->lists.p, db->boxes.p, db->corr.p, db->label.p,
                                                                                  db->row_off_dev.p, boxes_dev, labels_dev, targets_dev);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_roidb_sample(mpn_roidb *db, int32_t set, uint64_t seed, uint32_t step, int32_t n_slots, const int32_t *plan,
                     const uint8_t *const *images_hwc, const int32_t *hw0, const mpn_image_transform *tf, double scale, double max_size,
                     int32_t bg_each, int32_t fg_each, const float *mean, const float *std_, int32_t num_classes, int32_t *image_hw,
                     int32_t *rois_per_image) {
  if (!db) return MPN_ERR_ARG;
  mpn_ctx *ctx = db->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, plan && images_hwc && hw0 && tf && image_hw && rois_per_image && n_slots >= 1 && n_slots <= kMaxSlots,
                "roidb sample: an argument is missing");
  std::vector<int32_t> bg(n_slots), fg(n_slots), fl(n_slots), wd(n_slots);
  std::vector<double> sc(n_slots);
  if ((int)db->images.size() < n_slots) { db->images.resize(n_slots); db->raw.resize(n_slots); }
  for (int k = 0; k < n_slots; ++k) {
    MPN_CHECK_ARG(ctx, images_hwc[k] && hw0[2 * k] > 0 && hw0[2 * k + 1] > 0, "roidb sample: an image is missing or empty");
    int32_t h = 0, w = 0;
    MPN_CHECK_ARG(ctx, mpn_train_images_size(hw0[2 * k], hw0[2 * k + 1], scale, max_size, &h, &w, &sc[k]) == MPN_OK && h > 0 && w > 0,
                  "roidb sample: bad scale / max_size, or an image scales to nothing");
    image_hw[2 * k] = h; image_hw[2 * k + 1] = w;
    bg[k] = plan[4 * k + 1]; fg[k] = plan[4 * k + 2]; fl[k] = plan[4 * k + 3]; wd[k] = w;
    const size_t nb = (size_t)hw0[2 * k] * hw0[2 * k + 1] * 3;
    MPN_TRY(db->raw[k].alloc(ctx, nb));
    MPN_TRY(db->images[k].alloc(ctx, (size_t)3 * h * w));
    MPN_CUDA(ctx, cudaMemcpyAsync(db->raw[k].p, images_hwc[k], nb, cudaMemcpyHostToDevice, ctx->stream));
    MPN_TRY(mpn_get_images_u8_flip_launch(ctx, db->raw[k].p, hw0[2 * k], hw0[2 * k + 1], tf, h, w, fl[k], db->images[k].p));
  }
  const int64_t Rmax = (int64_t)n_slots * (bg_each + fg_each);
  MPN_TRY(db->b_boxes.alloc(ctx, 4 * std::max<int64_t>(Rmax, 1)));
  MPN_TRY(db->b_labels.alloc(ctx, std::max<int64_t>(Rmax, 1)));
  MPN_TRY(db->b_targets.alloc(ctx, 4 * (size_t)num_classes * std::max<int64_t>(Rmax, 1)));
  MPN_TRY(mpn_roidb_sample_dev(db, set, seed, step, n_slots, bg.data(), fg.data(), fl.data(), sc.data(), wd.data(), bg_each, fg_each, mean,
                               std_, num_classes, db->b_boxes.p, db->b_labels.p, db->b_targets.p, rois_per_image));
  int64_t R = 0;
  for (int k = 0; k < n_slots; ++k) R += rois_per_image[k];
  db->b_R = R; db->b_C = num_classes; db->b_slots = n_slots; db->b_set = set;
  db->batch_hw.assign(image_hw, image_hw + 2 * n_slots);
  db->batch_rois.assign(rois_per_image, rois_per_image + n_slots);
  return MPN_OK;
}

int mpn_roidb_batch_host(mpn_roidb *db, float *const *images, float *boxes, int32_t *labels, float *targets) {
  if (!db) return MPN_ERR_ARG;
  mpn_ctx *ctx = db->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, db->b_slots > 0, "roidb: no batch sampled yet");
  cudaStream_t st = ctx->stream;
  for (int k = 0; images && k < db->b_slots; ++k)
    if (images[k])
      MPN_CUDA(ctx, cudaMemcpyAsync(images[k], db->images[k].p, sizeof(float) * 3 * db->batch_hw[2 * k] * db->batch_hw[2 * k + 1],
                                    cudaMemcpyDeviceToHost, st));
  if (boxes) MPN_CUDA(ctx, cudaMemcpyAsync(boxes, db->b_boxes.p, sizeof(float) * 4 * db->b_R, cudaMemcpyDeviceToHost, st));
  if (labels) MPN_CUDA(ctx, cudaMemcpyAsync(labels, db->b_labels.p, sizeof(int32_t) * db->b_R, cudaMemcpyDeviceToHost, st));
  if (targets) MPN_CUDA(ctx, cudaMemcpyAsync(targets, db->b_targets.p, sizeof(float) * 4 * db->b_C * db->b_R, cudaMemcpyDeviceToHost, st));
  MPN_CUDA(ctx, cudaStreamSynchronize(st));
  return MPN_OK;
}

}  // extern "C"

int mpn_roidb_batch_view(mpn_roidb *db, MpnBatchView *v) {
  if (!db || !v) return MPN_ERR_ARG;
  MPN_CHECK_ARG(db->ctx, db->b_slots > 0, "roidb: no batch sampled yet");
  v->ctx = db->ctx; v->n_slots = db->b_slots; v->C = db->b_C; v->set = db->b_set; v->n_sets = db->n_sets;
  v->images.assign(db->b_slots, nullptr);
  for (int k = 0; k < db->b_slots; ++k) v->images[k] = db->images[k].p;
  v->hw = db->batch_hw.data(); v->rois = db->batch_rois.data();
  v->boxes = db->b_boxes.p; v->labels = db->b_labels.p; v->targets = db->b_targets.p;
  return MPN_OK;
}

extern "C" {

int mpn_model_train_step_batch(mpn_model *m, mpn_roidb *db, float *losses) {
  if (!m || !db || !losses) return MPN_ERR_ARG;
  mpn_ctx *ctx = db->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, db->b_slots > 0, "roidb: no batch sampled yet");
  const int K = mpn_model_n_cls_heads(m);
  if (K > 1) {                                     // integral: the batch's threshold set picks the class head it trains
    if (db->n_sets != K)
      return mpn_fail(ctx, MPN_ERR_ARG, "step_batch: the roidb has " + std::to_string(db->n_sets) + " threshold sets and the model " +
                                            std::to_string(K) + " class heads; an integral model trains head s on set s");
    MPN_TRY(mpn_model_train_select_head(m, db->b_set));
  }
  std::vector<const float *> ims(db->b_slots);
  for (int k = 0; k < db->b_slots; ++k) ims[k] = db->images[k].p;
  MPN_TRY(db->b_losses.alloc(ctx, 4));
  MPN_TRY(mpn_model_train_step_dev(m, db->b_slots, ims.data(), db->batch_hw.data(), db->batch_rois.data(), db->b_boxes.p, db->b_labels.p,
                                   db->b_targets.p, db->b_losses.p));
  MPN_CUDA(ctx, cudaMemcpyAsync(losses, db->b_losses.p, sizeof(float) * 3, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_TRY(mpn_ovf_copy_async(ctx, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return mpn_ovf_test(ctx);
}

// ---- host-only views of the rules (no GPU)
int mpn_debug_attach_proposals(int64_t n_ann, const double *ann_xywh, const double *ann_area, const int32_t *ann_class,
                               const int32_t *ann_flags, double min_area, int64_t n_prop, const float *prop_box, const float *prop_score,
                               int32_t best_number, double min_proposal_area, int32_t num_classes, float *boxes, float *overlap,
                               int32_t *corr, int32_t *label, int64_t capacity, int64_t *n_rows, int32_t *n_gt) {
  if (n_ann < 0 || n_prop < 0 || best_number < 1 || num_classes < 1 || (n_ann && (!ann_xywh || !ann_area || !ann_class || !ann_flags)) ||
      (n_prop && !prop_box))
    return MPN_ERR_ARG;
  ImageRows R;
  if (image_rows(n_ann, ann_xywh, ann_area, ann_class, ann_flags, min_area, n_prop, prop_box, prop_score, best_number, min_proposal_area,
                 num_classes, R))
    return MPN_ERR_ARG;
  const int G = (int)R.cls.size(), NC = (int)R.crowd.size() / 4;
  const int64_t n = G + (int64_t)R.props.size() / 4;
  if (n_rows) *n_rows = n;
  if (n_gt) *n_gt = G;
  if (!boxes || !overlap || !corr || !label) return MPN_OK;
  if (capacity < n) return MPN_ERR_ARG;
  for (int64_t i = 0; i < n; ++i) {
    const float *a = i < G ? &R.gt[4 * i] : &R.props[4 * (i - G)];
    for (int k = 0; k < 4; ++k) boxes[4 * i + k] = a[k];
    mpn_feed::attach_row(a, i < G, R.gt.data(), R.cls.data(), G, R.crowd.data(), NC, &overlap[i], &corr[i], &label[i]);
  }
  return MPN_OK;
}

int mpn_debug_sample_rows(int64_t R, const float *rois, const float *gtboxes, const int32_t *labels, double im_scale, int32_t width,
                          int32_t flip, const float *mean, const float *std_, int32_t num_classes, float *boxes, float *targets) {
  if (R < 0 || !rois || !gtboxes || !labels || !mean || !std_ || !boxes || !targets || num_classes < 2 || width < 1) return MPN_ERR_ARG;
  for (int64_t r = 0; r < R; ++r) {
    if (labels[r] < 1 || labels[r] > num_classes) return MPN_ERR_ARG;
    float roi[4], gt[4], t[4] = {0.f, 0.f, 0.f, 0.f};
    mpn_feed::train_box(rois + 4 * r, (float)im_scale, width, flip, roi);
    mpn_feed::train_box(gtboxes + 4 * r, (float)im_scale, width, flip, gt);
    if (labels[r] > 1) mpn_feed::target_block(roi, gt, mean, std_, t);
    for (int k = 0; k < 4; ++k) boxes[4 * r + k] = roi[k];
    for (int c = 0; c < 4 * num_classes; ++c) targets[r * 4 * num_classes + c] = (c / 4 == labels[r] - 1 && labels[r] > 1) ? t[c & 3] : 0.f;
  }
  return MPN_OK;
}

}  // extern "C"

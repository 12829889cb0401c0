/* ============================================================================
 * mpn_abi.h — C ABI of libmpn_b200.so: the drop-in boundary for the
 * multipathnet detection forward hot path on H100 (sm_90a).
 *
 * Plain C declarations only (no macros in prototypes, no torch/TH types) so the
 * block between MPN_CDEF_BEGIN/END can be pasted verbatim into LuaJIT
 * `ffi.cdef` (lua/mpn_ffi.lua does exactly that) and is what Python loads via
 * ctypes (multipathnet_b200/_lib.py). Every entry point names the reference
 * interface it replaces (paths relative to facebookresearch/multipathnet).
 *
 * Conventions
 *  - every function returns 0 on success, <0 on error; text via mpn_last_error.
 *    Nothing exits, throws, or longjmps across the boundary.
 *  - `*_dev` pointers are device pointers on the ctx's device; others are host
 *    pointers. The caller owns all I/O buffers; the library owns ctx/model only.
 *  - calls run on the ctx's stream; entry points taking/returning HOST buffers
 *    are synchronous (like the reference's blocking :float()/:cuda() copies),
 *    `_dev` entry points are stream-ordered and asynchronous.
 *  - boxes are 1-based pixel coordinates [x1,y1,x2,y2]; ROI rows are
 *    [batch_idx(1-based), x1, y1, x2, y2] (ImageDetect.lua:66-70).
 *  - no global mutable state: one mpn_ctx per (thread, device)
 *    (test_runner.lua:55-66 runs one replica per thread/GPU).
 * ==========================================================================*/
#ifndef MPN_ABI_H
#define MPN_ABI_H
#include <stdint.h>
#ifdef __cplusplus
extern "C" {
#endif
/* MPN_CDEF_BEGIN */

typedef struct mpn_ctx mpn_ctx;
typedef struct mpn_model mpn_model;

/* ---- context ------------------------------------------------------------- */
/* device: CUDA ordinal. cuda_stream: a cudaStream_t, or NULL for the legacy
 * default stream (what cutorch uses unless cutorch.setStream was called).   */
int mpn_ctx_create(int device, void *cuda_stream, mpn_ctx **out);
/* A context on a stream of its own (non-blocking, created and destroyed with the ctx; priority as cudaStreamCreateWithPriority,
 * clamped to the device's range, 0 = default): for SEVERAL model replicas on one GPU. The reference runs one model replica per
 * donkey thread (test_runner.lua:55-66); with K threads per GPU, each on its own ctx / stream, the layer-boundary and NMS-chain
 * bubbles of one replica are filled by the kernels of the others. Work of different
 * contexts is unordered; mpn_ctx_wait_ctx(ctx, other) makes everything enqueued on `ctx` afterwards wait for what `other` has
 * enqueued so far (the join before the end-of-run gather). mpn_ctx_stream returns the cudaStream_t (interop with the caller's
 * own kernels / events). */
int mpn_ctx_create_stream(int device, int priority, mpn_ctx **out);
void *mpn_ctx_stream(const mpn_ctx *ctx);
int mpn_ctx_wait_ctx(mpn_ctx *ctx, mpn_ctx *other);
void mpn_ctx_destroy(mpn_ctx *ctx);
const char *mpn_last_error(const mpn_ctx *ctx);   /* ctx may be NULL: last create error */
int mpn_ctx_synchronize(mpn_ctx *ctx);
/* number of kernels THIS library launched on ctx since creation (bench.py's gpu_launches) */
int64_t mpn_ctx_launch_count(const mpn_ctx *ctx);
const char *mpn_version(void);
/* run-time knobs of the product kernels, so that tests can cover every variant in one process; value < 0 restores the
 * default (the environment variable of the same meaning, else the built-in choice). Names:
 *   "fc_w16"          numerics of the big per-ROI Linears (fc6 / fc7: K >= 2048, >= 1024 outputs), read when a model plans
 *                     its heads: 1 = weight as ONE fp16 plane scaled by a power of two, two tensor-core products per
 *                     MAC (A_hi x W + A_lo x W); 0 = the three-product bf16 split every other layer uses. Unset: 1 for
 *                     single-tower graphs (Fast R-CNN: 4-5e-4 on the scores at full size), 0 for multi-tower graphs
 *                     (MultiPathNet measured 2.3e-3 with it: outside the 1e-3 contract). Environment: MPN_FC_W16.
 *                     Ignored while "bf16" or "fp8" is on.
 *   "bf16"            opt-in bf16 inference numerics, read when a model plans (its trunk for a new image size, its heads
 *                     for a new ROI count) and by mpn_gemm_check / mpn_conv_check (impl 0 and 1): 1 = every layer on the
 *                     wgmma engine (trunk convs after the first layer, the 1x1 conv_mix, ResNet's per-ROI layer4, fc6 /
 *                     fc7 and the cls / bbox heads) issues ONE bf16 product per MAC, A_hi x B_hi, on the hi planes
 *                     (rn_bf16 of the stored fp32 activation and weight), instead of three; 0 or < 0 = the default.
 *                     The first layer, the storage formats, ROI pooling, split-K, NMS and the per-ROI row invariance do
 *                     not change. The 1e-3 fp32 contract does NOT apply: its bars are 1e-3 normwise against an oracle
 *                     that rounds the same operands to bf16, bit-exact NMS on its own outputs, and chunked == full.
 *                     A weight that a model has already prepared as an fp16 plane (fc_w16) cannot be re-planned in this
 *                     mode: build the model with the option set. No environment variable.
 *   "fp8"             opt-in fp8 inference numerics, read when and where "bf16" is: 1 = every layer on the wgmma engine
 *                     except the cls / bbox heads (trunk convs after the first layer, the 1x1 conv_mix, ResNet's per-ROI
 *                     layer4, fc6 / fc7) issues ONE e4m3 tensor-core product per MAC; 0 or < 0 = the default. Operands:
 *                     q = rn_e4m3(2^e * h) of the hi planes h, e = the largest integer with max|h| * 2^e <= 448 (clamped
 *                     to [-60, 60]; 0 for an all-zero group), one e per output channel of a weight and one per sample of an
 *                     activation (the image in the trunk, the ROI in per-ROI layers, so chunked calls equal the full call
 *                     bit for bit); the epilogue multiplies by 2^-(e_a + e_w), exact. A group whose max is not finite fails
 *                     the next host-synchronous call (MPN_ERR_STATE). The heads keep the default three-product numerics;
 *                     the first layer, storage formats, ROI pooling, split-K and NMS do not change. "fp8" and "bf16" both
 *                     on fail the plan (and mpn_gemm_check / mpn_conv_check) with MPN_ERR_ARG. Bars (DESIGN 4): 1e-5
 *                     normwise against an fp64 product of the same e4m3 operands at the engine (5e-5 at K = 25088);
 *                     whole graphs against an oracle with the same operand rule. No environment variable.
 *   "train_bf16"      opt-in bf16 training numerics, read by mpn_model_train_begin and recorded there (a
 *                     change afterwards does not reach a training already begun), and by mpn_debug_conv_backward /
 *                     mpn_debug_pool_backward at each call: 1 = every engine GEMM of the step issues ONE bf16 product per
 *                     MAC on the hi planes. Forward: the layer numerics of "bf16" (every engine layer after the first,
 *                     fc_w16 off). Backward: dW = G^T X, dX = G W of the per-ROI layers and heads, the trunk's weight
 *                     gradient over the tap matrix, the rotated-weight 3x3 dgrad and the stride-2 column GEMM. The
 *                     operand producers write only hi planes (rn_bf16 of the fp32 gradient or weight, the activation's
 *                     stored hi plane). Unchanged: fp32 masters and momentum buffers, optim.sgd, ROI pooling and its
 *                     backward, the gathers, col2im, the criteria, the stored activations' split planes and the max /
 *                     ReLU / dropout rules on hi + lo. 0 or < 0 = the default BF16X3 step. The "bf16" / "fp8" inference
 *                     options still refuse a step. No environment variable.
 * Any other name fails with MPN_ERR_ARG.                                                                           */
int mpn_ctx_set_option(mpn_ctx *ctx, const char *name, int64_t value);
/* per-category kernel timing for roofline reporting: between begin and end every launch group is
 * bracketed by CUDA events on the ctx stream. ms_by_cat[7] = {conv/GEMM tensor cores, first-layer conv,
 * fused ROI pooling, NMS, elementwise glue, max/avg pooling, fp8 operand quantizer}; launches_by_cat likewise (may be NULL). */
int mpn_ctx_profile_begin(mpn_ctx *ctx);
int mpn_ctx_profile_end(mpn_ctx *ctx, double *ms_by_cat, int64_t *launches_by_cat);
/* in-kernel timeline of the tensor-core launches (diagnostics): between begin and end every tensor-core
 * launch i records %globaltimer stamps, min over CTAs in stamps_min[4i..]: {kernel entry, dependency wait passed, first
 * MMA issued, -}, max over CTAs in stamps_max[4i..]: {last MMA issued, last epilogue finished, kernel exit, the time
 * spent in tile epilogues summed over every tile of every CTA} (ns). */
int mpn_ctx_timeline_begin(mpn_ctx *ctx, int32_t max_launches);
int mpn_ctx_timeline_end(mpn_ctx *ctx, uint64_t *stamps_min, uint64_t *stamps_max, int32_t *n_launches);

/* ---- NMS: replaces utils.nms -> nms.c:NMS (utils.lua:29-33, nms.c:59-108) --
 * scored_boxes: N x 5 [x1,y1,x2,y2,score]. Writes the kept ROW INDICES
 * (0-based, selection order = the order nms.c emits its kept rows) into
 * keep_idx (capacity N) and the count into *n_keep. Bit-exact vs nms.c,
 * including its tie behaviour. Host buffers, synchronous.                   */
int mpn_nms(mpn_ctx *ctx, const float *scored_boxes, int64_t N, float thr,
            int32_t *keep_idx, int64_t *n_keep);
/* Batched form (one launch set for all classes of an image, Tester_FRCNN.lua:106-117):
 * segment s covers rows [seg_offsets[s], seg_offsets[s+1]) of scored_boxes;
 * keep_idx is written at the same offsets (indices local to the segment),
 * keep_counts[s] = number kept. Host buffers, synchronous.                  */
int mpn_nms_batched(mpn_ctx *ctx, const float *scored_boxes, const int64_t *seg_offsets,
                    int64_t nseg, float thr, int32_t *keep_idx, int64_t *keep_counts);
/* Same, device buffers, stream-ordered (seg_offsets stays on the host).     */
int mpn_nms_batched_dev(mpn_ctx *ctx, const float *scored_boxes_dev, const int64_t *seg_offsets,
                        int64_t nseg, float thr, int32_t *keep_idx_dev, int32_t *keep_counts_dev);
/* replaces utils.nms_dense (utils.lua:402-462, used by demo.lua:85): 0-based
 * original indices in descending-score order; ties broken by ascending index. */
int mpn_nms_dense(mpn_ctx *ctx, const float *scored_boxes, int64_t N, float thr,
                  int32_t *pick_idx, int64_t *n_pick);
/* replaces utils.bbox_vote -> nms.c:bbox_vote (utils.lua:35-39, nms.c:110-142) */
int mpn_bbox_vote(mpn_ctx *ctx, const float *nms_boxes, int64_t K, const float *scored_boxes,
                  int64_t N, float thr, float *res);

/* ---- region modules ------------------------------------------------------ */
/* nn.Foveal:updateOutput (modules/Foveal.lua:15-44): R x 5 -> 4R x 5, the four
 * regions of ROI i consecutive; fp64 arithmetic rounded once to fp32.       */
int mpn_foveal(mpn_ctx *ctx, const float *rois, int64_t R, float *out);
/* nn.ContextRegion(scale):updateOutput (modules/ContextRegion.lua:14-32)     */
int mpn_context_region(mpn_ctx *ctx, const float *rois, int64_t R, float scale, float *out);
/* nn.BBoxNorm:updateOutput, evaluate mode (modules/BBoxNorm.lua:18-32): in place */
int mpn_bbox_norm(mpn_ctx *ctx, float *deltas, int64_t R, int64_t C4, const float *mean4,
                  const float *std4);
/* the three modules on DEVICE buffers (CudaTensors), stream-ordered, no copies: the reference's Foveal takes its input to the
 * host and back on every forward (Foveal.lua:21-22,42). mean4 / std4 stay host pointers (4 floats each).                */
int mpn_foveal_dev(mpn_ctx *ctx, const float *rois_dev, int64_t R, float *out_dev);
int mpn_context_region_dev(mpn_ctx *ctx, const float *rois_dev, int64_t R, float scale, float *out_dev);
int mpn_bbox_norm_dev(mpn_ctx *ctx, float *deltas_dev, int64_t R, int64_t C4, const float *mean4,
                      const float *std4);
/* utils.convertFrom tensor branch applied per class block of 4
 * (ImageDetect.lua:183-185, utils.lua:226-246): deltas R x 4C, boxes R x 4.   */
int mpn_bbox_decode(mpn_ctx *ctx, const float *deltas, const float *boxes, int64_t R, int64_t C,
                    float *out);

/* ---- inn.ROIPooling(W,H,scale):updateOutput {data, rois} ------------------
 * (call sites vgg.lua:28, alexnet.lua:23, resnet.lua:48, model_utils.lua:215)
 * fmap N x C x H x W fp32 (NCHW as Torch holds it), rois R x 5, out
 * R x C x PH x PW, argmax (R*C*PH*PW int32, flat h*W+w or -1) may be NULL.
 * variant: 1 = Caffe port (end inclusive), 2 = imagine-nn v2 (default).     */
int mpn_roi_pool(mpn_ctx *ctx, const float *fmap, int64_t N, int64_t C, int64_t H, int64_t W,
                 const float *rois, int64_t R, int32_t PW, int32_t PH, float spatial_scale,
                 int32_t variant, float *out, int32_t *argmax);
int mpn_roi_pool_dev(mpn_ctx *ctx, const float *fmap_dev, int64_t N, int64_t C, int64_t H,
                     int64_t W, const float *rois_dev, int64_t R, int32_t PW, int32_t PH,
                     float spatial_scale, int32_t variant, float *out_dev, int32_t *argmax_dev);
/* inn.ROIPooling:updateGradInput, gradient w.r.t. the data: grad_out and argmax
 * R x C x PH x PW (argmax exactly as mpn_roi_pool wrote it), the forward's
 * geometry and rois -> grad_data N x C x H x W, every element written:
 *   grad_data[n,c,h,w] = sum of grad_out[r,c,ph,pw] over the bins of the ROIs
 *   of image n (1-based rois[r][0]) whose argmax is h*W+w; +0 where none is.
 * Each element is summed in fp32 from +0, ascending r, then ph, then pw (no
 * atomics): bit-exact and deterministic. imagine-nn accumulates with atomics,
 * so it agrees up to the rounding of a reordered sum. The gradient w.r.t. the
 * rois is zero. R == 0 writes zeros.                                          */
int mpn_roi_pool_backward(mpn_ctx *ctx, const float *grad_out, const int32_t *argmax, int64_t N,
                          int64_t C, int64_t H, int64_t W, const float *rois, int64_t R, int32_t PW,
                          int32_t PH, float spatial_scale, int32_t variant, float *grad_data);
int mpn_roi_pool_backward_dev(mpn_ctx *ctx, const float *grad_out_dev, const int32_t *argmax_dev,
                              int64_t N, int64_t C, int64_t H, int64_t W, const float *rois_dev,
                              int64_t R, int32_t PW, int32_t PH, float spatial_scale, int32_t variant,
                              float *grad_data_dev);

/* ---- model: the nn.Sequential graphs of models/{vgg,multipathnet,resnet}.lua
 * described as data. Layers operate on numbered tensor slots; slot 0 of the
 * trunk is the input image (1 x 3 x H x W fp32, post-transformer).          */
enum {
  MPN_LAYER_CONV = 1,       /* conv kh x kw, stride, pad, + bias [+ residual] [+ ReLU]; a Linear is a 1x1 conv on a 1x1 map */
  MPN_LAYER_MAXPOOL = 2,    /* k x k, stride, pad, ceil_mode */
  MPN_LAYER_AVGPOOL = 3,    /* global average over H x W (ResNet avgpool 7) */
  MPN_LAYER_FLATTEN = 4     /* (H,W,C) -> 1 x 1 x (H*W*C); reference order (c,ph,pw) is honoured by permuting the next weight */
};
typedef struct mpn_layer {
  int32_t kind;
  int32_t in_slot, out_slot;
  int32_t cin, cout, kh, kw, stride, pad;
  int32_t relu;             /* 1: ReLU fused after bias(+residual) */
  int32_t residual_slot;    /* slot added before ReLU, or -1 */
  int32_t ceil_mode;        /* pooling only */
  int32_t weight, bias;     /* indices into weights[], -1 = none; conv weight is Cout x Cin x kh x kw (Torch layout) */
} mpn_layer;

typedef struct mpn_tower {   /* one region tower of multipathnet.lua:73-113, or THE head of vgg/resnet */
  int32_t region;           /* 0 = the ROI itself, 1..3 = Foveal regions x1.5, x2, x4 (Foveal.lua:36-39) */
  int32_t n_levels;         /* 1..3 pooled trunk taps, channel-concat order (model_utils.lua:229-235) */
  int32_t level_slot[3];    /* trunk slot of each level */
  float   level_scale[3];   /* spatial scale of each level (1/16, 1/8, 1/4) */
  int32_t pooled_w, pooled_h;
  int32_t normalize;        /* 1: L2-normalise each level then x1000 (model_utils.lua:217-220,240) */
  int32_t n_layers;         /* per-ROI layers applied to the pooled R x PH x PW x C tensor (slot 0) */
  int32_t first_layer;      /* index into the model's tower_layers[] array */
  int32_t out_slot;         /* tower-local slot holding the R x 1 x 1 x F result */
} mpn_tower;

typedef struct mpn_head {    /* Linear over a column range of the towers' concat (multipathnet.lua:115-117) */
  int32_t col_begin, col_len;
  int32_t cout;
  int32_t weight, bias;
} mpn_head;

typedef struct mpn_model_desc {
  int32_t n_trunk_layers;  const mpn_layer *trunk_layers;
  int32_t n_towers;        const mpn_tower *towers;
  int32_t n_tower_layers;  const mpn_layer *tower_layers;
  int32_t n_cls_heads;     const mpn_head *cls_heads;   /* >1: integral head, eval = mean of softmaxes (model_utils.lua:296-313) */
  mpn_head bbox_head;
  int32_t num_classes;     /* C incl. background */
  int32_t roi_variant;     /* 1 or 2, see mpn_roi_pool */
  int32_t no_softmax;      /* model.noSoftMax (ImageDetect.lua:189): scores are already probabilities */
  int32_t has_bbox_norm;   /* nn.BBoxNorm appended (model_utils.lua:176-182) */
  float bbox_mean[4], bbox_std[4];
  int32_t max_rois;        /* capacity to allocate for */
  int32_t max_h, max_w;    /* largest scaled image */
} mpn_model_desc;

/* weights[i] are HOST fp32 arrays in Torch layout with n_elem[i] elements; they are
 * copied/re-laid-out at create, nothing is retained.                         */
int mpn_model_create(mpn_ctx *ctx, const mpn_model_desc *desc, const float *const *weights,
                     const int64_t *n_elem, int32_t n_weights, mpn_model **out);
void mpn_model_destroy(mpn_model *m);

/* model:get(1):forward — the conv trunk, once per image (ImageDetect.lua:107-108).
 * image: 3 x H x W fp32 host (or device with _dev), already transformed+scaled. */
int mpn_model_trunk(mpn_model *m, const float *image, int32_t H, int32_t W);
int mpn_model_trunk_dev(mpn_model *m, const float *image_dev, int32_t H, int32_t W);
/* ---- getImages on the device (SURVEY 8f-1): ImageDetect.lua:22-52 + modules/ImageTransformer.lua:19-33 ----------
 * fbcoco.ImageTransformer(mean, std, scale, swap) as plain data: out[c] = (im[swap[c]] * scale - mean[c]) / std[c],
 * each step fp32 in that order, `* scale` skipped when scale == 1, `/ std` when has_std == 0 (RossTransformer:
 * swap {3,2,1}, scale 255, Ross' BGR means, no std; ImagenetTransformer: swap {1,2,3}, scale 1, mean + std;
 * model_utils.lua:138-155).                                                                                  */
typedef struct mpn_image_transform {
  int32_t swap[3];   /* 1-based source channel of each output channel */
  float scale;
  float mean[3];
  float std[3];
  int32_t has_std;
} mpn_image_transform;
/* host-only (no GPU): the size getImages scales a H0 x W0 image to for the single test scale (`scale`, `max_size` as
 * ImageDetect.lua:17-18) and the im_scale it returns: im_scale = scale / min side, capped so that
 * round(im_scale * max side) <= max_size; h = trunc(H0 * im_scale), w = trunc(W0 * im_scale) (:31-39). */
int mpn_get_images_size(int32_t H0, int32_t W0, double scale, double max_size, int32_t *h, int32_t *w, double *im_scale);
/* transformer + image.scale(im, w, h) ('bilinear', the third-party `image` package: parity unpinned, see
 * csrc/image_scale.cuh) in one kernel. im: 3 x H0 x W0 fp32 RGB in [0,1] (loaders/loader.lua:79), out: 3 x h x w.
 * Host buffers, synchronous; _dev: device buffers, stream-ordered. */
int mpn_get_images(mpn_ctx *ctx, const float *im, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                   int32_t h, int32_t w, float *out);
int mpn_get_images_dev(mpn_ctx *ctx, const float *im_dev, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                       int32_t h, int32_t w, float *out_dev);
/* Same from the decoder's bytes: im_hwc H0 x W0 x 3 uint8, interleaved RGB; the sample value is byte / 255 in fp32 (what
 * image.load(path, 3, 'float') hands to the transformer): a quarter of the bytes to move over the bus. */
int mpn_get_images_u8(mpn_ctx *ctx, const uint8_t *im_hwc, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                      int32_t h, int32_t w, float *out);
int mpn_get_images_u8_dev(mpn_ctx *ctx, const uint8_t *im_hwc_dev, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                          int32_t h, int32_t w, float *out_dev);
/* BatchProviderBase:getImages' image (BatchProviderBase.lua:15-21): transformer, image.hflip when flip != 0, then
 * image.scale to h x w; flip = 0 is mpn_get_images_u8. Host buffers, synchronous; _dev: device buffers, stream-ordered. */
int mpn_get_images_u8_flip(mpn_ctx *ctx, const uint8_t *im_hwc, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                           int32_t h, int32_t w, int32_t flip, float *out);
int mpn_get_images_u8_flip_dev(mpn_ctx *ctx, const uint8_t *im_hwc_dev, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                               int32_t h, int32_t w, int32_t flip, float *out_dev);
/* getImages + model:get(1):forward: uploads the RAW image (host), transforms and scales it on the device into the
 * model's image buffer and runs the trunk; *im_scale, *h, *w as mpn_get_images_size. Follow with mpn_model_detect(...,
 * image = NULL, recompute_features = 0) on the cached features. */
int mpn_model_trunk_image(mpn_model *m, const float *im, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                          double scale, double max_size, double *im_scale, int32_t *h, int32_t *w);
/* modules 2..n on cached trunk features (recompute_features=false path,
 * ImageDetect.lua:109-124): rois R x 5 in scaled-image coords. Outputs are the
 * RAW network outputs: cls R x C (logits, or probabilities if no_softmax) and
 * bbox R x 4C (after BBoxNorm if present) = what model:forward returns.      */
int mpn_model_heads(mpn_model *m, const float *rois, int64_t R, float *cls_out, float *bbox_out);
int mpn_model_heads_dev(mpn_model *m, const float *rois_dev, int64_t R, float *cls_out_dev,
                        float *bbox_out_dev);

/* ImageDetect:detect (ImageDetect.lua:156-193) after getImages: trunk (if
 * recompute_features) + heads + convertFrom per class with the ORIGINAL boxes +
 * softmax unless no_softmax. boxes R x 4 original-image coords, im_scale from
 * getImages. scores R x C, bboxes R x 4C (host, synchronous).                */
int mpn_model_detect(mpn_model *m, const float *image, int32_t H, int32_t W, const float *boxes,
                     int64_t R, float im_scale, int32_t recompute_features, float *scores,
                     float *bboxes);
/* detect + Tester_FRCNN:testOne post-processing (Tester_FRCNN.lua:75-78,106-117)
 * in one stream-ordered pass: clamp to [1,W0]x[1,H0], per foreground class
 * gather [box,score] rows with score > score_thresh, NMS at nms_thr.
 * keep_idx: (C-1) x R int32 (row indices into the R proposals, selection order),
 * keep_counts: C-1. scores/bboxes as mpn_model_detect but bboxes are clamped.
 * All pointers host; any of scores/bboxes may be NULL to skip that copy.     */
int mpn_model_detect_nms(mpn_model *m, const float *image, int32_t H, int32_t W,
                         const float *boxes, int64_t R, float im_scale, float W0, float H0,
                         float score_thresh, float nms_thr, float *scores, float *bboxes,
                         int32_t *keep_idx, int32_t *keep_counts);
/* Pipelined form of mpn_model_detect_nms for throughput serving (test_runner.lua keeps one
 * image in flight per donkey thread; here one model keeps two): submit returns at once with a
 * ticket, at most 2 tickets may be outstanding. The host->device copy of a submission runs on
 * its own copy stream and overlaps the kernels of the previous submission, the device->host
 * copy of the results on a third stream. The caller's buffers (pinned memory for real overlap)
 * must stay valid and untouched until mpn_model_detect_nms_wait(ticket) returns; results are
 * bit-identical to the synchronous call.                                       */
int mpn_model_detect_nms_submit(mpn_model *m, const float *image, int32_t H, int32_t W,
                                const float *boxes, int64_t R, float im_scale, float W0, float H0,
                                float score_thresh, float nms_thr, float *scores, float *bboxes,
                                int32_t *keep_idx, int32_t *keep_counts, int32_t *ticket);
/* The same pipeline fed with the RAW image as the decoder leaves it (H0 x W0 x 3 uint8, interleaved RGB): getImages
 * (ImageDetect.lua:22-52: transformer, im_scale rule for `scale` / `max_size`, image.scale) runs on the device in front
 * of the trunk, boxes are original-image coordinates, the clamp is to the original W0 x H0. 0.9 MB cross the bus for a
 * 480 x 640 image instead of the 5.8 MB of its scaled fp32 form. Same ticket protocol as mpn_model_detect_nms_submit. */
int mpn_model_detect_nms_submit_u8(mpn_model *m, const uint8_t *im_hwc, int32_t H0, int32_t W0,
                                   const mpn_image_transform *tf, double scale, double max_size, const float *boxes,
                                   int64_t R, float score_thresh, float nms_thr, float *scores, float *bboxes,
                                   int32_t *keep_idx, int32_t *keep_counts, int32_t *ticket);
int mpn_model_detect_nms_wait(mpn_model *m, int32_t ticket);
/* Tester_FRCNN:testOne with its test-time options (Tester_FRCNN.lua:54-139) in one stream-ordered pass, nothing but the
 * inputs and the final results crossing the bus: pass 1 = detect on the proposals, clamped to the image (:72-78); passes
 * 2..num_iter = detect on nn.SelectBoxes of the previous pass (:82-89; cached trunk features, not clamped, as the
 * reference); use_rbox_scores: the scores of pass i + 1 with the boxes of pass i (:91-97); the joined rows (:99-100,
 * n_out = R * (num_iter - use_rbox_scores)) are gathered per class with score > score_thresh and NMS'ed (:106-117);
 * bbox_voting: utils.bbox_vote of every kept box over its class's gathered rows, scores raised to vote_score_pow
 * (:118-124; 1 = untouched; other powers use the device powf, not libm's).
 * Outputs (host, synchronous; any may be NULL): scores n_out x C, bboxes n_out x 4C (the joined raw outputs :138),
 * keep_idx (C-1) x n_out rows into them in emission order, keep_counts C-1, voted (C-1) x n_out x 5 (row i of class j =
 * the voted box of keep_idx[j][i]; required when bbox_voting).                                                      */
typedef struct mpn_test_opts {
  int32_t num_iter;          /* opt.test_num_iterative_loc (>= 1) */
  int32_t use_rbox_scores;   /* opt.test_use_rbox_scores */
  int32_t bbox_voting;       /* opt.test_bbox_voting */
  float score_thresh;        /* Tester.thresh (-1.5, Tester_FRCNN.lua:50) */
  float nms_thr;             /* opt.test_nms_threshold (0.3) */
  float vote_thr;            /* opt.test_bbox_voting_nms_threshold (0.5) */
  float vote_score_pow;      /* opt.test_bbox_voting_score_pow (1) */
} mpn_test_opts;
int mpn_model_test_one(mpn_model *m, const float *image, int32_t H, int32_t W, const float *boxes, int64_t R,
                       float im_scale, float W0, float H0, const mpn_test_opts *opts, float *scores, float *bboxes,
                       int32_t *keep_idx, int32_t *keep_counts, float *voted);
/* Same with every buffer resident on the device, fully asynchronous (the
 * throughput path: bench.py `value`). */
int mpn_model_detect_nms_dev(mpn_model *m, const float *image_dev, int32_t H, int32_t W,
                             const float *boxes_dev, int64_t R, float im_scale, float W0, float H0,
                             float score_thresh, float nms_thr, float *scores_dev,
                             float *bboxes_dev, int32_t *keep_idx_dev, int32_t *keep_counts_dev);

/* ---- the detect tail after the network for a RANGE of classes (BASELINE configs[4], "NMS + BBoxNorm sweep": classes
 * shard across GPUs): nn.BBoxNorm (modules/BBoxNorm.lua:18-32; mean4 / std4 NULL = none) + utils.convertFrom per class
 * block (utils.lua:226-246) + clamp to [1,W0] x [1,H0] (Tester_FRCNN.lua:75-78) of deltas R x 4C against boxes R x 4
 * -> bboxes R x 4C, then for the foreground classes c in [c_begin, c_end) (1 <= c < C): rows with scores[:, c] >
 * score_thresh gathered and NMS'ed (Tester_FRCNN.lua:106-117). keep_idx (c_end - c_begin) x R proposal rows in emission
 * order, keep_counts c_end - c_begin. Device buffers, stream-ordered.                                              */
int mpn_post_detect_dev(mpn_ctx *ctx, const float *scores_dev, const float *deltas_dev, const float *boxes_dev, int64_t R,
                        int32_t C, const float *mean4, const float *std4, float W0, float H0, float score_thresh,
                        float nms_thr, int32_t c_begin, int32_t c_end, float *bboxes_dev, int32_t *keep_idx_dev,
                        int32_t *keep_counts_dev);

/* ---- after NMS, on the device (SURVEY 8f-2/3, 8e) --------------------------------------------------------------
 * Detection record of one image = the result of utils.keep_top_k (utils.lua:75-96; Tester:keepTopKPerImage,
 * Tester_FRCNN.lua:163-168, test_runner.lua:121) over the image's per-class NMS output, in a fixed size so that the
 * end-of-run all-gather needs no size exchange: MPN_REC_FLOATS floats = [count, MPN_MAX_DET x (x1,y1,x2,y2,score,class)],
 * class = 1-based foreground class (the index of the reference's per-class table), rows class-major and in NMS
 * emission order inside a class (= the reference's tables after keep_top_k), unused rows zero. keep_top_k keeps every
 * row with score >= the top_k-th largest score, so ties at the cut make count exceed top_k; count > MPN_MAX_DET means
 * the record overflowed (rows beyond MPN_MAX_DET are dropped; the host mirrors raise).                              */
enum { MPN_MAX_DET = 128, MPN_REC_FLOATS = 769, MPN_DIST_ID_BYTES = 128 };
/* scores R x C, bboxes R x 4C (detect outputs), keep_idx (C-1) x cap proposal rows in emission order, keep_counts C-1
 * (the outputs of mpn_model_detect_nms*, cap = R there). Device buffers, stream-ordered; host form synchronous.   */
int mpn_pack_detections_dev(mpn_ctx *ctx, const float *scores_dev, const float *bboxes_dev, int64_t R, int32_t C,
                            const int32_t *keep_idx_dev, const int32_t *keep_counts_dev, int64_t cap, int32_t top_k,
                            float *record_dev);
int mpn_pack_detections(mpn_ctx *ctx, const float *scores, const float *bboxes, int64_t R, int32_t C,
                        const int32_t *keep_idx, const int32_t *keep_counts, int64_t cap, int32_t top_k, float *record);
/* nn.SelectBoxes:updateOutput (modules/SelectBoxes.lua:26-56; Tester_FRCNN.lua:82-90): out[r] = the 4 box values of
 * the class with the largest score in row r (first maximum, background included), * std4 + mean4 when both are given
 * (NULL, NULL: the "dry run" of SelectBoxes.lua:46-47). classes R x C, ys R x 4C, out R x 4.                      */
int mpn_select_boxes(mpn_ctx *ctx, const float *classes, const float *ys, int64_t R, int32_t C, const float *mean4,
                     const float *std4, float *out);
int mpn_select_boxes_dev(mpn_ctx *ctx, const float *classes_dev, const float *ys_dev, int64_t R, int32_t C,
                         const float *mean4, const float *std4, float *out_dev);
/* From now on every mpn_model_detect_nms / _dev / _submit call also packs the image's record (top_k, normally 100)
 * into records_dev[n * MPN_REC_FLOATS], n = 0, 1, ... (stream-ordered, one extra launch per image); the call fails
 * once `capacity` records were written. records_dev = NULL switches the sink off; setting it resets the count.      */
int mpn_model_set_detection_sink(mpn_model *m, float *records_dev, int64_t capacity, int32_t top_k);
int mpn_model_detection_sink_count(const mpn_model *m, int64_t *n_records);

/* ---- the path's ONE collective (SURVEY 8e; test_runner.lua:96-103,121-122 joins the per-image results of all
 * replicas): an NCCL all-gather of the packed records, issued by the library on the ctx stream. One process (or
 * thread) per GPU: rank 0 calls mpn_dist_unique_id and hands the MPN_DIST_ID_BYTES bytes to every rank by whatever
 * channel the host has (torch.distributed / a file / threads' shared memory), then every rank calls mpn_dist_init
 * concurrently. NCCL is bound at run time (the libnccl.so.2 already in the process, else the system one); without
 * it these calls fail with a message and nothing else is affected. A ctx without a communicator is a world of 1.    */
int mpn_dist_unique_id(mpn_ctx *ctx, uint8_t *id);
int mpn_dist_init(mpn_ctx *ctx, const uint8_t *id, int32_t rank, int32_t world);
int mpn_dist_world(const mpn_ctx *ctx, int32_t *rank, int32_t *world);
/* recv = world x n_floats, rank-major; every rank contributes n_floats (its records, padded to the same count).
 * _dev: device buffers, stream-ordered (send may alias its own slot of recv). Host form: recv_host, synchronous.    */
int mpn_dist_all_gather_dev(mpn_ctx *ctx, const float *send_dev, int64_t n_floats, float *recv_dev);
int mpn_dist_all_gather(mpn_ctx *ctx, const float *send_dev, int64_t n_floats, float *recv_host);
int mpn_dist_destroy(mpn_ctx *ctx);
int mpn_dist_nccl_version(mpn_ctx *ctx, int32_t *version);

/* ---- the score: replaces testCoco/coco.lua:24-38 (Coco:evaluate -> pycocotools COCOeval(cocoGt, cocoGt.loadRes(res)),
 * iouType 'bbox', default Params, params.imgIds = the sorted distinct image ids of the rows; testCoco/init.lua:30-88).
 * Ground truth: image_ids[n_images] and cat_ids[n_cats] ascending and unique (the GT images and categories; categories are
 * the K axis of the outputs); G annotations with gt_img / gt_cat = 0-based indices into those tables, gt_box G x 4
 * (x, y, w, h), gt_area (the json "area" field), gt_crowd in {0, 1} (= "ignore"), in the json's annotation order.
 * dets: D x 7 float rows [image_id, x, y, w, h, score, category_id] (the tensor testCoco/init.lua:65-86 builds); ids are
 * truncated to integers; a row of an unknown category is not scored but still puts its image into the evaluated set.
 * Outputs (host): precision [10][101][n_cats][4][3] and recall [10][n_cats][4][3] = pycocotools' eval['precision'] /
 * eval['recall'] (IoU thresholds .5:.05:.95, recall points 0:.01:1, area ranges all / small / medium / large, maxDets
 * 1 / 10 / 100; -1 where a (category, area) has no non-ignored annotation), stats[12] = COCOeval.stats. Synchronous,
 * deterministic (two calls give the same bits). MPN_ERR_ARG (with a message): D < 1, a NaN / infinite row value, a row
 * whose image is not a GT image, an id table not ascending, a GT index out of range, iscrowd not 0 / 1, a non-finite
 * GT box or area. Rules and the pycocotools quirks they keep: DESIGN 4.                                             */
int mpn_coco_eval(mpn_ctx *ctx, int32_t n_images, const int64_t *image_ids, int32_t n_cats, const int64_t *cat_ids,
                  int64_t G, const int32_t *gt_img, const int32_t *gt_cat, const double *gt_box, const double *gt_area,
                  const int32_t *gt_crowd, int64_t D, const float *dets, double *precision, double *recall,
                  double *stats);

/* introspection for tests: rows [r0, r0 + n) of the pooled tensor the LAST heads / detect call fed to tower `tower` —
 * the output of the fused Foveal + ROI pooling (+ per-level L2 normalise x 1000) kernel on the product path — as fp32
 * n x (PH*PW) x Ctot (channels-last, levels concatenated along channels; value = hi + lo of the split planes).
 * out may be NULL to query *R_total / *bins / *Ctot only. Host buffer, synchronous.                                 */
int mpn_model_get_pooled(mpn_model *m, int32_t tower, int64_t r0, int64_t n, float *out, int64_t capacity,
                         int64_t *R_total, int32_t *bins, int32_t *Ctot);
/* introspection for tests/profiling: copy a trunk slot to host as N x C x H x W fp32 */
int mpn_model_get_trunk_slot(mpn_model *m, int32_t slot, float *out_nchw, int64_t capacity,
                             int32_t *C, int32_t *H, int32_t *W);
/* test hook: slot `slot` of the last trunk pass (tower = -1; rows are images, r0 = 0, n = 1) or of tower `tower` of the
 * last heads pass (rows are ROIs) as raw 16-bit planes, NHWC dense: hi / lo n x H x W x C (a concat column slice is
 * returned without its row stride); *fmt = 0 bf16 / 1 fp16; dims[4] = {N_total, H, W, C}. q8 / e8 may be NULL;
 * otherwise they receive the slot's e4m3 plane (n x H x W x C) and per-sample exponents (n) from the last pass, and the
 * call fails with MPN_ERR_ARG if the current plan keeps no e4m3 plane for the slot. Also MPN_ERR_ARG: a slot elided by
 * the conv+pool fusion, an unknown slot / tower, no pass yet, rows out of range, capacity (elements) too small.
 * hi == NULL: dims / fmt only. Host buffers, synchronous.                                                            */
int mpn_model_get_slot_planes(mpn_model *m, int32_t tower, int32_t slot, int64_t r0, int64_t n, uint16_t *hi,
                              uint16_t *lo, uint8_t *q8, int32_t *e8, int64_t capacity, int32_t *fmt, int64_t *dims);
/* test hook: the raw head outputs of the last heads pass: cls K x R x C logits (before softmax / mean), bbox R x 4C.
 * detect, detect_nms and test_one leave bbox before BBoxNorm (test_one: its last pass); heads / heads_dev apply
 * BBoxNorm to it in place. NULL pointers: *R / *K only. Host buffers, synchronous.                                    */
int mpn_model_get_head_outputs(mpn_model *m, float *cls_logits, float *bbox_raw, int64_t *R, int32_t *K);
/* test hook: the detect tail kernel after the heads, launched as every detect pass launches it: logits K x R x C -> scores
 * R x C (softmax of head 0, or the mean of the K softmaxes; do_softmax = 0 copies head 0 and needs K = 1), and deltas
 * R x 4C against boxes R x 4 -> bboxes R x 4C (nn.BBoxNorm y * std4 + mean4 when has_norm, convertFrom, clamp to
 * [1, W0] x [1, H0] when do_clamp). mean4 / std4 may be NULL without has_norm. Host buffers, synchronous.          */
int mpn_debug_detect_tail(mpn_ctx *ctx, const float *logits, int32_t K, int64_t R, int32_t C, int32_t do_softmax, const float *deltas,
                          const float *boxes, int32_t do_clamp, float W0, float H0, int32_t has_norm, const float *mean4,
                          const float *std4, float *scores, float *bboxes);
/* select conv/GEMM implementation: 0 = wgmma tensor-core path (default, product),
 * 1 = plain fp32 CUDA-core check kernel (debug/verification only, very slow),
 * 2 = wgmma path with the conv -> 2x2 max-pool epilogue fusion disabled, so every trunk slot is
 *     materialised (mpn_model_get_trunk_slot fails loudly for a slot the fusion elided). */
int mpn_model_set_conv_impl(mpn_model *m, int32_t impl);
/* algorithmic FLOPs of the last trunk / heads call (SURVEY 8d definition)    */
int mpn_model_last_flops(const mpn_model *m, double *trunk_flops, double *head_flops);

/* standalone GEMM check entry (tests): C[M,N] = A[M,K] * B[N,K]^T + bias, fp32 host
 * buffers, computed with the same split-bf16 wgmma kernel the model uses (impl 0), the CUDA-core fp32 check kernel
 * (impl 1), or the fp16-weight two-product kernels of fc6 / fc7 (impl 2; needs N >= 1024).  */
int mpn_gemm_check(mpn_ctx *ctx, const float *A, const float *B, const float *bias, int64_t M,
                   int64_t N, int64_t K, int32_t relu, int32_t impl, float *C);
/* engine microbenchmark (diagnostics): times `iters` back-to-back launches of the wgmma engine on
 * device-resident random operands, C[M,N] = A[M,K] * B[N,K]^T, returns the mean milliseconds per launch and the chosen
 * configuration (BN, CTA group = 1, split-K). */
int mpn_gemm_bench(mpn_ctx *ctx, int64_t M, int64_t N, int64_t K, int32_t iters, double *ms_per_launch,
                   int32_t *bn, int32_t *cta_group, int32_t *splitk);
/* conv microbenchmark: mean milliseconds per launch and the chosen configuration. dbg16 (may be NULL) is zero-filled:
 * the wgmma engine keeps no pipeline-wait counters. *cta_group is always 1; *mode: bit 0 = 16 x 8 patches (3x3 / stride 1). */
int mpn_conv_bench(mpn_ctx *ctx, int64_t N, int64_t Cin, int64_t H, int64_t W, int64_t Cout, int32_t k, int32_t stride,
                   int32_t pad, int32_t iters, double *ms_per_launch, int32_t *bn, int32_t *cta_group, int32_t *mode,
                   uint64_t *dbg16);
/* host-only view of the planner (no GPU): the engine configuration chosen for a conv / Linear layer (Cin multiple of 8) on
 * a device with sm_count SMs; per_roi = 1 for per-ROI layers (rounding-relevant choices from (Cout, K) only).
 * out[8] = {mode (bit 0: 16 x 8 patches of a 3x3 / stride 1 conv), CTA group (1), N tile, split-K, stream-K (0), patch tn, th, tw}. */
int mpn_debug_plan(int64_t N, int64_t Cin, int64_t H, int64_t W, int64_t Cout, int32_t k, int32_t stride, int32_t pad,
                   int32_t per_roi, int32_t sm_count, int32_t *out);
/* host-only view of the fp8 operand rule (no GPU), the code the device quantizers run: h = n_samples x sample_elems values,
 * per sample e_out = the scale exponent of max |h|, q_out = the e4m3 codes of 2^e * h. MPN_ERR_ARG: a sample without a scale. */
int mpn_debug_fp8(const float *h, int64_t n_samples, int64_t sample_elems, int32_t *e_out, uint8_t *q_out);
/* standalone conv check entry (tests): x N x Cin x H x W, w Cout x Cin x kh x kw (Torch layouts) */
int mpn_conv_check(mpn_ctx *ctx, const float *x, int64_t N, int64_t Cin, int64_t H, int64_t W,
                   const float *w, const float *bias, int64_t Cout, int32_t kh, int32_t kw,
                   int32_t stride, int32_t pad, int32_t relu, int32_t impl, float *y);
/* mpn_conv_check on an input view (impl 0 or 1): x's Cin channels are the first of split planes with pixel stride ld
 * (ld >= Cin, a multiple of 8) whose channels [Cin, ld) hold NaN. The engine must not read them: a K block past Cin is the
 * TMA's zero fill, so the output equals mpn_conv_check's bit for bit. */
int mpn_conv_check_view(mpn_ctx *ctx, const float *x, int64_t N, int64_t Cin, int64_t H, int64_t W, int64_t ld,
                        const float *w, const float *bias, int64_t Cout, int32_t kh, int32_t kw,
                        int32_t stride, int32_t pad, int32_t relu, int32_t impl, float *y);

/* ---- training: one SGD step (train.lua:221-370; csrc/train.cu, DESIGN 3.4) -------------------------------------------
 * A step runs the trunk per image, pools image i's ROIs into rows [off_i, off_i + R_i) of one per-ROI batch, runs towers
 * and heads in training mode (nn.Dropout after the ReLU of every per-ROI Linear, BF16X3 numerics whatever fc_w16 says,
 * raw logits and raw deltas), the criteria CrossEntropy + bbox_regression x BBoxRegression, the backward GEMMs on the
 * wgmma engine, and optim.sgd once per tensor. Every inference entry of the model uses the updated weights afterwards.
 * What trains is an mpn_train_spec (below). A step refuses (MPN_ERR_ARG) labels outside 1..C, R = 0 or R > max_rois and
 * images beyond max_h x max_w. */
typedef struct mpn_train_config {
  float lr, momentum, dampening, weight_decay;   /* optim.sgd; weight decay is 0 for biases (Optim.lua:50-51)            */
  float dropout;                                  /* nn.Dropout p; 0 = train_remove_dropouts                             */
  float bbox_regression;                          /* weight of the bbox criterion                                        */
  uint64_t seed;                                  /* dropout masks: Philox4x32-10 over (seed, step, tower, layer, element) */
} mpn_train_config;
/* What a training trains, and under which rules. The per-ROI layers and the heads always train: the per-ROI layers must
 * be 1x1 convolutions, FLATTENs or Linears (a recorded layer below aside), no parameter tensor may be shared between
 * layers, and the class and bbox heads read the same or disjoint columns.
 *  trunk_from  0: the trunk is frozen (MultiPathNet's sits under nn.NoBackprop). k > 0: the trunk range k .. n-1 trains
 *              too (vgg.lua:18-19 freezes conv1_1 .. pool2: k = 6 for vgg16_fast_rcnn). The step keeps each image's
 *              trunk slots from layer k's input upward, and runs the trunk backward per image: ROI pooling (gather at
 *              the forward's argmax), the 2x2 max pools (the window's first maximum on the stored planes), ReLU gates,
 *              and for every trained 3x3 convolution dgrad (a 3x3 convolution of the gradient with the weight rotated
 *              by 180 degrees; skipped for the lowest trained one) and wgrad (one GEMM over the minibatch's pixels) on
 *              the wgmma engine. Refused: k out of range (1 <= k < n); a trained layer other than a 3x3 / stride 1 /
 *              pad 1 convolution with ReLU and no residual or a 2x2 / stride 2 / pad 0 max pool; without phase 2, more
 *              than one tower, or a tower that pools from anything but the last trunk layer's output alone, or whose
 *              first layer is not a FLATTEN followed by a Linear.
 *  phase2      1: MultiPathNet's two phases (multipathnet.lua:123-124, utils.vggSetPhase2_outer, train.lua:239-269).
 *              The trunk range trains only from mpn_model_train_phase2 on; until then the steps and bits are those of
 *              trunk_from = 0, but the range's fp32 masters are kept. It then trains through every tower's ROI pooling
 *              backward (foveal regions, several levels, the per-(ROI, level) L2 normalisation x 1000) and the graph
 *              backward. Refused: trunk_from 0; fixed-batch-norm records; the range's layer rules above; a tower level
 *              that pools a slot no trained layer writes; more than 8 levels on one slot; a tower whose first layer
 *              is not a convolution of the pooled map or a FLATTEN and a Linear, or another of whose layers reads the
 *              pooled map.
 *  integral    1: an integral model (K >= 1 class heads over the same columns and of the same width,
 *              model_utils.integral) trains the integral loss: a step trains one selected head k
 *              (mpn_model_train_select_head; head 0 by default) as train.lua's nn.SelectTable does. Only head k's
 *              logits reach the criteria and the outputs hook, head k gets dW / db and the dX into the concat, the
 *              other heads' gradients are zero and they still take optim.sgd's step with a zero gradient (w -= lr *
 *              momentum buffer, weight decay included). 0: K > 1 class heads are refused. Refused: class heads that
 *              differ in columns or width.
 *  n_fixed, fixed_weight, fixed_scale
 *              fixed batch norm (resnet.lua's BNtoFixed: inn.ConstAffine y = a[c] * x + b[c] after a bias-free
 *              convolution W). The description holds the folded layer, W' = a * W with bias b. fixed_weight[0 ..
 *              n_fixed-1] name the convolutions (weight-table indices) that carry such a record, fixed_scale[j] (host,
 *              Cout floats, copied at begin) its a. A recorded layer may be a k x k convolution, k in {1, 3}, stride 1
 *              or 2, pad (k - 1) / 2, Cout a multiple of 64, with or without ReLU and residual, per ROI or in the
 *              trained trunk range, whose layers may then form a graph; a tower holding one has no FLATTEN and ends in
 *              a global AVGPOOL that the heads read. It trains W with a and b constant: the step computes g' = dL/dW'
 *              and optim.sgd runs on W' with g' scaled by a^2 per output channel (buf' = a * buf exactly in real
 *              arithmetic), so mpn_model_train_get reports W', g' and buf'. A recorded layer's bias is the constant b:
 *              no gradient, no momentum buffer, no update. Layers without a record follow the rules above. Refused: n <
 *              0; a record that names no convolution, or one twice; a recorded layer outside the shapes above.
 * The rules run in this order and the first refusal is reported: phase 2 with records, the records, the trunk range,
 * the per-ROI layers and heads.                                                                                     */
typedef struct mpn_train_spec {
  int32_t trunk_from;               /* first trained trunk layer; 0: the trunk is frozen                                */
  int32_t phase2;                   /* 1: layers trunk_from .. are kept but idle until mpn_model_train_phase2           */
  int32_t integral;                 /* 1: K >= 1 class heads over the same columns train the integral loss              */
  int32_t n_fixed;                  /* fixed batch norm: n_fixed recorded convolutions (0: none)                        */
  const int32_t *fixed_weight;      /* their weight-table indices                                                       */
  const float *const *fixed_scale;  /* per record, Cout floats of a; read by begin only (check may pass NULL)           */
} mpn_train_spec;
/* The optim method of every trained tensor (train.lua's `method` and `learningRateDecay`, engines/Optim.lua:46-81; as
 * recalled, parity unpinned; the op order is csrc/train_rule.cuh's). t = the steps done before a step (mpn_train_state.
 * step, the same for every tensor), T = t + 1, clr = lr / (1 + t * lr_decay), g = the gradient + weight_decay * w (0 for
 * biases):
 *   sgd      the mpn_train_config rule with clr for lr (lr_decay 0: clr = lr exactly); state: the momentum buffer
 *   adam     m = b1 m + (1 - b1) g; v = b2 v + (1 - b2) g g; w -= clr sqrt(1 - b2^T) / (1 - b1^T) * m / (sqrt(v) + eps)
 *   adamax   m = b1 m + (1 - b1) g; u = max(b2 u, |g| + eps); w -= lr / (1 - b1^T) * m / u          (lr_decay ignored)
 *   adagrad  s += g g; w -= clr * g / (sqrt(s) + 1e-10)                                             (epsilon ignored)
 *   rmsprop  m = alpha m + (1 - alpha) g g; w -= lr * g / (sqrt(m) + eps)                           (lr_decay ignored)
 * momentum and dampening apply to sgd only. States start at 0. A phase-2 trunk tensor joins at the switch with zero
 * state and the global t. A fixed-batch-norm weight keeps sgd's a^2 rule; the other methods keep their state in the
 * space of W: g_W = a g', W = W' / a, W' -= a * (the step of W); a scale of 0 is refused. Refused (mpn_train_check_optim):
 * a method out of range, beta1 or beta2 outside [0, 1), alpha outside [0, 1], a negative or non-finite epsilon or
 * lr_decay.                                                                                                            */
enum { MPN_OPTIM_SGD = 0, MPN_OPTIM_ADAM = 1, MPN_OPTIM_ADAMAX = 2, MPN_OPTIM_ADAGRAD = 3, MPN_OPTIM_RMSPROP = 4 };
typedef struct mpn_train_optim {
  int32_t method;                           /* MPN_OPTIM_*                                                              */
  double lr_decay, beta1, beta2, epsilon, alpha;
} mpn_train_optim;
/* host-only (no GPU): MPN_OK if the description can train under s with optim o (NULL: optim.sgd, lr_decay 0), else
 * MPN_ERR_ARG and the reason in msg (none for a NULL d or s). o is checked first. mpn_train_check is o = NULL.          */
int mpn_train_check_optim(const mpn_model_desc *d, const mpn_train_spec *s, const mpn_train_optim *o, char *msg, int32_t msg_cap);
int mpn_train_check(const mpn_model_desc *d, const mpn_train_spec *s, char *msg, int32_t msg_cap);
/* start training under s and o (NULL: optim.sgd, lr_decay 0): the checks of mpn_train_check_optim, then the fp32
 * weights of the trained tensors (and of an idle phase-2 range) are kept as masters, with a gradient and the method's
 * state each (a second state tensor for adam / adamax only). Must come before the model's first heads / detect call
 * (those release the fp32 copies), and with a trunk range before its first trunk call too (the trunk plan releases the
 * trunk's copies). Refused besides: a trained layer that reads a K tail; a config out of range; the "bf16" / "fp8"
 * options. The "train_bf16" option is read here. mpn_model_train_begin is o = NULL.                                    */
int mpn_model_train_begin_optim(mpn_model *m, const mpn_train_config *cfg, const mpn_train_spec *s, const mpn_train_optim *o);
int mpn_model_train_begin(mpn_model *m, const mpn_train_config *cfg, const mpn_train_spec *s);
/* one step. images: n_images transformed 3 x H_i x W_i fp32 images (image_hw: H_i, W_i pairs); boxes: R x 4 ROIs in
 * scaled-image coordinates (1-based, as the heads take them), image 0's rows first; labels: R int32 in 1..C; bbox_targets:
 * R x 4C normalised targets. losses[3] = {total, cross entropy, bbox (before its weight)}. Synchronous.                */
int mpn_model_train_step(mpn_model *m, int32_t n_images, const float *const *images, const int32_t *image_hw,
                         const int32_t *rois_per_image, const float *boxes, const int32_t *labels, const float *bbox_targets,
                         float *losses);
/* the same on device buffers (images_dev: a host array of device pointers; losses_dev: 3 floats on the device),
 * stream-ordered. A label outside 1..C zeroes its row's gradient and fails the next host-synchronous call.
 * After a step the model holds no cached trunk features: heads / detect without recompute need a new trunk call first. */
int mpn_model_train_step_dev(mpn_model *m, int32_t n_images, const float *const *images_dev, const int32_t *image_hw,
                             const int32_t *rois_per_image, const float *boxes_dev, const int32_t *labels_dev,
                             const float *bbox_targets_dev, float *losses_dev);
/* device time of the last step's phases (CUDA events on the ctx's stream, waits for the step): ms[4] = {trunks + ROI
 * pooling, per-ROI forward + criteria, backward, update}                                                              */
int mpn_model_train_phase_ms(mpn_model *m, float *ms);
/* the class head (0 .. K-1) the next steps train; MPN_ERR_ARG out of range                                            */
int mpn_model_train_select_head(mpn_model *m, int32_t k);
int mpn_model_train_set_lr(mpn_model *m, float lr);
/* train.lua's onEndEpoch: lr *= factor and, under sgd, every momentum buffer *= factor (the other methods' state is
 * not u.dfdx: only the rate changes)                                                                                  */
int mpn_model_train_decay(mpn_model *m, float factor);
/* a trained tensor (its index in the weight table) in Torch layout: what 0 = weight, 1 = gradient of the last step,
 * 2 = the method's first state (sgd's momentum buffer, adam's / adamax's / rmsprop's m, adagrad's s), 3 = its second
 * (adam's v, adamax's u; refused for the other methods). Host buffer, synchronous.                                     */
int mpn_model_train_get(mpn_model *m, int32_t weight, int32_t what, float *out, int64_t capacity);
/* test hook: the keep mask (R x cout bytes) the last step's dropout applied after layer `layer` of tower `tower`;
 * out NULL: *n_out only                                                                                                */
int mpn_model_train_dropout_mask(mpn_model *m, int32_t tower, int32_t layer, uint8_t *out, int64_t capacity, int64_t *n_out);
/* test hook: the gate the last step's backward took through the ReLU of layer `layer` of tower `tower` (1 where the stored
 * output, after dropout, is > 0), R x H x W x cout bytes; out NULL: *n_out only                                        */
int mpn_model_train_relu_gate(mpn_model *m, int32_t tower, int32_t layer, uint8_t *out, int64_t capacity, int64_t *n_out);
/* test hook: the last step's raw logits (R x C) and raw deltas (R x 4C), until the next inference call                 */
int mpn_model_train_outputs(mpn_model *m, float *cls_logits, float *bbox_deltas);
/* test hook (trunk training): image `image`'s stored activation of trunk slot `slot` from the last step, C x H x W fp32
 * (out NULL: the shape only); the slots kept are layer trunk_from's input and every slot written at or above it        */
int mpn_model_train_trunk_slot(mpn_model *m, int32_t image, int32_t slot, float *out_nchw, int64_t capacity, int32_t *C,
                               int32_t *H, int32_t *W);
/* test hooks of the trunk-training kernels on host buffers (synchronous). Split planes are the raw bf16 bits (hi, lo).
 * mpn_debug_roi_backward_nhwc: one image's H x W x C map and its R ROI rows (R x 5) with grad_out R x PH x PW x C fp32 ->
 *   grad H x W x C fp32: per (ROI, bin, channel) the first cell in (h, w) order whose hi + lo is > the running max, then a
 *   gather per cell from +0 in ascending roi, ph, pw.
 * mpn_debug_pool_backward: a convolution's stored output y (H x W x C) and the 2x2 / stride 2 ceil-mode pool output's
 *   gradient ((H + 1) / 2 x (W + 1) / 2 x C fp32) -> H x W x C fp32: the window's gradient at its first maximum in
 *   row-major order on hi + lo, gated by y > 0.
 * mpn_debug_conv_backward: a k x k / stride s / pad (k - 1) / 2 convolution, k in {1, 3}, s in {1, 2}, over n_images
 *   maps (image_hw pairs: the INPUT maps) stacked in order: inputs x (pixels x cin planes), gated output gradients g
 *   (output pixels x cout fp32), weight w (Torch cout x cin x k x k) -> dw (Torch layout, one GEMM over the tap matrix
 *   of all pixels) and dx (input pixels x cin fp32: a GEMM for 1x1 / 1, the rotated-weight convolution per map for
 *   3x3 / 1, GEMM + col2im for stride 2), as the training step's graph backward computes them.                        */
int mpn_debug_roi_backward_nhwc(mpn_ctx *ctx, const uint16_t *hi, const uint16_t *lo, int32_t H, int32_t W, int32_t C, const float *rois,
                                int64_t R, int32_t PW, int32_t PH, float scale, int32_t variant, const float *grad_out, float *grad);
int mpn_debug_pool_backward(mpn_ctx *ctx, const uint16_t *y_hi, const uint16_t *y_lo, int32_t H, int32_t W, int32_t C, const float *grad_pool,
                            float *grad);
int mpn_debug_conv_backward(mpn_ctx *ctx, int32_t n_images, const int32_t *image_hw, int32_t cin, int32_t cout, int32_t k, int32_t stride,
                            const uint16_t *x_hi, const uint16_t *x_lo, const float *g, const float *w, float *dw, float *dx);
/* stop training: frees gradients and momentum buffers; the model keeps the trained weights                            */
int mpn_model_train_end(mpn_model *m);
/* host-only views of the training rules (no GPU), the code the device runs: dropout keep bits of elements
 * elem0 .. elem0 + n - 1; both criteria on R rows (losses as in mpn_model_train_step); optim.sgd on n elements.        */
int mpn_debug_dropout(uint64_t seed, uint32_t step, int32_t tower, int32_t layer, uint64_t elem0, int64_t n, float p, uint8_t *out);
int mpn_debug_criteria(const float *x, const float *d, const int32_t *labels, const float *t, int64_t R, int32_t C, float bbox_w,
                       float *gx, float *gd, float *losses);
int mpn_debug_sgd(float *w, const float *g, float *buf, int64_t n, float lr, float momentum, float dampening, float wd, int32_t first);
/* host-only view of the update under optim o (NULL: sgd, lr_decay 0) on n elements: t steps done before this one, lr the
 * rate in force, wd the weight decay. s1 / s2 the method's states (s2 read for adam / adamax only); g NULL: the
 * no-gradient variant; a (NULL: none) a per-element fixed-batch-norm scale (sgd: the gradient times fl(a * a)).        */
int mpn_debug_optim(float *w, const float *g, float *s1, float *s2, const float *a, int64_t n, const mpn_train_optim *o, float lr,
                    float momentum, float dampening, float wd, int64_t t);

/* ---- training feed: DataSetJSON + BatchProviderROI (DataSetJSON.lua:101-390, BatchProviderROI.lua, BatchProviderBase.lua)
 * Images are 0-based here. A roidb holds every image's all_boxes (its GT rows first, then its proposals), the matching
 * (overlap, 1-based correspondance, label) per row and, per threshold set s (thresholds[3s .. 3s+2] = fg, bg_lo, bg_hi),
 * the bg rows (bg_lo <= overlap < bg_hi) and fg rows (overlap >= fg) of every image in row order.
 * mpn_roidb_create: per image i, annotations ann_off[i] .. ann_off[i+1]-1 (json bbox x y w h, json area, 1-based class id,
 *   flags bit 0 = crowd, bit 1 = difficult) and proposals prop_off[i] .. prop_off[i+1]-1 (x1 y1 x2 y2; scores may be NULL).
 *   Annotations with area > min_area are kept; GT = kept, not difficult, not crowd; crowds mask proposals. Proposals with
 *   (x2 - x1) * (y2 - y1) > min_proposal_area (0: no filter), then the best_number highest scores (stable order).
 *   Uploads the tables and runs the matching pass on the device; synchronous.                                          */
typedef struct mpn_roidb mpn_roidb;
int mpn_roidb_create(mpn_ctx *ctx, int32_t n_images, const int64_t *ann_off, const double *ann_xywh, const double *ann_area,
                     const int32_t *ann_class, const int32_t *ann_flags, double min_area, const int64_t *prop_off,
                     const float *prop_box, const float *prop_score, int32_t best_number, double min_proposal_area,
                     int32_t num_classes, int32_t n_sets, const float *thresholds, mpn_roidb **out);
void mpn_roidb_destroy(mpn_roidb *db);
/* counts[(s * 2 + kind) * n_images + i]: the bg (kind 0) / fg (kind 1) rows of image i in set s; *n_rows: all rows      */
int mpn_roidb_counts(mpn_roidb *db, int32_t *counts, int64_t *n_rows);
/* test hooks: image `image`'s all_boxes, overlap, correspondance and label rows (NULLs: the sizes only); its bg / fg
 * list in set `set` as row indices within the image                                                                      */
int mpn_roidb_image_rows(mpn_roidb *db, int32_t image, float *boxes, float *overlap, int32_t *corr, int32_t *label, int64_t capacity,
                         int64_t *n_rows, int32_t *n_gt);
int mpn_roidb_list(mpn_roidb *db, int32_t set, int32_t kind, int32_t image, int32_t *rows, int64_t capacity, int64_t *n_out);
/* setupData (BatchProviderROI.lua:53-69): convertTo(rois, gtboxes) of the fg rows of set `set` in images 0 .. n_first-1,
 * per coordinate the mean and the unbiased std (fixed-order double sums, rounded to fp32)                              */
int mpn_roidb_regression_stats(mpn_roidb *db, int32_t set, int32_t n_first, float *mean, float *std_);
/* host-only: permuteIdx's draws for n_slots images of one step from the per-image bg / fg counts of a set: the image each
 * slot trains on, the images its bg and fg rows come from (a kind found by an earlier draw of the slot stays) and its flip.
 * MPN_ERR_STATE when no image has a bg row or none has a fg row.                                                       */
int mpn_sample_plan(const int32_t *n_bg, const int32_t *n_fg, int32_t n_images, uint64_t seed, uint32_t step, int32_t set, int32_t n_slots,
                    int32_t *image, int32_t *bg_src, int32_t *fg_src, int32_t *flip);
/* host-only: the threshold set of an integral model's step, train.lua's `loaders[torch.random(#loaders)]` restated as
 * *set = rand_int(draw_u32(seed, step, slot 0, set 0, DRAW_INTEGRAL, draw 0), n_sets) - 1 (roidb_rule.cuh)             */
int mpn_integral_set(uint64_t seed, uint32_t step, int32_t n_sets, int32_t *set);
/* host-only: getImages' training size rule (BatchProviderBase.lua:23-41): im_scale = scale / min side, then per dim in
 * order divided down where that dim exceeds max_size; h, w truncated                                                   */
int mpn_train_images_size(int32_t H0, int32_t W0, double scale, double max_size, int32_t *h, int32_t *w, double *im_scale);
/* selectBBoxes + sample's targets for a plan, stream-ordered: per slot k, min(bg_each, n_bg) rows drawn with replacement
 * from bg_src[k]'s bg list, then min(fg_each, n_fg) from fg_src[k]'s fg list, scaled by im_scale[k] and flipped against
 * width[k]. Writes R x 4 boxes, R labels (1 = bg, 1 + class) and R x 4C targets, C = num_classes (dataset classes + 1),
 * in the layout mpn_model_train_step_dev reads; rois_per_image[k] (host) the rows of slot k.                           */
int mpn_roidb_sample_dev(mpn_roidb *db, int32_t set, uint64_t seed, uint32_t step, int32_t n_slots, const int32_t *bg_src,
                         const int32_t *fg_src, const int32_t *flip, const double *im_scale, const int32_t *width, int32_t bg_each,
                         int32_t fg_each, const float *mean, const float *std_, int32_t num_classes, float *boxes_dev,
                         int32_t *labels_dev, float *targets_dev, int32_t *rois_per_image);
/* the whole step's batch into buffers the roidb owns (valid until its next sample): plan rows (image, bg_src, fg_src, flip)
 * per slot, each slot's decoded H0 x W0 x 3 image (host) uploaded, flipped and scaled to image_hw (out), then
 * mpn_roidb_sample_dev. mpn_roidb_batch_host copies that batch back (NULL: skip); mpn_model_train_step_batch runs one
 * training step of m (on the roidb's ctx) on it, losses as mpn_model_train_step. Synchronous. For an integral model it
 * first selects the class head of the batch's set (MPN_ERR_ARG unless the roidb has one set per class head).             */
int mpn_roidb_sample(mpn_roidb *db, int32_t set, uint64_t seed, uint32_t step, int32_t n_slots, const int32_t *plan,
                     const uint8_t *const *images_hwc, const int32_t *hw0, const mpn_image_transform *tf, double scale, double max_size,
                     int32_t bg_each, int32_t fg_each, const float *mean, const float *std_, int32_t num_classes, int32_t *image_hw,
                     int32_t *rois_per_image);
int mpn_roidb_batch_host(mpn_roidb *db, float *const *images, float *boxes, int32_t *labels, float *targets);
int mpn_model_train_step_batch(mpn_model *m, mpn_roidb *db, float *losses);
/* host-only views of the rules, the code the device runs: one image's attachProposals from its raw annotations and
 * proposals (as mpn_roidb_create; NULL outputs: sizes only); the boxes and targets of given drawn rows (roi and gt box
 * unscaled, label 1 = bg)                                                                                              */
int mpn_debug_attach_proposals(int64_t n_ann, const double *ann_xywh, const double *ann_area, const int32_t *ann_class,
                               const int32_t *ann_flags, double min_area, int64_t n_prop, const float *prop_box, const float *prop_score,
                               int32_t best_number, double min_proposal_area, int32_t num_classes, float *boxes, float *overlap,
                               int32_t *corr, int32_t *label, int64_t capacity, int64_t *n_rows, int32_t *n_gt);
int mpn_debug_sample_rows(int64_t R, const float *rois, const float *gtboxes, const int32_t *labels, double im_scale, int32_t width,
                          int32_t flip, const float *mean, const float *std_, int32_t num_classes, float *boxes, float *targets);

/* ---- MultiPathNet's switch to phase 2 (train.lua:239-269) on a training begun with mpn_train_spec.phase2 = 1: from the
 * next step the trunk range trains (see mpn_train_spec). lr >= 0: the rate becomes lr and, under sgd, every momentum
 * buffer is zeroed (the other methods' state is kept); lr < 0 keeps both. The trunk tensors join with zero state and
 * the ordinary update.                                                                                                 */
int mpn_model_train_phase2(mpn_model *m, float lr);

/* ---- resuming a training (train.lua's checkpoint / resume, train.lua:188-235). mpn_model_train_set is the inverse of
 * mpn_model_train_get for what 0 (the fp32 master, Torch layout), 2 (the momentum buffer, or the method's first state)
 * and 3 (the second state of adam / adamax): the raw arrays, so a
 * fixed-batch-norm tensor takes W' and a * buf as _get gave them. Setting a master rewrites every plane derived from it
 * as the update of a step leaves them (the split planes, the W^T / rotated dgrad planes: the same kernel without the
 * step); planes an inference plan derived from it are rebuilt by the next plan. Synchronous.
 * mpn_train_state: the scalars of a training besides the tensors. step = steps done (the next step's dropout counter;
 * 0 = optim.sgd's first-step rule applies next), lr = the rate in force (fp32, after any set_lr / decay / switch),
 * head = the class head the next step trains, last_head = the last step's, phase2 = the switch to phase 2 was made.
 * mpn_model_train_set_state with phase2 = 1 on a training begun with mpn_train_spec.phase2 = 1 makes the switch as
 * mpn_model_train_phase2(m, -1) does (the buffers stay). Refused (MPN_ERR_ARG): no training begun; a weight that does
 * not train; what other than 0 / 2 (and 3 under adam / adamax); an element count other than the tensor's; step
 * outside 0..2^32-1; lr negative or not finite; a head outside 0..K-1; phase2 on a training without phase 2;
 * phase2 1 -> 0.                                                                                                       */
typedef struct mpn_train_state {
  int64_t step;
  float lr;
  int32_t head, last_head, phase2;
} mpn_train_state;
int mpn_model_train_set(mpn_model *m, int32_t weight, int32_t what, const float *src, int64_t n);
int mpn_model_train_get_state(mpn_model *m, mpn_train_state *out);
int mpn_model_train_set_state(mpn_model *m, const mpn_train_state *s);
/* test hook (synchronous, host buffers): the ROI pooling backward of n_jobs (tower, level) jobs that pool one H x W x C
 * map (raw bf16 hi / lo bits) with R ROI rows (R x 5). Job k: foveal region[k] (0..3), scale[k], normalize[k], and its
 * pooled gradient grad_out[k] (R x PH x PW rows of ld[k] floats, the level's C channels at ch_off[k]) -> grad H x W x C
 * fp32 (per cell and channel the sum from +0 in job order, then roi, ph, pw, of g or, normalised, fl(fl(a g) - fl(b x)),
 * x the cell's value); ab (NULL: skipped) n_jobs x R x 2 doubles, the normalised jobs' (a, b) = (1000 / n,
 * 1000 (x . g) / n^3), n = sqrt(sum x^2 + 1e-10f), zeros for the others; argmax (NULL: skipped) n_jobs x R x PH x PW x C
 * int32 (-1: empty bin).                                                                                                */
int mpn_debug_roi_backward_jobs(mpn_ctx *ctx, const uint16_t *hi, const uint16_t *lo, int32_t H, int32_t W, int32_t C, const float *rois,
                                int64_t R, int32_t PW, int32_t PH, int32_t variant, int32_t n_jobs, const int32_t *region, const float *scale,
                                const int32_t *normalize, const int64_t *ld, const int32_t *ch_off, const float *const *grad_out, float *grad,
                                double *ab, int32_t *argmax);

/* MPN_CDEF_END */
#ifdef __cplusplus
}
#endif
#endif /* MPN_ABI_H */

// model.cu — executor for the detection graphs of models/{vgg,multipathnet,resnet}.lua,
// described as data (mpn_model_desc). Mirrors the reference's own trunk / heads split:
//   mpn_model_trunk  == model:get(1):forward            (ImageDetect.lua:107-108)
//   mpn_model_heads  == modules 2..n on cached features  (ImageDetect.lua:114-124)
//   mpn_model_detect == ImageDetect:detect tail          (ImageDetect.lua:176-192)
//   mpn_model_detect_nms adds Tester_FRCNN:testOne's clamp / per-class gather / NMS
//   (Tester_FRCNN.lua:75-78,106-117) so one stream-ordered pass produces final keep lists.
// All activations live in HBM as NHWC split-bf16 planes; every conv / Linear runs on the
// wgmma engine (gemm_tc.cu) except the Cin=3 first layer (conv_simt.cu).
#include "conv_gemm.cuh"
#include "roi.cuh"
#include <algorithm>
#include <cmath>
#include <map>
#include <memory>
#include <set>
#include "train_rule.cuh"

// launchers defined in the other TUs
int mpn_maxpool_launch(mpn_ctx *, const DTensor &, int, int, int, DTensor &);
int mpn_avgpool_launch(mpn_ctx *, const DTensor &, DTensor &);
int mpn_weight_permute_split_launch(mpn_ctx *, const float *, int64_t, int, int, int, __nv_bfloat16 *, __nv_bfloat16 *, int);
int mpn_nhwc_split_to_nchw_launch(mpn_ctx *, const DTensor &, float *);
int mpn_project_rois_launch(mpn_ctx *, const float *, int64_t, float, float *);
int mpn_get_images_launch(mpn_ctx *, const float *, int32_t, int32_t, const mpn_image_transform *, int32_t, int32_t, float *);
int mpn_get_images_size_impl(int32_t, int32_t, double, double, int32_t *, int32_t *, double *);
int mpn_get_images_u8_launch(mpn_ctx *, const uint8_t *, int32_t, int32_t, const mpn_image_transform *, int32_t, int32_t, float *);
int mpn_bbox_norm_launch(mpn_ctx *, float *, int64_t, int64_t, const float *, const float *);
int mpn_bbox_decode_launch(mpn_ctx *, const float *, const float *, int64_t, int, int, float, float, float *);
int mpn_softmax_mean_launch(mpn_ctx *, const float *, int64_t, int, int, int, float *);
int mpn_detect_tail_launch(mpn_ctx *, const float *, int64_t, int, int, int, float *, const float *, const float *, int, float, float,
                           float *, int, const float *, const float *);
int mpn_gather_scored_launch(mpn_ctx *, const float *, const float *, int, int, float, float *, int32_t *, int32_t *);
int mpn_nms_launch(mpn_ctx *, const float *, int, int, const int32_t *, const int32_t *, float, int32_t *, int32_t *);
int mpn_pack_detections_launch(mpn_ctx *, const float *, const float *, int, const int32_t *, const int32_t *, int, int, float *);
int mpn_select_boxes_launch(mpn_ctx *, const float *, const float *, int64_t, int, const float *, const float *, float *);
int mpn_bbox_vote_batched_launch(mpn_ctx *, const float *, const int32_t *, const int32_t *, const int32_t *, const float *, const float *, int, int,
                                 float, float, float *);
int mpn_join_rows_launch(mpn_ctx *, const __nv_bfloat16 *, const __nv_bfloat16 *, int64_t, int64_t, int64_t, int, float *);
int mpn_absmax(mpn_ctx *, const float *, int64_t, float *);
int mpn_weight_permute_half_launch(mpn_ctx *, const float *, int64_t, int, int, int, float, void *);
// train.cu
int mpn_train_criteria_launch(mpn_ctx *, const float *, const float *, const int32_t *, const float *, int, int, float, float *, float *, float *);
int mpn_train_rois5_launch(mpn_ctx *, const float *, int64_t, float *);
int mpn_train_dropout_launch(mpn_ctx *, const DTensor &, int64_t, int64_t, uint64_t, uint32_t, int, int, float);
int mpn_train_dropout_mask_launch(mpn_ctx *, int64_t, uint64_t, uint32_t, int, int, float, uint8_t *);
int mpn_train_gate_mask_launch(mpn_ctx *, const DTensor &, int64_t, int64_t, uint8_t *);
int mpn_train_gate_split_launch(mpn_ctx *, float *, int64_t, int64_t, int64_t, const DTensor *, float, __nv_bfloat16 *, __nv_bfloat16 *,
                                int64_t, int64_t);
int mpn_train_transpose_launch(mpn_ctx *, const float *, const __nv_bfloat16 *, const __nv_bfloat16 *, int64_t, int64_t, int64_t, int, int, int,
                               __nv_bfloat16 *, __nv_bfloat16 *, int64_t, int64_t);
int mpn_train_colsum_launch(mpn_ctx *, const float *, int64_t, int64_t, int64_t, float *);
int mpn_train_sgd_launch(mpn_ctx *, int, float *, const float *, float *, int64_t, float, float, float, float, int, float *, const mpn_optim_step &);
int mpn_train_scale_launch(mpn_ctx *, float *, int64_t, float);
int mpn_train_sgd_split_launch(mpn_ctx *, int, float *, const float *, float *, int, int, int, float, float, float, float, int, __nv_bfloat16 *,
                               __nv_bfloat16 *, __nv_bfloat16 *, __nv_bfloat16 *, int64_t, int64_t, int, const float *, float *,
                               const mpn_optim_step &);
int mpn_train_split_planes_launch(mpn_ctx *, const float *, int, int, int, __nv_bfloat16 *, __nv_bfloat16 *, __nv_bfloat16 *, __nv_bfloat16 *,
                                  int64_t, int64_t, int);
int mpn_train_pool_gate_split_launch(mpn_ctx *, const float *, const DTensor &, float *, __nv_bfloat16 *, __nv_bfloat16 *);
int mpn_train_tap_transpose_launch(mpn_ctx *, const DTensor &, int, int, int, int64_t, int64_t, __nv_bfloat16 *, __nv_bfloat16 *, int64_t,
                                   int64_t);
int mpn_train_col2im_add_launch(mpn_ctx *, const float *, const DTensor &, int, int, int, int64_t, int64_t, float *);
int mpn_train_avgpool_backward_launch(mpn_ctx *, const float *, int64_t, int64_t, int, int, float *);
int mpn_train_add_launch(mpn_ctx *, float *, const float *, int64_t);
int mpn_train_gemm(mpn_ctx *, const __nv_bfloat16 *, const __nv_bfloat16 *, int64_t, int64_t, int64_t, const __nv_bfloat16 *,
                   const __nv_bfloat16 *, int64_t, float *, int64_t, int = 0, int = 0);

namespace {

struct DevBuf {           // owning device allocation
  void *p = nullptr; size_t bytes = 0;
  ~DevBuf() { if (p) cudaFree(p); }
  int ensure(mpn_ctx *ctx, size_t n) {
    if (n <= bytes) return MPN_OK;
    if (p) { cudaFree(p); p = nullptr; bytes = 0; }
    MPN_CUDA(ctx, cudaMalloc(&p, n));
    bytes = n;
    return MPN_OK;
  }
};

struct SplitBuf {         // owning hi/lo planes (with_lo false: the hi plane only, lo stays unallocated)
  DevBuf hi, lo;
  int ensure(mpn_ctx *ctx, size_t elems, bool with_lo = true) {
    MPN_TRY(hi.ensure(ctx, elems * 2 + 256));
    return with_lo ? lo.ensure(ctx, elems * 2 + 256) : MPN_OK;
  }
};

struct WeightDev {
  DevBuf hi, lo;          // split [Cout][K] for tensor-core convs
  DevBuf h16; float h16_scale = 0.f;   // "w16" layers (fc6 / fc7): ONE fp16 plane of w * h16_scale (a power of two)
  DevBuf f32;             // raw fp32 (Torch layout) for the direct first layer / biases
  DevBuf q8, e8; bool has8 = false;   // fp8 numerics: e4m3 plane [Cout][K] of the hi plane, one exponent per output channel
  int64_t n = 0;
  int64_t row = 0;        // elements per output channel of hi / lo (conv_weight_row), set when they are prepared
};

struct Fp8Buf {           // fp8 numerics: the e4m3 plane of one slot and its per-sample exponents
  DevBuf q, e;
  int ensure(mpn_ctx *ctx, const DTensor &x) {
    MPN_TRY(q.ensure(ctx, (size_t)(x.N * x.H * x.W * x.C) + 256));
    return e.ensure(ctx, sizeof(int) * (size_t)x.N + 256);
  }
};

struct LayerExec {
  mpn_layer L;
  ConvProblem prob;
  ConvPlan plan;
  bool is_direct = false;  // Cin not a multiple of 64: CUDA-core direct conv from the NCHW fp32 image
  DTensor in, out;
  // conv -> 2x2/2 max pool fusion (trunk): the conv's epilogue also writes the NEXT layer's (pool) output;
  // pool_only: the full-resolution conv output has no other reader and is not written at all.
  bool fused_pool = false, pool_only = false;
  DTensor pool_out_t;
  bool quant = false;      // fp8 numerics: this layer is the first reader of its input slot's e4m3 plane: quantize first
};

// ---- training state (mpn_model_train_*): fp32 masters stay in WeightDev::f32 (Torch layout); per parameter tensor the
// gradient of the last step and the optim method's state (buf: sgd's momentum buffer or the method's first state; buf2:
// adam's / adamax's second, unallocated for the other methods); the operands of the backward GEMMs are step-local workspaces.
struct TrainParam {
  int w = -1; int64_t n = 0; bool bias = false;
  int cout = 0, cin = 0, kh = 1, kw = 1;   // a weight's geometry as the planner prepares it ((c, h, w) of a FLATTEN for fc6)
  DevBuf grad, buf, buf2;
  // K-major split planes of W^T ([Kin][wt_ld], this weight's rows at column wt_col0) for the dX GEMM of a layer that has a
  // trained layer below; rewritten by every update (sgd_split_kernel). Null for layers without dX.
  // flip: a trained trunk convolution's dgrad planes instead, [Cin][ky][kx][Cout] of the weight rotated by 180 degrees
  __nv_bfloat16 *wt_hi = nullptr, *wt_lo = nullptr; int64_t wt_ld = 0, wt_col0 = 0; bool flip = false;
  int head = -1;                           // class head k's weight or bias (k < K), -1 for every other tensor
  // a fixed-batch-norm convolution (mpn_train_spec.n_fixed): per output channel a^2 under sgd, a under the other methods
  bool fixed = false; DevBuf a2;
  bool idle = false;                       // a phase-2 trunk tensor before the switch (mpn_model_train_phase2): kept, not trained
};
struct TrainState {
  mpn_train_config cfg;
  mpn_train_optim optim = {MPN_OPTIM_SGD, 0.0, 0.0, 0.0, 0.0, 0.0};   // mpn_model_train_begin_optim
  int trunk_from = 0;                      // first trained trunk layer (0: the trunk is frozen)
  // MultiPathNet's phase 2 (mpn_train_spec.phase2): the first trunk layer that trains after the switch (0: no phase 2);
  // trunk_from becomes phase2_from at the switch
  int phase2_from = 0; bool phase2 = false;
  uint32_t step = 0;                      // steps done; the dropout counter of the next step
  int head = 0, last_head = 0;             // the class head the next step trains (mpn_model_train_select_head), the last step's
  bool plan = false;                       // the current heads plan is the training plan (BF16X3 everywhere, BF16X1 when bf16)
  // the "train_bf16" option at begin: every engine GEMM of the step, forward and backward, in BF16X1 on the hi planes;
  // the operand producers write, and the step-local operand buffers and W^T / rotated planes allocate, no lo plane
  bool bf16 = false;
  int64_t last_R = 0; int last_images = 0;
  std::vector<TrainParam> params; std::map<int, int> param_of;   // weight index -> params[]
  std::vector<DevBuf> images;
  DevBuf boxes, rois5, labels, targets, losses, dlogits, dbbox, dconcat, dx[2];
  SplitBuf opA, opGT, opXT;
  std::vector<std::unique_ptr<SplitBuf>> wt_bufs;
  // trunk training (trunk_from > 0): per image of the step, a copy of every trunk slot the backward reads (layer
  // trunk_from's input and each slot written at or above it), taken after the image's forward; per tower the dX of its
  // first layer (the pooled rows' gradient); the ROI argmax and normalisation (a, b) workspaces; the split planes of a
  // gated gradient; the tap planes of the wgrad GEMM
  std::vector<std::map<int, std::unique_ptr<SplitBuf>>> img_bufs; std::vector<std::map<int, DTensor>> img_slots;
  std::vector<std::unique_ptr<DevBuf>> dpooled;
  DevBuf roi_argmax, roi_ab;
  SplitBuf grad_split, opTap;
  // fixed batch norm: the recorded weights; whether each tower trains through the graph backward (the trunk always does)
  std::set<int> fixed;
  std::vector<bool> graph_tower;
  // the graph backward's slot gradients (fp32): a slot takes a buffer at its first contribution and returns it after its
  // producer's backward, so a chain holds two; the free ones by size. And a workspace for a contribution that adds.
  std::vector<std::unique_ptr<DevBuf>> grad_bufs; std::multimap<size_t, DevBuf *> grad_free;
  DevBuf dtmp;
  cudaEvent_t ev[5] = {};                  // step phases: start | trunk + pooling | forward + criteria | backward | update
  ~TrainState() { for (cudaEvent_t e : ev) if (e) cudaEventDestroy(e); }
};

int pool_out(int in, int k, int s, int p, int ceil_mode) {
  int o = ceil_mode ? (in + 2 * p - k + s - 1) / s + 1 : (in + 2 * p - k) / s + 1;
  if (ceil_mode && (o - 1) * s >= in + p) --o;
  return o;
}

}  // namespace

struct mpn_model {
  mpn_ctx *ctx = nullptr;
  mpn_model_desc d;
  std::vector<mpn_layer> trunk_layers, tower_layers;
  std::vector<mpn_tower> towers;
  std::vector<mpn_head> cls_heads;
  std::vector<std::unique_ptr<WeightDev>> weights;
  std::vector<int64_t> w_elems;
  std::vector<std::vector<float>> w_host_small;   // host copies of small arrays (first-layer filter bank / bias travel as kernel parameters)
  std::vector<int> w_prepared;     // 0 = raw only, 1 = split prepared with (Cin,kh,kw) below
  int conv_impl = 0;

  // ---- trunk state
  int tH = 0, tW = 0; bool trunk_valid = false;
  std::vector<LayerExec> trunk_exec;
  std::map<int, DTensor> trunk_slots; std::map<int, std::unique_ptr<SplitBuf>> trunk_bufs;
  std::map<int, std::unique_ptr<Fp8Buf>> trunk_q8;   // fp8 numerics: e4m3 planes of the slots fp8 layers read
  DevBuf image_dev, raw_image_dev;
  int merged_w = -1, merged_b = -1;   // weight-table entries of the concatenated head weights / biases (plan_heads)
  bool merged_stale = false;          // a head's master was set (mpn_model_train_set): the next plan copies the heads again
  std::set<int> elided_slots;      // conv outputs the last trunk forward did not materialise (conv+pool fusion)
  double trunk_flops = 0, head_flops = 0;
  // max pyramids of the trunk slots that towers pool from (roi.cu): level k>=1 buffers per slot
  struct Pyramid { std::vector<std::unique_ptr<DevBuf>> lv; int nlev = 1; };   // fp32 levels 0..nlev-1
  std::map<int, Pyramid> pyramids;

  // ---- heads state
  int64_t hR = 0; bool heads_planned = false;
  struct TowerExec {
    std::unique_ptr<SplitBuf> pooled_buf; DTensor pooled; int ctot = 0;
    std::vector<LayerExec> layers; std::map<int, DTensor> slots; std::map<int, std::unique_ptr<SplitBuf>> bufs;
    int out_features = 0, col_off = 0;
    std::map<int, int> slot_fmt;           // tower slot -> 1 when it is stored as fp16 hi / lo planes (input of a "w16" Linear)
    std::map<int, std::unique_ptr<Fp8Buf>> q8;   // fp8 numerics: e4m3 planes of the slots fp8 layers read
  };
  std::vector<TowerExec> tex;
  SplitBuf concat_buf; int concat_width = 0;
  std::vector<LayerExec> head_exec;     // cls heads then bbox head
  DevBuf rois_dev, boxes_dev, cls_logits, bbox_raw, scores_dev, bboxes_dev;
  DevBuf sb_dev, src_idx_dev, counts_dev, keep_idx_dev, keep_counts_dev;
  RoiJobs jobs;
  // ---- pipelined submit/wait (two slots): per-slot input staging + a private copy of the outputs, copy streams, events
  struct PipeSlot {
    DevBuf image, raw_u8, boxes, scores, bboxes, keep_idx, keep_counts;
    cudaEvent_t h2d = nullptr, compute = nullptr, done = nullptr;
    bool busy = false; int ticket = -1;
  };
  PipeSlot pipe[2];
  cudaStream_t s_h2d = nullptr, s_d2h = nullptr;
  int next_ticket = 0;
  // ---- mpn_model_test_one: per-pass outputs, joined rows, per-class workspaces of capacity n_rows
  DevBuf to_pass_scores, to_pass_bboxes, to_new_boxes, to_scores, to_bboxes, to_sb, to_src, to_counts, to_keep, to_keep_counts, to_voted;
  // ---- detection sink (mpn_model_set_detection_sink): every detect+NMS pass also packs the image's record
  float *sink = nullptr; int64_t sink_cap = 0, sink_n = 0; int sink_top_k = 100;
  // ---- training (mpn_model_train_begin .. _end): while set, the fp32 copies of the trainable weights are kept
  std::unique_ptr<TrainState> train;
  bool plan_split_only = false;    // plan_heads: no "w16" layers (the training plan)
  // a bf16 training step is planning (TrainState::bf16): every engine layer takes BF16X1, whatever ctx->opt_bf16 says;
  // trunk_train_bf16: the current trunk plan was made so (an inference call replans it)
  bool plan_train_bf16 = false, trunk_train_bf16 = false;
  ~mpn_model() {
    for (auto &q : pipe) { if (q.h2d) cudaEventDestroy(q.h2d); if (q.compute) cudaEventDestroy(q.compute); if (q.done) cudaEventDestroy(q.done); }
    if (s_h2d) cudaStreamDestroy(s_h2d);
    if (s_d2h) cudaStreamDestroy(s_d2h);
  }
};

namespace {

int upload_weight_raw(mpn_model *m, int idx, const float *host, int64_t n) {
  WeightDev &w = *m->weights[idx];
  w.n = n;
  MPN_TRY(w.f32.ensure(m->ctx, sizeof(float) * (size_t)std::max<int64_t>(n, 1)));
  MPN_CUDA(m->ctx, cudaMemcpyAsync(w.f32.p, host, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice, m->ctx->stream));
  return MPN_OK;
}

// Torch [Cout][Cin][kh][kw] -> split [Cout][kh][kw][conv_k_pad(Cin)] (the pad zero; dense when Cin % 64 == 0); flat: a
// Linear over a FLATTENed (kh, kw, Cin) map, planned as a 1x1 on that vector: [Cout][conv_k_pad(kh * kw * Cin)], dense
// with the pad at the end (conv_weight_row). Raw fp32 copy is then released.
int prepare_conv_weight(mpn_model *m, int idx, int Cout, int Cin, int kh, int kw, bool flat = false) {
  mpn_ctx *ctx = m->ctx;
  MPN_CHECK_ARG(ctx, idx >= 0 && idx < (int)m->weights.size(), "layer weight index out of range");
  WeightDev &w = *m->weights[idx];
  MPN_CHECK_ARG(ctx, w.n == (int64_t)Cout * Cin * kh * kw, "weight element count does not match layer geometry");
  if (m->w_prepared[idx] == 1) return MPN_OK;
  MPN_CHECK_ARG(ctx, m->w_prepared[idx] == 0, "weight already prepared as an fp16 plane");
  w.row = conv_weight_row(Cin, kh, kw, flat ? 1 : 0);
  const size_t elems = (size_t)((int64_t)Cout * w.row);
  MPN_TRY(w.hi.ensure(ctx, elems * 2 + 256));
  MPN_TRY(w.lo.ensure(ctx, elems * 2 + 256));
  MPN_TRY(mpn_weight_permute_split_launch(ctx, (const float *)w.f32.p, Cout, Cin, kh, kw, (__nv_bfloat16 *)w.hi.p,
                                          (__nv_bfloat16 *)w.lo.p, flat ? 1 : 0));
  m->w_prepared[idx] = 1;
  // the fp32 staging copy is no longer needed (cudaFree synchronises with the split kernel), unless it is a training master
  if (!m->train || !m->train->param_of.count(idx)) { cudaFree(w.f32.p); w.f32.p = nullptr; w.f32.bytes = 0; }
  return MPN_OK;
}

// Torch [Cout][Cin][kh][kw] -> ONE fp16 plane [Cout][kh][kw][Cin] of w * 2^e, 2^e chosen so that max|w| * 2^e lies in
// [8192, 16384) (fp16 overflows at 65504; weights 2^-27 below the largest one fall into fp16's subnormals, where they
// contribute nothing measurable); raw fp32 copy is then released.
int prepare_conv_weight_w16(mpn_model *m, int idx, int Cout, int Cin, int kh, int kw) {
  mpn_ctx *ctx = m->ctx;
  MPN_CHECK_ARG(ctx, idx >= 0 && idx < (int)m->weights.size(), "layer weight index out of range");
  WeightDev &w = *m->weights[idx];
  MPN_CHECK_ARG(ctx, w.n == (int64_t)Cout * Cin * kh * kw, "weight element count does not match layer geometry");
  if (m->w_prepared[idx] == 2) return MPN_OK;
  MPN_CHECK_ARG(ctx, m->w_prepared[idx] == 0, "weight already prepared in the split-bf16 layout");
  float amax = 0.f;
  MPN_TRY(mpn_absmax(ctx, (const float *)w.f32.p, w.n, &amax));
  MPN_CHECK_ARG(ctx, std::isfinite(amax), "weight holds a non-finite value");
  int e = 0;
  if (amax > 0.f) { (void)std::frexp(amax, &e); e = 14 - e; }          // amax = f * 2^e0, f in [0.5, 1) -> amax * 2^(14 - e0) in [8192, 16384)
  e = std::max(-60, std::min(60, e));
  w.h16_scale = std::ldexp(1.0f, e);
  MPN_TRY(w.h16.ensure(ctx, (size_t)w.n * 2 + 256));
  MPN_TRY(mpn_weight_permute_half_launch(ctx, (const float *)w.f32.p, Cout, Cin, kh, kw, w.h16_scale, w.h16.p));
  m->w_prepared[idx] = 2;
  if (!m->train || !m->train->param_of.count(idx)) { cudaFree(w.f32.p); w.f32.p = nullptr; w.f32.bytes = 0; }
  return MPN_OK;
}

// fp8 numerics: the e4m3 plane of the weight's hi plane (split-bf16 preparation first; the fp32 copy may be gone) and one
// exponent per output channel (fp8.cu; exponents readable up to Cout rounded up to 128, as the engine's N tiles need).
// A model built without the option switches to it on its next plan.
int prepare_conv_weight_fp8(mpn_model *m, int idx, int Cout, int Cin, int kh, int kw, bool flat = false) {
  mpn_ctx *ctx = m->ctx;
  MPN_CHECK_ARG(ctx, m->w_prepared[idx] != 2, "fp8 numerics: the weight was prepared as an fp16 plane (fc_w16); build the model with the option set");
  MPN_TRY(prepare_conv_weight(m, idx, Cout, Cin, kh, kw, flat));
  WeightDev &w = *m->weights[idx];
  if (w.has8) return MPN_OK;
  const int64_t rows_pad = ((int64_t)Cout + 127) / 128 * 128;
  MPN_TRY(w.q8.ensure(ctx, (size_t)(Cout * w.row) + 256));
  MPN_TRY(w.e8.ensure(ctx, sizeof(int) * (size_t)rows_pad));
  MPN_TRY(mpn_fp8_weight_launch(ctx, (const __nv_bfloat16 *)w.hi.p, Cout, w.row, rows_pad, (uint8_t *)w.q8.p, (int *)w.e8.p));
  w.has8 = true;
  return MPN_OK;
}

DTensor make_split_view(SplitBuf &b, int64_t N, int64_t H, int64_t W, int64_t C) {
  DTensor t; t.hi = (__nv_bfloat16 *)b.hi.p; t.lo = (__nv_bfloat16 *)b.lo.p; t.N = N; t.H = H; t.W = W; t.C = C; t.ld = C;
  return t;
}

// Build the executable form of one CONV layer (weights prepared, problem + plan filled).
// flat_from: if the layer consumes a FLATTENed (h,w,c) tensor, its Linear weight [Cout][c*h*w]
// in (c,h,w) order is re-laid as a (kh=h,kw=w,Cin=c) conv weight => (h,w,c) K order.
// q8: the e4m3 plane of `in` when the layer runs the fp8 numerics (option "fp8"), null otherwise (the cls / bbox heads).
int build_conv(mpn_model *m, LayerExec &e, const DTensor &in, DTensor out, int fh, int fw, int fc, bool per_roi = false,
               Fp8Buf *q8 = nullptr) {
  mpn_ctx *ctx = m->ctx;
  const mpn_layer &L = e.L;
  e.in = in; e.out = out;
  ConvProblem &p = e.prob;
  p = ConvProblem();
  p.x = in; p.Cout = L.cout; p.kh = L.kh; p.kw = L.kw; p.stride = L.stride; p.pad = L.pad; p.relu = L.relu;
  p.y = out; p.y_f32_ld = out.ld;
  p.m_invariant = per_roi ? 1 : 0;
  // bf16 inference numerics (mpn_ctx_set_option "bf16"), read when the model plans: one bf16 product per MAC on the hi
  // planes; a bf16 training step's plan takes the same numerics from the training state
  p.bf16 = (m->plan_train_bf16 || ctx->opt_bf16 == 1) ? 1 : 0;
  MPN_CHECK_ARG(ctx, L.weight >= 0 && L.weight < (int)m->weights.size(), "conv layer without weight");
  if (q8) {                // fp8 numerics: one e4m3 product per MAC, per-sample / per-channel power-of-two scales
    MPN_CHECK_ARG(ctx, in.fmt == 0, "fp8 numerics: the input must be split-bf16 planes");
    if (in.C % 64 != 0) {    // the quantizer's groups are 64 channels wide: a K tail has no scale of its own
      char b[200];
      snprintf(b, sizeof b, "fp8 numerics: the %dx%d convolution %d -> %d (%s) reads %lld input channels, not a multiple of 64; "
               "build the model without the \"fp8\" option", L.kh, L.kw, L.cin, L.cout, per_roi ? "per-ROI" : "trunk", (long long)in.C);
      return mpn_fail(ctx, MPN_ERR_ARG, b);
    }
    MPN_TRY(q8->ensure(ctx, in));
    if (fc > 0) { MPN_TRY(prepare_conv_weight_fp8(m, L.weight, L.cout, fc, fh, fw, /*flat=*/true)); }
    else { MPN_TRY(prepare_conv_weight_fp8(m, L.weight, L.cout, L.cin, L.kh, L.kw)); }
    WeightDev &w = *m->weights[L.weight];
    p.fp8 = 1; p.bf16 = 0;
    p.w_hi = (const __nv_bfloat16 *)w.hi.p; p.w_lo = (const __nv_bfloat16 *)w.lo.p;
    p.w8 = (const uint8_t *)w.q8.p; p.w8_exp = (const int *)w.e8.p;
    p.x8 = (const uint8_t *)q8->q.p; p.x8_exp = (const int *)q8->e.p;
    if (L.bias >= 0) {
      MPN_CHECK_ARG(ctx, L.bias < (int)m->weights.size() && m->weights[L.bias]->n == L.cout, "bias size mismatch");
      p.bias = (const float *)m->weights[L.bias]->f32.p;
    }
    return conv_tc_plan(ctx, p, e.plan);
  }
  // the big per-ROI Linears (fc6 / fc7) take the "w16" numerics — weight = one scaled fp16 plane, activation = fp16 hi / lo
  // planes, two tensor-core products per MAC instead of three — exactly when plan_heads gave their input fp16 planes
  const bool w16 = (in.fmt == 1);
  MPN_CHECK_ARG(ctx, !w16 || (per_roi && L.kh == 1 && L.kw == 1 && L.stride == 1 && L.pad == 0 && in.H == 1 && in.W == 1),
                "fp16 activation planes reached a layer that is not a per-ROI Linear");
  WeightDev &w = *m->weights[L.weight];
  if (w16) {
    MPN_TRY(prepare_conv_weight_w16(m, L.weight, L.cout, fc > 0 ? fc : L.cin, fc > 0 ? fh : L.kh, fc > 0 ? fw : L.kw));
    p.w16 = w.h16.p; p.w16_inv_scale = 1.0f / w.h16_scale;
  } else {
    if (fc > 0) { MPN_TRY(prepare_conv_weight(m, L.weight, L.cout, fc, fh, fw, /*flat=*/true)); }
    else { MPN_TRY(prepare_conv_weight(m, L.weight, L.cout, L.cin, L.kh, L.kw)); }
    p.w_hi = (const __nv_bfloat16 *)w.hi.p; p.w_lo = (const __nv_bfloat16 *)w.lo.p;
  }
  if (L.bias >= 0) {
    MPN_CHECK_ARG(ctx, L.bias < (int)m->weights.size() && m->weights[L.bias]->n == L.cout, "bias size mismatch");
    p.bias = (const float *)m->weights[L.bias]->f32.p;
  }
  MPN_TRY(conv_tc_plan(ctx, p, e.plan));
  return MPN_OK;
}

int run_conv(mpn_model *m, LayerExec &e) {
  if (e.quant) MPN_TRY(mpn_fp8_quantize_launch(m->ctx, e.prob.x, const_cast<uint8_t *>(e.prob.x8), const_cast<int *>(e.prob.x8_exp)));
  if (m->conv_impl == 1) return conv_ref_launch(m->ctx, e.prob);
  return conv_tc_launch(m->ctx, e.prob, e.plan);
}

// ------------------------------------------------------------------ trunk planning
int plan_trunk(mpn_model *m, int H, int W) {
  mpn_ctx *ctx = m->ctx;
  m->trunk_exec.clear(); m->trunk_slots.clear();
  m->trunk_flops = 0;
  MPN_CHECK_ARG(ctx, !(ctx->opt_fp8 == 1 && ctx->opt_bf16 == 1), "the \"fp8\" and \"bf16\" options are both on");
  const bool fp8 = ctx->opt_fp8 == 1;
  std::set<int> quantized;         // fp8: slots whose e4m3 plane is current at this point of the forward pass
  DTensor img; img.N = 1; img.H = H; img.W = W; img.C = 3; img.ld = 3;   // slot 0: NCHW fp32 image (special)
  m->trunk_slots[0] = img;
  for (const mpn_layer &L : m->trunk_layers) {
    MPN_CHECK_ARG(ctx, m->trunk_slots.count(L.in_slot), "trunk layer reads an undefined slot");
    const DTensor in = m->trunk_slots[L.in_slot];
    LayerExec e; e.L = L;
    DTensor out; out.N = in.N;
    if (L.kind == MPN_LAYER_CONV) {
      MPN_CHECK_ARG(ctx, L.cin == in.C, "trunk conv cin does not match its input");
      out.H = (in.H + 2 * L.pad - L.kh) / L.stride + 1; out.W = (in.W + 2 * L.pad - L.kw) / L.stride + 1; out.C = L.cout;
    } else if (L.kind == MPN_LAYER_MAXPOOL) {
      out.H = pool_out((int)in.H, L.kh, L.stride, L.pad, L.ceil_mode);
      out.W = pool_out((int)in.W, L.kw, L.stride, L.pad, L.ceil_mode); out.C = in.C;
    } else {
      return mpn_fail(ctx, MPN_ERR_ARG, "unsupported trunk layer kind");
    }
    MPN_CHECK_ARG(ctx, out.H > 0 && out.W > 0, "trunk layer output is empty");
    MPN_CHECK_ARG(ctx, L.out_slot > 0, "trunk layers may not write slot 0");
    auto &buf = m->trunk_bufs[L.out_slot];
    if (!buf) buf.reset(new SplitBuf());
    MPN_TRY(buf->ensure(ctx, (size_t)(out.N * out.H * out.W * out.C)));
    out = make_split_view(*buf, out.N, out.H, out.W, out.C);
    if (L.kind == MPN_LAYER_CONV) {
      if (L.in_slot == 0) {
        e.is_direct = true; e.in = in; e.out = out;
        MPN_CHECK_ARG(ctx, L.weight >= 0 && m->weights[L.weight]->n == (int64_t)L.cout * L.cin * L.kh * L.kw,
                      "first-layer weight size mismatch");
      } else {
        DTensor o2 = out;
        Fp8Buf *q8 = nullptr;
        if (fp8) {
          auto &qb = m->trunk_q8[L.in_slot];
          if (!qb) qb.reset(new Fp8Buf());
          q8 = qb.get();
          e.quant = quantized.insert(L.in_slot).second;
        }
        MPN_TRY(build_conv(m, e, in, o2, 0, 0, 0, false, q8));
        if (L.residual_slot >= 0) {
          MPN_CHECK_ARG(ctx, m->trunk_slots.count(L.residual_slot), "residual slot undefined");
          e.prob.res = m->trunk_slots[L.residual_slot];
        }
      }
      m->trunk_flops += 2.0 * L.cin * L.cout * L.kh * L.kw * (double)out.H * out.W * out.N;
    } else {
      e.in = in; e.out = out;
    }
    m->trunk_slots[L.out_slot] = out;
    quantized.erase(L.out_slot);
    m->trunk_exec.push_back(e);
  }
  // conv(3x3 / stride 1 plan, 16 x 8 patches) immediately followed by a 2x2/2 pad-0 max pool of its output: fuse the pool into the epilogue
  {
    const char *envf = getenv("MPN_TC_FUSE_POOL");
    const bool allow = !(envf && envf[0] == '0');
    for (size_t i = 0; allow && i + 1 < m->trunk_exec.size(); ++i) {
      LayerExec &c = m->trunk_exec[i]; const LayerExec &q = m->trunk_exec[i + 1];
      if (c.L.kind != MPN_LAYER_CONV || c.is_direct || q.L.kind != MPN_LAYER_MAXPOOL) continue;
      if (q.L.in_slot != c.L.out_slot || q.L.kh != 2 || q.L.kw != 2 || q.L.stride != 2 || q.L.pad != 0) continue;
      if (c.plan.mode != 1 || c.plan.splitk != 1 || c.L.residual_slot >= 0 || (c.L.cout % 8) != 0) continue;
      if (q.out.H != (c.out.H + 1) / 2 || q.out.W != (c.out.W + 1) / 2) continue;      // floor-mode pools with odd sizes stay separate
      bool other_reader = false;
      for (size_t j = 0; j < m->trunk_exec.size(); ++j) {
        if (j == i + 1) continue;
        const mpn_layer &L2 = m->trunk_exec[j].L;
        if (j > i && (L2.in_slot == c.L.out_slot || L2.residual_slot == c.L.out_slot)) other_reader = true;
      }
      for (const mpn_tower &T : m->towers)
        for (int l = 0; l < T.n_levels; ++l) if (T.level_slot[l] == c.L.out_slot) other_reader = true;
      // a trained convolution's output is read by the pool backward
      if (m->train && m->train->trunk_from > 0 && (int)i >= m->train->trunk_from) other_reader = true;
      c.fused_pool = true; c.pool_only = !other_reader; c.pool_out_t = q.out;
    }
  }
  // max pyramids for every slot a tower pools from: levels with 2^k <= min(H, W), at most ROI_MAX_LEVELS-1 extra copies
  for (const mpn_tower &T : m->towers)
    for (int l = 0; l < T.n_levels; ++l) {
      const int slot = T.level_slot[l];
      MPN_CHECK_ARG(ctx, m->trunk_slots.count(slot) && slot > 0, "tower level reads an undefined trunk slot");
      const DTensor &f = m->trunk_slots[slot];
      mpn_model::Pyramid &P = m->pyramids[slot];
      // a level with block 2^k is only ever used for a bin window whose smaller side is >= 2^k cells; a bin of this tower
      // spans at most ceil(region_scale * map_side / pooled_side) + 1 cells of the (clipped) region, so higher levels are dead
      const double rs = T.region == 0 ? 1.0 : (T.region == 1 ? 1.5 : (T.region == 2 ? 2.0 : 4.0));
      const long long max_bin = std::min<long long>(std::min(f.H, f.W),
          (long long)std::ceil(rs * (double)std::max(f.H, f.W) / (double)std::min(T.pooled_h, T.pooled_w)) + 2);
      int nlev = 1;
      while (nlev < ROI_MAX_LEVELS && (1ll << nlev) <= max_bin) ++nlev;
      nlev = std::max(nlev, P.nlev);                                   // several towers may share the slot: keep the deepest
      P.nlev = nlev;
      P.lv.resize(nlev);
      for (int k = 0; k < nlev; ++k) {
        if (!P.lv[k]) P.lv[k].reset(new DevBuf());
        MPN_TRY(P.lv[k]->ensure(ctx, sizeof(float) * (size_t)(f.N * f.H * f.W * f.C) + 256));
      }
    }
  m->tH = H; m->tW = W; m->trunk_valid = false; m->heads_planned = false;
  m->trunk_train_bf16 = m->plan_train_bf16;
  return MPN_OK;
}

int run_trunk(mpn_model *m, const float *image_dev) {
  mpn_ctx *ctx = m->ctx;
  m->elided_slots.clear();
  for (size_t li = 0; li < m->trunk_exec.size(); ++li) {
    LayerExec &e = m->trunk_exec[li];
    const mpn_layer &L = e.L;
    if (e.fused_pool && m->conv_impl == 0) {
      if (e.quant) MPN_TRY(mpn_fp8_quantize_launch(ctx, e.prob.x, const_cast<uint8_t *>(e.prob.x8), const_cast<int *>(e.prob.x8_exp)));
      ConvProblem pf = e.prob;
      pf.pool = e.pool_out_t; pf.pool_only = e.pool_only ? 1 : 0;
      MPN_TRY(conv_tc_launch(ctx, pf, e.plan));
      if (e.pool_only) m->elided_slots.insert(L.out_slot);
      ++li;                                  // the pool layer's output is already written
      continue;
    }
    if (L.kind == MPN_LAYER_CONV) {
      if (e.is_direct) {
        const float *bias = L.bias >= 0 ? (const float *)m->weights[L.bias]->f32.p : nullptr;
        MPN_TRY(conv_direct_nchw_launch(ctx, image_dev, 1, L.cin, (int)e.in.H, (int)e.in.W,
                                        (const float *)m->weights[L.weight]->f32.p, bias, L.cout, L.kh, L.kw, L.stride,
                                        L.pad, L.relu, e.out,
                                        m->w_host_small[L.weight].empty() ? nullptr : m->w_host_small[L.weight].data(),
                                        (L.bias >= 0 && !m->w_host_small[L.bias].empty()) ? m->w_host_small[L.bias].data() : nullptr));
      } else {
        MPN_TRY(run_conv(m, e));
      }
    } else {
      MPN_TRY(mpn_maxpool_launch(ctx, e.in, L.kh, L.stride, L.pad, e.out));
    }
  }
  for (auto &kv : m->pyramids) {
    const DTensor &f = m->trunk_slots[kv.first];
    float *lv[ROI_MAX_LEVELS] = {nullptr};
    for (int k = 0; k < kv.second.nlev; ++k) lv[k] = (float *)kv.second.lv[k]->p;
    int too_big = 0;       // small maps (conv5): every level in one launch
    MPN_TRY(mpn_maxpyr_all_launch(ctx, f.hi, f.lo, (int)f.N, (int)f.H, (int)f.W, (int)f.C, f.ld, kv.second.nlev, lv, &too_big));
    if (!too_big) continue;
    MPN_TRY(mpn_pyr_level0_launch(ctx, f.hi, f.lo, (int)f.N, (int)f.H, (int)f.W, (int)f.C, f.ld, lv[0]));
    for (int k = 1; k < kv.second.nlev; ++k)
      MPN_TRY(mpn_maxpyr_launch(ctx, lv[k - 1], (int)f.N, (int)f.H, (int)f.W, (int)f.C, 1 << (k - 1), lv[k]));
  }
  m->trunk_valid = true;
  return MPN_OK;
}

// ------------------------------------------------------------------ heads planning
int plan_heads(mpn_model *m, int64_t R) {
  mpn_ctx *ctx = m->ctx;
  const int C = m->d.num_classes;
  m->head_flops = 0;
  MPN_CHECK_ARG(ctx, !(ctx->opt_fp8 == 1 && ctx->opt_bf16 == 1), "the \"fp8\" and \"bf16\" options are both on");
  const bool fp8 = ctx->opt_fp8 == 1;
  m->tex.clear(); m->tex.resize(m->towers.size());
  m->jobs.n = 0;
  // concat width = sum of tower output features
  int width = 0;
  std::vector<int> feat(m->towers.size(), 0);
  for (size_t t = 0; t < m->towers.size(); ++t) {
    const mpn_tower &T = m->towers[t];
    // find the producing layer of out_slot to learn its feature count
    int f = -1;
    for (int i = 0; i < T.n_layers; ++i) {
      const mpn_layer &L = m->tower_layers[T.first_layer + i];
      if (L.out_slot == T.out_slot) f = (L.kind == MPN_LAYER_CONV) ? L.cout : -2;
    }
    MPN_CHECK_ARG(ctx, f != -1, "tower out_slot is never written");
    feat[t] = f;   // -2: resolved below (avgpool/flatten output)
  }
  // first pass to resolve shapes and features
  for (size_t t = 0; t < m->towers.size(); ++t) {
    const mpn_tower &T = m->towers[t];
    mpn_model::TowerExec &X = m->tex[t];
    X.ctot = 0;
    for (int l = 0; l < T.n_levels; ++l) {
      MPN_CHECK_ARG(ctx, m->trunk_slots.count(T.level_slot[l]) && T.level_slot[l] > 0, "tower level reads an undefined trunk slot");
      X.ctot += (int)m->trunk_slots[T.level_slot[l]].C;
    }
    X.pooled_buf.reset(new SplitBuf());
    MPN_TRY(X.pooled_buf->ensure(ctx, (size_t)R * T.pooled_h * T.pooled_w * X.ctot));
    X.pooled = make_split_view(*X.pooled_buf, R, T.pooled_h, T.pooled_w, X.ctot);
    // ROI jobs
    int ch_off = 0;
    for (int l = 0; l < T.n_levels; ++l) {
      MPN_CHECK_ARG(ctx, m->jobs.n < MAX_ROI_JOBS, "too many (tower, level) ROI jobs");
      const DTensor &f = m->trunk_slots[T.level_slot[l]];
      RoiJob &j = m->jobs.j[m->jobs.n++];
      j.H = (int)f.H; j.W = (int)f.W; j.C = (int)f.C; j.scale = T.level_scale[l];
      j.region = T.region; j.out_hi = X.pooled.hi; j.out_lo = X.pooled.lo; j.out_ld = X.ctot; j.out_ch_off = ch_off;
      j.normalize = T.normalize; j.out_fmt = 0; j.ovf = nullptr; j.tower = (int)t;
      const mpn_model::Pyramid &P = m->pyramids[T.level_slot[l]];
      j.nlev = P.nlev;
      for (int k = 0; k < ROI_MAX_LEVELS; ++k) j.lv[k] = (const float *)P.lv[std::min(k, P.nlev - 1)]->p;
      ch_off += (int)f.C;
    }
    // shape walk
    std::map<int, DTensor> shp; shp[0] = X.pooled;
    for (int i = 0; i < T.n_layers; ++i) {
      const mpn_layer &L = m->tower_layers[T.first_layer + i];
      MPN_CHECK_ARG(ctx, shp.count(L.in_slot), "tower layer reads an undefined slot");
      const DTensor in = shp[L.in_slot]; DTensor out; out.N = R;
      if (L.kind == MPN_LAYER_CONV) {
        MPN_CHECK_ARG(ctx, L.cin == in.C, "tower conv cin does not match its input");
        out.H = (in.H + 2 * L.pad - L.kh) / L.stride + 1; out.W = (in.W + 2 * L.pad - L.kw) / L.stride + 1; out.C = L.cout;
      } else if (L.kind == MPN_LAYER_FLATTEN) { out.H = 1; out.W = 1; out.C = in.H * in.W * in.C; }
      else if (L.kind == MPN_LAYER_AVGPOOL) { out.H = 1; out.W = 1; out.C = in.C; }
      else if (L.kind == MPN_LAYER_MAXPOOL) {
        out.H = pool_out((int)in.H, L.kh, L.stride, L.pad, L.ceil_mode); out.W = pool_out((int)in.W, L.kw, L.stride, L.pad, L.ceil_mode);
        out.C = in.C;
      } else return mpn_fail(ctx, MPN_ERR_ARG, "unsupported tower layer kind");
      shp[L.out_slot] = out;
    }
    // ---- plane formats of the tower's slots: the input of a "w16" Linear (fc6 / fc7: K >= 2048, >= 1024 outputs;
    // tools/split_emulation.py estimates the error) is stored as fp16 hi / lo planes by whoever produces it (the ROI kernel for slot 0,
    // the previous layer's epilogue otherwise); every reader of such a slot must be a w16 Linear (or the FLATTEN in front
    // of one), else the slot stays bf16. mpn_ctx_set_option("fc_w16", 0) / MPN_FC_W16=0 switches the scheme off.
    {
      // Default (option / environment unset): ON for single-tower graphs (Fast R-CNN: cfg 2 measures 4-5e-4 on the scores, the
      // figure the CPU emulation predicted), OFF for multi-tower graphs — the first GPU run of cfg 3 with w16 in all five
      // towers measured 2.3e-3: the class Linear reads a 4 x 4096 concat of w16 outputs and its logits are large enough that
      // the weight plane's 2^-12 becomes a visible softmax error (tests/test_model_gpu.py::test_multipathnet_full_size_cfg3).
      static const int w16_env = [] { const char *e = getenv("MPN_FC_W16"); return !e ? -1 : (e[0] == '0' ? 0 : 1); }();
      // Under the bf16 numerics (option "bf16") every engine layer takes BF16X1 and fc_w16 is ignored: no fp16 planes.
      // The same under the fp8 numerics (option "fp8"): the tower layers take FP8X1, the heads BF16X3.
      const int w16_on = (ctx->opt_bf16 == 1 || fp8 || m->plan_split_only) ? 0
                         : (ctx->opt_fc_w16 >= 0 ? ctx->opt_fc_w16 : (w16_env >= 0 ? w16_env : (m->towers.size() == 1 ? 1 : 0)));
      std::map<int, int> &fmt = X.slot_fmt;
      fmt.clear();
      auto wants = [&](const mpn_layer &L) {
        if (!w16_on || L.kind != MPN_LAYER_CONV || L.residual_slot >= 0) return false;
        const DTensor &in = shp[L.in_slot];
        if (L.weight >= 0 && L.weight < (int)m->w_prepared.size() && m->w_prepared[L.weight] == 2) return true;   // the fp16 plane is what there is
        return L.kh == 1 && L.kw == 1 && L.stride == 1 && L.pad == 0 && in.H == 1 && in.W == 1 && in.C >= 2048 && L.cout >= 1024 &&
               L.weight >= 0 && L.weight < (int)m->w_prepared.size() && m->w_prepared[L.weight] != 1;
      };
      for (int i = 0; i < T.n_layers; ++i) { const mpn_layer &L = m->tower_layers[T.first_layer + i]; if (wants(L)) fmt[L.in_slot] = 1; }
      for (int pass = 0; pass < 4; ++pass) {
        for (int i = T.n_layers - 1; i >= 0; --i) {                 // a FLATTEN's output aliases its input
          const mpn_layer &L = m->tower_layers[T.first_layer + i];
          if (L.kind == MPN_LAYER_FLATTEN && fmt.count(L.out_slot) && fmt[L.out_slot]) fmt[L.in_slot] = 1;
        }
        for (int i = 0; i < T.n_layers; ++i) {                      // any other reader vetoes
          const mpn_layer &L = m->tower_layers[T.first_layer + i];
          auto veto = [&](int slot) {
            if (!fmt.count(slot) || !fmt[slot]) return;
            fmt[slot] = 0;
            for (int j = 0; j < T.n_layers; ++j) {                  // and so does the alias on the other side of a FLATTEN
              const mpn_layer &F = m->tower_layers[T.first_layer + j];
              if (F.kind == MPN_LAYER_FLATTEN && (F.in_slot == slot || F.out_slot == slot)) { fmt[F.in_slot] = 0; fmt[F.out_slot] = 0; }
            }
          };
          if (L.kind == MPN_LAYER_CONV) { if (!wants(L)) veto(L.in_slot); if (L.residual_slot >= 0) veto(L.residual_slot); }
          else if (L.kind == MPN_LAYER_FLATTEN) { if (fmt.count(L.in_slot) && fmt[L.in_slot] && !(fmt.count(L.out_slot) && fmt[L.out_slot])) veto(L.in_slot); }
          else veto(L.in_slot);
        }
        if (fmt.count(T.out_slot) && fmt[T.out_slot]) fmt[T.out_slot] = 0;      // the concat feeds the (three-product) heads
      }
    }
    MPN_CHECK_ARG(ctx, shp.count(T.out_slot), "tower out_slot undefined");
    const DTensor o = shp[T.out_slot];
    MPN_CHECK_ARG(ctx, o.H == 1 && o.W == 1, "tower output must be R x 1 x 1 x F");
    X.out_features = (int)o.C; X.col_off = width; width += (int)o.C;
  }
  for (int ji = 0; ji < m->jobs.n; ++ji) {                          // pooled tensors that feed a w16 Linear: fp16 planes
    RoiJob &j = m->jobs.j[ji];
    mpn_model::TowerExec &X = m->tex[j.tower];
    if (X.slot_fmt.count(0) && X.slot_fmt[0]) { j.out_fmt = 1; MPN_TRY(mpn_ovf_flag(ctx, &j.ovf)); X.pooled.fmt = 1; }
  }
  m->concat_width = width;
  MPN_CHECK_ARG(ctx, width % 8 == 0, "concat width must be a multiple of 8");
  MPN_TRY(m->concat_buf.ensure(ctx, (size_t)R * width));
  // second pass: allocate + build
  for (size_t t = 0; t < m->towers.size(); ++t) {
    const mpn_tower &T = m->towers[t];
    mpn_model::TowerExec &X = m->tex[t];
    X.slots.clear(); X.slots[0] = X.pooled; X.layers.clear();
    int flat_h = 0, flat_w = 0, flat_c = 0; int flat_slot = -1;
    std::set<int> quantized;       // fp8: slots whose e4m3 plane is current at this point of the tower
    for (int i = 0; i < T.n_layers; ++i) {
      const mpn_layer &L = m->tower_layers[T.first_layer + i];
      const DTensor in = X.slots[L.in_slot];
      LayerExec e; e.L = L;
      DTensor out; out.N = R;
      if (L.kind == MPN_LAYER_FLATTEN) {
        MPN_CHECK_ARG(ctx, in.ld == in.C, "flatten needs a dense input");
        out = in; out.H = 1; out.W = 1; out.C = in.H * in.W * in.C; out.ld = out.C;
        flat_h = (int)in.H; flat_w = (int)in.W; flat_c = (int)in.C; flat_slot = L.out_slot;
        X.slots[L.out_slot] = out; e.in = in; e.out = out; X.layers.push_back(e);
        quantized.erase(L.out_slot);
        continue;
      }
      if (L.kind == MPN_LAYER_CONV) {
        out.H = (in.H + 2 * L.pad - L.kh) / L.stride + 1; out.W = (in.W + 2 * L.pad - L.kw) / L.stride + 1; out.C = L.cout;
      } else if (L.kind == MPN_LAYER_AVGPOOL) { out.H = 1; out.W = 1; out.C = in.C; }
      else { out.H = pool_out((int)in.H, L.kh, L.stride, L.pad, L.ceil_mode); out.W = pool_out((int)in.W, L.kw, L.stride, L.pad, L.ceil_mode); out.C = in.C; }
      if (L.out_slot == T.out_slot) {      // write straight into this tower's column slice of the concat
        out.hi = (__nv_bfloat16 *)m->concat_buf.hi.p + X.col_off; out.lo = (__nv_bfloat16 *)m->concat_buf.lo.p + X.col_off;
        out.ld = width;
      } else {
        auto &buf = X.bufs[L.out_slot];
        if (!buf) buf.reset(new SplitBuf());
        MPN_TRY(buf->ensure(ctx, (size_t)(out.N * out.H * out.W * out.C)));
        DTensor v = make_split_view(*buf, out.N, out.H, out.W, out.C); out = v;
      }
      out.fmt = (X.slot_fmt.count(L.out_slot) && X.slot_fmt[L.out_slot]) ? 1 : 0;
      if (L.kind == MPN_LAYER_CONV) {
        const bool from_flat = (L.in_slot == flat_slot) && L.kh == 1 && L.kw == 1;
        Fp8Buf *q8 = nullptr;
        if (fp8) {                 // samples = ROIs: the pooled row for fc6, the ROI's map for ResNet's layer4
          auto &qb = X.q8[L.in_slot];
          if (!qb) qb.reset(new Fp8Buf());
          q8 = qb.get();
          e.quant = quantized.insert(L.in_slot).second;
        }
        MPN_TRY(build_conv(m, e, in, out, from_flat ? flat_h : 0, from_flat ? flat_w : 0, from_flat ? flat_c : 0, /*per_roi=*/true, q8));
        if (L.residual_slot >= 0) {
          MPN_CHECK_ARG(ctx, X.slots.count(L.residual_slot), "tower residual slot undefined");
          e.prob.res = X.slots[L.residual_slot];
        }
        m->head_flops += 2.0 * (double)L.cin * L.cout * L.kh * L.kw * (double)out.H * out.W * (double)R;
      } else { e.in = in; e.out = out; }
      X.slots[L.out_slot] = out;
      quantized.erase(L.out_slot);
      X.layers.push_back(e);
    }
  }
  // heads: cls (K of them) then bbox, fp32 outputs
  const int K = (int)m->cls_heads.size();
  MPN_TRY(m->cls_logits.ensure(ctx, sizeof(float) * (size_t)K * R * C + 256));
  MPN_TRY(m->bbox_raw.ensure(ctx, sizeof(float) * (size_t)R * 4 * C + 256));
  MPN_TRY(m->scores_dev.ensure(ctx, sizeof(float) * (size_t)R * C + 256));
  MPN_TRY(m->bboxes_dev.ensure(ctx, sizeof(float) * (size_t)R * 4 * C + 256));
  m->head_exec.clear();
  auto add_head = [&](const mpn_head &h, float *out_ptr) -> int {
    MPN_CHECK_ARG(ctx, h.col_begin % 8 == 0 && h.col_begin + h.col_len <= width && h.col_len % 64 == 0, "head column range invalid");
    LayerExec e; mpn_layer L; memset(&L, 0, sizeof L);
    L.kind = MPN_LAYER_CONV; L.cin = h.col_len; L.cout = h.cout; L.kh = L.kw = 1; L.stride = 1; L.pad = 0; L.relu = 0;
    L.residual_slot = -1; L.weight = h.weight; L.bias = h.bias;
    e.L = L;
    DTensor in; in.hi = (__nv_bfloat16 *)m->concat_buf.hi.p + h.col_begin; in.lo = (__nv_bfloat16 *)m->concat_buf.lo.p + h.col_begin;
    in.N = R; in.H = 1; in.W = 1; in.C = h.col_len; in.ld = width;
    DTensor out; out.f32 = out_ptr; out.N = R; out.H = 1; out.W = 1; out.C = h.cout; out.ld = h.cout;
    MPN_TRY(build_conv(m, e, in, out, 0, 0, 0, /*per_roi=*/true));
    m->head_flops += 2.0 * (double)h.col_len * h.cout * (double)R;
    m->head_exec.push_back(e);
    return MPN_OK;
  };
  for (int k = 0; k < K; ++k) MPN_CHECK_ARG(ctx, m->cls_heads[k].cout == C, "cls head width must equal num_classes");
  MPN_CHECK_ARG(ctx, m->d.bbox_head.cout == 4 * C, "bbox head width must be 4*num_classes");
  // Optional (MPN_MERGE_HEADS=1; off by default: measured neutral, 687.8k vs 691.7k proposals/s on the same box): heads that
  // read the same columns and together have <= 128 outputs (Fast R-CNN: 21 + 84) run as ONE split-K GEMM whose reduce pass
  // scatters the column ranges to the dense per-head buffers: one launch pair instead of one per head.
  bool merged = false;
  {
    const mpn_head &b = m->d.bbox_head;
    int total = b.cout; bool same = K >= 1 && K < 7;
    for (int k = 0; k < K; ++k) { same = same && m->cls_heads[k].col_begin == b.col_begin && m->cls_heads[k].col_len == b.col_len; total += m->cls_heads[k].cout; }
    const char *envm = getenv("MPN_MERGE_HEADS");
    if (same && total <= 128 && envm && envm[0] == '1') {
      std::vector<const mpn_head *> hs;
      for (int k = 0; k < K; ++k) hs.push_back(&m->cls_heads[k]);
      hs.push_back(&b);
      if (m->merged_w < 0 || m->merged_stale) {
        // concatenate the split weight planes [cout_k][col_len] and the biases once (again after a head's master was set)
        const size_t Kc = (size_t)b.col_len;
        if (m->merged_w < 0) {
          m->weights.emplace_back(new WeightDev()); m->w_elems.push_back((int64_t)total * Kc); m->w_prepared.push_back(1); m->w_host_small.emplace_back();
          m->merged_w = (int)m->weights.size() - 1;
          m->weights.emplace_back(new WeightDev()); m->w_elems.push_back(total); m->w_prepared.push_back(0); m->w_host_small.emplace_back();
          m->merged_b = (int)m->weights.size() - 1;
        }
        m->merged_stale = false;
        WeightDev &mw = *m->weights[m->merged_w], &mb = *m->weights[m->merged_b];
        mw.n = (int64_t)total * Kc; mb.n = total;
        MPN_TRY(mw.hi.ensure(ctx, mw.n * 2 + 256)); MPN_TRY(mw.lo.ensure(ctx, mw.n * 2 + 256));
        MPN_TRY(mb.f32.ensure(ctx, sizeof(float) * total));
        MPN_CUDA(ctx, cudaMemsetAsync(mb.f32.p, 0, sizeof(float) * total, ctx->stream));
        size_t row = 0;
        for (const mpn_head *h : hs) {
          MPN_TRY(prepare_conv_weight(m, h->weight, h->cout, h->col_len, 1, 1));
          const WeightDev &w = *m->weights[h->weight];
          MPN_CUDA(ctx, cudaMemcpyAsync((char *)mw.hi.p + row * Kc * 2, w.hi.p, (size_t)h->cout * Kc * 2, cudaMemcpyDeviceToDevice, ctx->stream));
          MPN_CUDA(ctx, cudaMemcpyAsync((char *)mw.lo.p + row * Kc * 2, w.lo.p, (size_t)h->cout * Kc * 2, cudaMemcpyDeviceToDevice, ctx->stream));
          if (h->bias >= 0)
            MPN_CUDA(ctx, cudaMemcpyAsync((float *)mb.f32.p + row, m->weights[h->bias]->f32.p, sizeof(float) * h->cout, cudaMemcpyDeviceToDevice, ctx->stream));
          row += (size_t)h->cout;
        }
      }
      mpn_head mh = b; mh.cout = total; mh.weight = m->merged_w; mh.bias = m->merged_b;
      MPN_TRY(add_head(mh, (float *)m->bbox_raw.p));            // the dense destination below replaces this pointer
      LayerExec &e = m->head_exec.back();
      if (e.plan.splitk > 1) {
        OutScatter sc; int c0 = 0;
        for (int k = 0; k < K; ++k) { sc.seg[sc.n++] = OutSeg{c0, c0 + C, (float *)m->cls_logits.p + (size_t)k * R * C, (long long)C}; c0 += C; }
        sc.seg[sc.n++] = OutSeg{c0, c0 + 4 * C, (float *)m->bbox_raw.p, (long long)4 * C};
        e.prob.scatter = sc;
        merged = true;
      } else {
        m->head_exec.pop_back();                                 // small K: no split-K plan, keep one GEMM per head
        m->head_flops -= 2.0 * (double)mh.col_len * mh.cout * (double)R;
      }
    }
  }
  if (!merged) {
    for (int k = 0; k < K; ++k) MPN_TRY(add_head(m->cls_heads[k], (float *)m->cls_logits.p + (size_t)k * R * C));
    MPN_TRY(add_head(m->d.bbox_head, (float *)m->bbox_raw.p));
  }
  // post-processing buffers
  MPN_TRY(m->sb_dev.ensure(ctx, sizeof(float) * (size_t)(C - 1) * R * 5 + 256));
  MPN_TRY(m->src_idx_dev.ensure(ctx, sizeof(int32_t) * (size_t)(C - 1) * R + 256));
  MPN_TRY(m->counts_dev.ensure(ctx, sizeof(int32_t) * (size_t)C + 256));
  MPN_TRY(m->keep_idx_dev.ensure(ctx, sizeof(int32_t) * (size_t)(C - 1) * R + 256));
  MPN_TRY(m->keep_counts_dev.ensure(ctx, sizeof(int32_t) * (size_t)C + 256));
  m->hR = R; m->heads_planned = true;
  return MPN_OK;
}

// towers + heads on the pooled rows; tr: the training forward — nn.Dropout after the ReLU of every per-ROI Linear
int run_towers_heads(mpn_model *m, int64_t R, const TrainState *tr = nullptr) {
  mpn_ctx *ctx = m->ctx;
  for (size_t t = 0; t < m->towers.size(); ++t) {
    for (size_t li = 0; li < m->tex[t].layers.size(); ++li) {
      LayerExec &e = m->tex[t].layers[li];
      switch (e.L.kind) {
        case MPN_LAYER_CONV:
          MPN_TRY(run_conv(m, e));
          if (tr && tr->cfg.dropout > 0.f && e.L.relu && e.out.H == 1 && e.out.W == 1)
            MPN_TRY(mpn_train_dropout_launch(ctx, e.out, R, e.L.cout, tr->cfg.seed, tr->step, (int)t, (int)li, tr->cfg.dropout));
          break;
        case MPN_LAYER_FLATTEN: break;
        case MPN_LAYER_AVGPOOL: MPN_TRY(mpn_avgpool_launch(ctx, e.in, e.out)); break;
        case MPN_LAYER_MAXPOOL: MPN_TRY(mpn_maxpool_launch(ctx, e.in, e.L.kh, e.L.stride, e.L.pad, e.out)); break;
        default: return mpn_fail(ctx, MPN_ERR_ARG, "bad tower layer");
      }
    }
  }
  // training: only the selected class head's logits reach the criteria (nn.SelectTable), the idle heads' GEMMs are skipped
  const size_t K = m->cls_heads.size();
  for (size_t i = 0; i < m->head_exec.size(); ++i)
    if (!tr || i >= K || (int)i == tr->head) MPN_TRY(run_conv(m, m->head_exec[i]));
  return MPN_OK;
}

int run_heads(mpn_model *m, const float *rois_dev, int64_t R, bool apply_bbox_norm = true) {
  mpn_ctx *ctx = m->ctx;
  const mpn_tower &T0 = m->towers[0];
  MPN_TRY(mpn_roi_pool_fused_launch(ctx, m->jobs, rois_dev, R, T0.pooled_w, T0.pooled_h, m->d.roi_variant));
  MPN_TRY(run_towers_heads(m, R));
  if (m->d.has_bbox_norm && apply_bbox_norm)
    MPN_TRY(mpn_bbox_norm_launch(ctx, (float *)m->bbox_raw.p, R, 4 * m->d.num_classes, m->d.bbox_mean, m->d.bbox_std));
  return MPN_OK;
}

// the trained weights' derived planes (split / fp16 / e4m3) are rebuilt from the fp32 masters by the next plan, exactly
// as a model built from those weights would build them
void forget_derived_planes(mpn_model *m) {
  for (const TrainParam &p : m->train->params)
    if (!p.bias) { m->w_prepared[p.w] = 0; m->weights[p.w]->has8 = false; }
  if (m->train->trunk_from > 0) { m->tH = 0; m->tW = 0; }     // the trunk plan re-derives its trained planes too
}
// a trunk plan made by a bf16 training step is not an inference plan, nor the reverse. Leaving a bf16 step's plan for
// inference, the trained weights' lo planes (which the step's updates did not write) are derived again from the masters.
// That drops the planes the training heads plan reads too, so that plan is given up (plan_trunk also unsets
// heads_planned): the next step plans its heads again, and the next inference heads call plans its own.
int ensure_trunk(mpn_model *m, int H, int W) {
  const bool scheme = m->trunk_train_bf16 != m->plan_train_bf16;
  if (scheme && m->trunk_train_bf16 && m->train) {
    forget_derived_planes(m);
    m->train->plan = false;
  }
  if (m->trunk_exec.empty() || m->tH != H || m->tW != W || scheme) MPN_TRY(plan_trunk(m, H, W));
  return MPN_OK;
}
int ensure_heads(mpn_model *m, int64_t R) {
  mpn_ctx *ctx = m->ctx;
  MPN_CHECK_ARG(ctx, !m->trunk_exec.empty(), "heads called before any trunk forward (ImageDetect.lua:95 asserts the same)");
  MPN_CHECK_ARG(ctx, R > 0 && R <= m->d.max_rois, "R out of range (0 < R <= max_rois)");
  const bool from_training = m->train && m->train->plan;
  if (!m->heads_planned || m->hR != R || from_training) {
    if (from_training) { forget_derived_planes(m); m->train->plan = false; }
    MPN_TRY(plan_heads(m, R));
  }
  return MPN_OK;
}

}  // namespace

// ================================================================== C ABI
extern "C" {

int mpn_model_create(mpn_ctx *ctx, const mpn_model_desc *desc, const float *const *weights, const int64_t *n_elem,
                     int32_t n_weights, mpn_model **out) {
  if (!ctx || !desc || !out) return MPN_ERR_ARG;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, desc->n_towers >= 1 && desc->n_trunk_layers >= 1 && desc->n_cls_heads >= 1, "empty model description");
  MPN_CHECK_ARG(ctx, desc->num_classes >= 2, "num_classes must be >= 2");
  MPN_CHECK_ARG(ctx, desc->roi_variant == 1 || desc->roi_variant == 2, "roi_variant must be 1 or 2");
  mpn_model *m = new mpn_model();
  m->ctx = ctx; m->d = *desc;
  m->trunk_layers.assign(desc->trunk_layers, desc->trunk_layers + desc->n_trunk_layers);
  m->tower_layers.assign(desc->tower_layers, desc->tower_layers + desc->n_tower_layers);
  m->towers.assign(desc->towers, desc->towers + desc->n_towers);
  m->cls_heads.assign(desc->cls_heads, desc->cls_heads + desc->n_cls_heads);
  m->d.trunk_layers = nullptr; m->d.tower_layers = nullptr; m->d.towers = nullptr; m->d.cls_heads = nullptr;
  for (size_t t = 1; t < m->towers.size(); ++t) {
    if (m->towers[t].pooled_w != m->towers[0].pooled_w || m->towers[t].pooled_h != m->towers[0].pooled_h) {
      delete m; return mpn_fail(ctx, MPN_ERR_ARG, "all towers must share the pooled size");
    }
  }
  m->weights.resize(n_weights); m->w_elems.assign(n_elem, n_elem + n_weights); m->w_prepared.assign(n_weights, 0);
  m->w_host_small.resize(n_weights);
  for (int i = 0; i < n_weights; ++i) {
    if (n_elem[i] <= 4096) m->w_host_small[i].assign(weights[i], weights[i] + n_elem[i]);
    m->weights[i].reset(new WeightDev());
    int r = upload_weight_raw(m, i, weights[i], n_elem[i]);
    if (r != MPN_OK) { delete m; return r; }
  }
  // the host arrays may be freed by the caller once we return
  cudaError_t e = cudaStreamSynchronize(ctx->stream);
  if (e != cudaSuccess) { delete m; return mpn_fail(ctx, MPN_ERR_CUDA, cudaGetErrorString(e)); }
  *out = m;
  return MPN_OK;
}

void mpn_model_destroy(mpn_model *m) {
  if (!m) return;
  cudaSetDevice(m->ctx->device);
  cudaStreamSynchronize(m->ctx->stream);
  if (m->s_d2h) cudaStreamSynchronize(m->s_d2h);
  delete m;
}

int mpn_model_set_conv_impl(mpn_model *m, int32_t impl) {
  if (!m) return MPN_ERR_ARG;
  MPN_CHECK_ARG(m->ctx, impl >= 0 && impl <= 2, "impl must be 0 (wgmma engine), 1 (fp32 check kernel) or 2 (wgmma engine without conv+pool fusion)");
  m->conv_impl = impl;
  return MPN_OK;
}

int mpn_model_last_flops(const mpn_model *m, double *trunk_flops, double *head_flops) {
  if (!m) return MPN_ERR_ARG;
  if (trunk_flops) *trunk_flops = m->trunk_flops;
  if (head_flops) *head_flops = m->head_flops;
  return MPN_OK;
}

int mpn_model_trunk_dev(mpn_model *m, const float *image_dev, int32_t H, int32_t W) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, image_dev && H > 0 && W > 0 && H <= m->d.max_h && W <= m->d.max_w, "image missing or larger than max_h x max_w");
  MPN_TRY(ensure_trunk(m, H, W));
  return run_trunk(m, image_dev);
}

int mpn_model_trunk(mpn_model *m, const float *image, int32_t H, int32_t W) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, image && H > 0 && W > 0, "image missing");
  const size_t bytes = sizeof(float) * 3 * (size_t)H * W;
  MPN_TRY(m->image_dev.ensure(ctx, bytes));
  MPN_CUDA(ctx, cudaMemcpyAsync(m->image_dev.p, image, bytes, cudaMemcpyHostToDevice, ctx->stream));
  MPN_TRY(mpn_model_trunk_dev(m, (const float *)m->image_dev.p, H, W));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

int mpn_model_trunk_image(mpn_model *m, const float *im, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                          double scale, double max_size, double *im_scale, int32_t *h_out, int32_t *w_out) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, im && tf && H0 > 0 && W0 > 0, "image or transformer missing");
  int32_t h = 0, w = 0; double s = 0;
  MPN_CHECK_ARG(ctx, mpn_get_images_size_impl(H0, W0, scale, max_size, &h, &w, &s) == MPN_OK && h > 0 && w > 0, "bad scale / max_size");
  MPN_CHECK_ARG(ctx, h <= m->d.max_h && w <= m->d.max_w, "scaled image larger than max_h x max_w");
  const size_t braw = sizeof(float) * 3 * (size_t)H0 * W0, bimg = sizeof(float) * 3 * (size_t)h * w;
  MPN_TRY(m->raw_image_dev.ensure(ctx, braw));
  MPN_TRY(m->image_dev.ensure(ctx, bimg));
  MPN_CUDA(ctx, cudaMemcpyAsync(m->raw_image_dev.p, im, braw, cudaMemcpyHostToDevice, ctx->stream));
  MPN_TRY(mpn_get_images_launch(ctx, (const float *)m->raw_image_dev.p, H0, W0, tf, h, w, (float *)m->image_dev.p));
  MPN_TRY(mpn_model_trunk_dev(m, (const float *)m->image_dev.p, h, w));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  if (im_scale) *im_scale = s;
  if (h_out) *h_out = h;
  if (w_out) *w_out = w;
  return MPN_OK;
}

int mpn_model_heads_dev(mpn_model *m, const float *rois_dev, int64_t R, float *cls_out_dev, float *bbox_out_dev) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->trunk_valid, "heads called before a trunk forward");
  MPN_TRY(ensure_heads(m, R));
  MPN_TRY(run_heads(m, rois_dev, R));
  const int C = m->d.num_classes, K = (int)m->cls_heads.size();
  if (cls_out_dev) {
    if (K == 1) {   // a single head's own output: what the Linear produced (the same rule as detect: any softmax is applied there)
      MPN_CUDA(ctx, cudaMemcpyAsync(cls_out_dev, m->cls_logits.p, sizeof(float) * (size_t)R * C, cudaMemcpyDeviceToDevice, ctx->stream));
    } else {   // integral head: the model's own output is the mean of K softmaxes
      MPN_TRY(mpn_softmax_mean_launch(ctx, (const float *)m->cls_logits.p, R, C, K, 1, cls_out_dev));
    }
  }
  if (bbox_out_dev)
    MPN_CUDA(ctx, cudaMemcpyAsync(bbox_out_dev, m->bbox_raw.p, sizeof(float) * (size_t)R * 4 * C, cudaMemcpyDeviceToDevice, ctx->stream));
  return MPN_OK;
}

int mpn_model_heads(mpn_model *m, const float *rois, int64_t R, float *cls_out, float *bbox_out) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, rois && R > 0, "rois missing");
  const int C = m->d.num_classes;
  MPN_TRY(m->rois_dev.ensure(ctx, sizeof(float) * 5 * (size_t)R));
  MPN_CUDA(ctx, cudaMemcpyAsync(m->rois_dev.p, rois, sizeof(float) * 5 * (size_t)R, cudaMemcpyHostToDevice, ctx->stream));
  MPN_TRY(ensure_heads(m, R));
  MPN_TRY(mpn_model_heads_dev(m, (const float *)m->rois_dev.p, R, (float *)m->scores_dev.p, nullptr));
  if (cls_out) MPN_CUDA(ctx, cudaMemcpyAsync(cls_out, m->scores_dev.p, sizeof(float) * (size_t)R * C, cudaMemcpyDeviceToHost, ctx->stream));
  if (bbox_out) MPN_CUDA(ctx, cudaMemcpyAsync(bbox_out, m->bbox_raw.p, sizeof(float) * (size_t)R * 4 * C, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_TRY(mpn_ovf_copy_async(ctx, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return mpn_ovf_test(ctx);
}

// one detect pass on the cached trunk features: project_im_rois -> heads -> scores (softmax / integral mean) | BBoxNorm +
// decode (+ clamp) into caller-chosen buffers (ImageDetect.lua:161-192 after getImages; Tester_FRCNN.lua:75-78 clamp)
static int run_detect_pass(mpn_model *m, const float *boxes_dev, int64_t R, float im_scale, int do_clamp, float W0, float H0,
                           float *scores_dst, float *bboxes_dst) {
  mpn_ctx *ctx = m->ctx;
  const int C = m->d.num_classes, K = (int)m->cls_heads.size();
  MPN_TRY(ensure_heads(m, R));
  MPN_TRY(m->rois_dev.ensure(ctx, sizeof(float) * 5 * (size_t)R));
  MPN_TRY(mpn_project_rois_launch(ctx, boxes_dev, R, im_scale, (float *)m->rois_dev.p));
  MPN_TRY(run_heads(m, (const float *)m->rois_dev.p, R, /*apply_bbox_norm=*/false));
  // class_values: softmax unless model.noSoftMax; an integral head IS its mean of softmaxes (noSoftMax=true).
  // One launch: softmax (+mean) | BBoxNorm + decode (+ clamp to the image for the NMS path, Tester_FRCNN.lua:75-78)
  const int do_softmax = (K > 1) ? 1 : (m->d.no_softmax ? 0 : 1);
  return mpn_detect_tail_launch(ctx, (const float *)m->cls_logits.p, R, C, K, do_softmax, scores_dst, (const float *)m->bbox_raw.p, boxes_dev,
                                do_clamp, W0, H0, bboxes_dst, m->d.has_bbox_norm ? 1 : 0, m->d.bbox_mean, m->d.bbox_std);
}

// shared tail: heads -> scores (softmax / integral mean) -> decode (+clamp) [-> gather -> NMS]
static int detect_tail_dev(mpn_model *m, const float *boxes_dev, int64_t R, float im_scale, int do_nms, float W0,
                           float H0, float score_thresh, float nms_thr) {
  mpn_ctx *ctx = m->ctx;
  const int C = m->d.num_classes;
  MPN_TRY(ensure_heads(m, R));
  MPN_TRY(run_detect_pass(m, boxes_dev, R, im_scale, do_nms, W0, H0, (float *)m->scores_dev.p, (float *)m->bboxes_dev.p));
  if (do_nms) {
    MPN_TRY(mpn_gather_scored_launch(ctx, (const float *)m->scores_dev.p, (const float *)m->bboxes_dev.p, (int)R, C,
                                     score_thresh, (float *)m->sb_dev.p, (int32_t *)m->src_idx_dev.p, (int32_t *)m->counts_dev.p));
    MPN_TRY(mpn_nms_launch(ctx, (const float *)m->sb_dev.p, (int)R, C - 1, (const int32_t *)m->counts_dev.p,
                           (const int32_t *)m->src_idx_dev.p, nms_thr, (int32_t *)m->keep_idx_dev.p,
                           (int32_t *)m->keep_counts_dev.p));
    if (m->sink) {     // keep_top_k + fixed-size record of this image, appended to the caller's sink (SURVEY 8e)
      MPN_CHECK_ARG(ctx, m->sink_n < m->sink_cap, "detection sink is full (mpn_model_set_detection_sink capacity)");
      MPN_TRY(mpn_pack_detections_launch(ctx, (const float *)m->scores_dev.p, (const float *)m->bboxes_dev.p, C,
                                         (const int32_t *)m->keep_idx_dev.p, (const int32_t *)m->keep_counts_dev.p, (int)R,
                                         m->sink_top_k, m->sink + (size_t)m->sink_n * MPN_REC_FLOATS));
      ++m->sink_n;
    }
  }
  return MPN_OK;
}

int mpn_model_detect(mpn_model *m, const float *image, int32_t H, int32_t W, const float *boxes, int64_t R,
                     float im_scale, int32_t recompute_features, float *scores, float *bboxes) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, boxes && R > 0, "boxes missing");
  const int C = m->d.num_classes;
  if (recompute_features) {
    MPN_CHECK_ARG(ctx, image, "image missing");
    const size_t bytes = sizeof(float) * 3 * (size_t)H * W;
    MPN_TRY(m->image_dev.ensure(ctx, bytes));
    MPN_CUDA(ctx, cudaMemcpyAsync(m->image_dev.p, image, bytes, cudaMemcpyHostToDevice, ctx->stream));
    MPN_TRY(mpn_model_trunk_dev(m, (const float *)m->image_dev.p, H, W));
  } else {
    MPN_CHECK_ARG(ctx, m->trunk_valid, "recompute_features=false needs cached trunk features (ImageDetect.lua:109-111)");
  }
  MPN_TRY(m->boxes_dev.ensure(ctx, sizeof(float) * 4 * (size_t)R));
  MPN_CUDA(ctx, cudaMemcpyAsync(m->boxes_dev.p, boxes, sizeof(float) * 4 * (size_t)R, cudaMemcpyHostToDevice, ctx->stream));
  MPN_TRY(detect_tail_dev(m, (const float *)m->boxes_dev.p, R, im_scale, 0, 0.f, 0.f, 0.f, 0.f));
  if (scores) MPN_CUDA(ctx, cudaMemcpyAsync(scores, m->scores_dev.p, sizeof(float) * (size_t)R * C, cudaMemcpyDeviceToHost, ctx->stream));
  if (bboxes) MPN_CUDA(ctx, cudaMemcpyAsync(bboxes, m->bboxes_dev.p, sizeof(float) * (size_t)R * 4 * C, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_TRY(mpn_ovf_copy_async(ctx, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return mpn_ovf_test(ctx);
}

int mpn_model_detect_nms_dev(mpn_model *m, const float *image_dev, int32_t H, int32_t W, const float *boxes_dev,
                             int64_t R, float im_scale, float W0, float H0, float score_thresh, float nms_thr,
                             float *scores_dev, float *bboxes_dev, int32_t *keep_idx_dev, int32_t *keep_counts_dev) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, image_dev && boxes_dev && R > 0, "image/boxes missing");
  const int C = m->d.num_classes;
  MPN_TRY(mpn_model_trunk_dev(m, image_dev, H, W));
  MPN_TRY(detect_tail_dev(m, boxes_dev, R, im_scale, 1, W0, H0, score_thresh, nms_thr));
  if (scores_dev) MPN_CUDA(ctx, cudaMemcpyAsync(scores_dev, m->scores_dev.p, sizeof(float) * (size_t)R * C, cudaMemcpyDeviceToDevice, ctx->stream));
  if (bboxes_dev) MPN_CUDA(ctx, cudaMemcpyAsync(bboxes_dev, m->bboxes_dev.p, sizeof(float) * (size_t)R * 4 * C, cudaMemcpyDeviceToDevice, ctx->stream));
  if (keep_idx_dev) MPN_CUDA(ctx, cudaMemcpyAsync(keep_idx_dev, m->keep_idx_dev.p, sizeof(int32_t) * (size_t)(C - 1) * R, cudaMemcpyDeviceToDevice, ctx->stream));
  if (keep_counts_dev) MPN_CUDA(ctx, cudaMemcpyAsync(keep_counts_dev, m->keep_counts_dev.p, sizeof(int32_t) * (size_t)(C - 1), cudaMemcpyDeviceToDevice, ctx->stream));
  return MPN_OK;
}

int mpn_model_detect_nms(mpn_model *m, const float *image, int32_t H, int32_t W, const float *boxes, int64_t R,
                         float im_scale, float W0, float H0, float score_thresh, float nms_thr, float *scores,
                         float *bboxes, int32_t *keep_idx, int32_t *keep_counts) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, image && boxes && R > 0, "image/boxes missing");
  const int C = m->d.num_classes;
  const size_t bytes = sizeof(float) * 3 * (size_t)H * W;
  MPN_TRY(m->image_dev.ensure(ctx, bytes));
  MPN_TRY(m->boxes_dev.ensure(ctx, sizeof(float) * 4 * (size_t)R));
  MPN_CUDA(ctx, cudaMemcpyAsync(m->image_dev.p, image, bytes, cudaMemcpyHostToDevice, ctx->stream));
  MPN_CUDA(ctx, cudaMemcpyAsync(m->boxes_dev.p, boxes, sizeof(float) * 4 * (size_t)R, cudaMemcpyHostToDevice, ctx->stream));
  MPN_TRY(mpn_model_trunk_dev(m, (const float *)m->image_dev.p, H, W));
  MPN_TRY(detect_tail_dev(m, (const float *)m->boxes_dev.p, R, im_scale, 1, W0, H0, score_thresh, nms_thr));
  if (scores) MPN_CUDA(ctx, cudaMemcpyAsync(scores, m->scores_dev.p, sizeof(float) * (size_t)R * C, cudaMemcpyDeviceToHost, ctx->stream));
  if (bboxes) MPN_CUDA(ctx, cudaMemcpyAsync(bboxes, m->bboxes_dev.p, sizeof(float) * (size_t)R * 4 * C, cudaMemcpyDeviceToHost, ctx->stream));
  if (keep_idx) MPN_CUDA(ctx, cudaMemcpyAsync(keep_idx, m->keep_idx_dev.p, sizeof(int32_t) * (size_t)(C - 1) * R, cudaMemcpyDeviceToHost, ctx->stream));
  if (keep_counts) MPN_CUDA(ctx, cudaMemcpyAsync(keep_counts, m->keep_counts_dev.p, sizeof(int32_t) * (size_t)(C - 1), cudaMemcpyDeviceToHost, ctx->stream));
  MPN_TRY(mpn_ovf_copy_async(ctx, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return mpn_ovf_test(ctx);
}

// image != null: the transformed + scaled fp32 image (H x W); else raw_u8: the RAW H0 x W0 x 3 byte image, transformed and
// scaled on the device (get_images_kernel) to the size getImages prescribes
static int submit_common(mpn_model *m, const float *image, int32_t H, int32_t W, const uint8_t *raw_u8, int32_t H0r, int32_t W0r,
                         const mpn_image_transform *tf, double scale, double max_size, const float *boxes, int64_t R, float im_scale,
                         float W0, float H0, float score_thresh, float nms_thr, float *scores, float *bboxes, int32_t *keep_idx,
                         int32_t *keep_counts, int32_t *ticket) {
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, (image || raw_u8) && boxes && R > 0 && ticket, "image/boxes/ticket missing");
  const int C = m->d.num_classes;
  mpn_model::PipeSlot &q = m->pipe[m->next_ticket & 1];
  if (q.busy) return mpn_fail(ctx, MPN_ERR_STATE, "two submissions are already in flight: call mpn_model_detect_nms_wait first");
  if (!m->s_h2d) {
    MPN_CUDA(ctx, cudaStreamCreateWithFlags(&m->s_h2d, cudaStreamNonBlocking));
    MPN_CUDA(ctx, cudaStreamCreateWithFlags(&m->s_d2h, cudaStreamNonBlocking));
  }
  if (!q.h2d) {
    MPN_CUDA(ctx, cudaEventCreateWithFlags(&q.h2d, cudaEventDisableTiming));
    MPN_CUDA(ctx, cudaEventCreateWithFlags(&q.compute, cudaEventDisableTiming));
    MPN_CUDA(ctx, cudaEventCreateWithFlags(&q.done, cudaEventDisableTiming));
  }
  if (raw_u8) {
    MPN_CHECK_ARG(ctx, tf && H0r > 0 && W0r > 0, "raw image: transformer / size missing");
    double s = 0;
    MPN_CHECK_ARG(ctx, mpn_get_images_size_impl(H0r, W0r, scale, max_size, &H, &W, &s) == MPN_OK && H > 0 && W > 0, "bad scale / max_size");
    MPN_CHECK_ARG(ctx, H <= m->d.max_h && W <= m->d.max_w, "scaled image larger than max_h x max_w");
    im_scale = (float)s; W0 = (float)W0r; H0 = (float)H0r;          // clamp to the ORIGINAL image (Tester_FRCNN.lua:75-78)
  }
  const size_t img_bytes = sizeof(float) * 3 * (size_t)H * W;
  MPN_TRY(q.image.ensure(ctx, img_bytes));
  MPN_TRY(q.boxes.ensure(ctx, sizeof(float) * 4 * (size_t)R));
  MPN_TRY(q.scores.ensure(ctx, sizeof(float) * (size_t)R * C));
  MPN_TRY(q.bboxes.ensure(ctx, sizeof(float) * (size_t)R * 4 * C));
  MPN_TRY(q.keep_idx.ensure(ctx, sizeof(int32_t) * (size_t)(C - 1) * R));
  MPN_TRY(q.keep_counts.ensure(ctx, sizeof(int32_t) * (size_t)(C - 1)));
  // inputs: the slot's previous occupant was waited for (busy == false), so its staging buffers are free
  if (raw_u8) {
    MPN_TRY(q.raw_u8.ensure(ctx, (size_t)H0r * W0r * 3));
    MPN_CUDA(ctx, cudaMemcpyAsync(q.raw_u8.p, raw_u8, (size_t)H0r * W0r * 3, cudaMemcpyHostToDevice, m->s_h2d));
  } else {
    MPN_CUDA(ctx, cudaMemcpyAsync(q.image.p, image, img_bytes, cudaMemcpyHostToDevice, m->s_h2d));
  }
  MPN_CUDA(ctx, cudaMemcpyAsync(q.boxes.p, boxes, sizeof(float) * 4 * (size_t)R, cudaMemcpyHostToDevice, m->s_h2d));
  MPN_CUDA(ctx, cudaEventRecord(q.h2d, m->s_h2d));
  MPN_CUDA(ctx, cudaStreamWaitEvent(ctx->stream, q.h2d, 0));
  if (raw_u8) MPN_TRY(mpn_get_images_u8_launch(ctx, (const uint8_t *)q.raw_u8.p, H0r, W0r, tf, H, W, (float *)q.image.p));
  MPN_TRY(mpn_model_detect_nms_dev(m, (const float *)q.image.p, H, W, (const float *)q.boxes.p, R, im_scale, W0, H0, score_thresh,
                                   nms_thr, scores ? (float *)q.scores.p : nullptr, bboxes ? (float *)q.bboxes.p : nullptr,
                                   keep_idx ? (int32_t *)q.keep_idx.p : nullptr, keep_counts ? (int32_t *)q.keep_counts.p : nullptr));
  MPN_CUDA(ctx, cudaEventRecord(q.compute, ctx->stream));
  MPN_CUDA(ctx, cudaStreamWaitEvent(m->s_d2h, q.compute, 0));
  if (scores) MPN_CUDA(ctx, cudaMemcpyAsync(scores, q.scores.p, sizeof(float) * (size_t)R * C, cudaMemcpyDeviceToHost, m->s_d2h));
  if (bboxes) MPN_CUDA(ctx, cudaMemcpyAsync(bboxes, q.bboxes.p, sizeof(float) * (size_t)R * 4 * C, cudaMemcpyDeviceToHost, m->s_d2h));
  if (keep_idx) MPN_CUDA(ctx, cudaMemcpyAsync(keep_idx, q.keep_idx.p, sizeof(int32_t) * (size_t)(C - 1) * R, cudaMemcpyDeviceToHost, m->s_d2h));
  if (keep_counts) MPN_CUDA(ctx, cudaMemcpyAsync(keep_counts, q.keep_counts.p, sizeof(int32_t) * (size_t)(C - 1), cudaMemcpyDeviceToHost, m->s_d2h));
  MPN_TRY(mpn_ovf_copy_async(ctx, m->s_d2h));
  MPN_CUDA(ctx, cudaEventRecord(q.done, m->s_d2h));
  q.busy = true; q.ticket = m->next_ticket;
  *ticket = m->next_ticket++;
  return MPN_OK;
}

int mpn_model_detect_nms_submit(mpn_model *m, const float *image, int32_t H, int32_t W, const float *boxes, int64_t R,
                                float im_scale, float W0, float H0, float score_thresh, float nms_thr, float *scores,
                                float *bboxes, int32_t *keep_idx, int32_t *keep_counts, int32_t *ticket) {
  if (!m) return MPN_ERR_ARG;
  MPN_CHECK_ARG(m->ctx, image, "image missing");
  return submit_common(m, image, H, W, nullptr, 0, 0, nullptr, 0, 0, boxes, R, im_scale, W0, H0, score_thresh, nms_thr, scores, bboxes,
                       keep_idx, keep_counts, ticket);
}

int mpn_model_detect_nms_submit_u8(mpn_model *m, const uint8_t *im_hwc, int32_t H0, int32_t W0, const mpn_image_transform *tf,
                                   double scale, double max_size, const float *boxes, int64_t R, float score_thresh, float nms_thr,
                                   float *scores, float *bboxes, int32_t *keep_idx, int32_t *keep_counts, int32_t *ticket) {
  if (!m) return MPN_ERR_ARG;
  MPN_CHECK_ARG(m->ctx, im_hwc, "image missing");
  return submit_common(m, nullptr, 0, 0, im_hwc, H0, W0, tf, scale, max_size, boxes, R, 0.f, 0.f, 0.f, score_thresh, nms_thr, scores, bboxes,
                       keep_idx, keep_counts, ticket);
}

int mpn_model_detect_nms_wait(mpn_model *m, int32_t ticket) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  mpn_model::PipeSlot &q = m->pipe[ticket & 1];
  MPN_CHECK_ARG(ctx, ticket >= 0 && q.busy && q.ticket == ticket, "unknown or already completed ticket");
  MPN_CUDA(ctx, cudaEventSynchronize(q.done));
  q.busy = false;
  return mpn_ovf_test(ctx);
}

// Tester_FRCNN:testOne (Tester_FRCNN.lua:54-139) entirely on the device: see include/mpn_abi.h
int mpn_model_test_one(mpn_model *m, const float *image, int32_t H, int32_t W, const float *boxes, int64_t R, float im_scale, float W0,
                       float H0, const mpn_test_opts *o, float *scores, float *bboxes, int32_t *keep_idx, int32_t *keep_counts, float *voted) {
  if (!m || !o) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, image && boxes && R > 0, "image/boxes missing");
  MPN_CHECK_ARG(ctx, o->num_iter >= 1 && o->num_iter <= 8, "num_iter must be in 1..8");
  MPN_CHECK_ARG(ctx, !o->use_rbox_scores || o->num_iter > 1, "test_use_rbox_scores needs test_num_iterative_loc > 1 (Tester_FRCNN.lua:92)");
  MPN_CHECK_ARG(ctx, !o->bbox_voting || voted, "bbox voting needs the `voted` output");
  const int C = m->d.num_classes, n_it = o->num_iter;
  const int64_t n_out = R * (n_it - (o->use_rbox_scores ? 1 : 0));        // rows of the joined outputs
  MPN_CHECK_ARG(ctx, n_out < (1ll << 30), "too many rows");
  const size_t bs = sizeof(float) * (size_t)R * C, bb = sizeof(float) * (size_t)R * 4 * C;
  MPN_TRY(m->image_dev.ensure(ctx, sizeof(float) * 3 * (size_t)H * W));
  MPN_TRY(m->boxes_dev.ensure(ctx, sizeof(float) * 4 * (size_t)R));
  MPN_TRY(m->to_pass_scores.ensure(ctx, bs * n_it)); MPN_TRY(m->to_pass_bboxes.ensure(ctx, bb * n_it));
  MPN_TRY(m->to_new_boxes.ensure(ctx, sizeof(float) * 4 * (size_t)R));
  MPN_TRY(m->to_scores.ensure(ctx, sizeof(float) * (size_t)n_out * C)); MPN_TRY(m->to_bboxes.ensure(ctx, sizeof(float) * (size_t)n_out * 4 * C));
  MPN_TRY(m->to_sb.ensure(ctx, sizeof(float) * 5 * (size_t)(C - 1) * n_out)); MPN_TRY(m->to_src.ensure(ctx, sizeof(int32_t) * (size_t)(C - 1) * n_out));
  MPN_TRY(m->to_counts.ensure(ctx, sizeof(int32_t) * (size_t)C)); MPN_TRY(m->to_keep.ensure(ctx, sizeof(int32_t) * (size_t)(C - 1) * n_out));
  MPN_TRY(m->to_keep_counts.ensure(ctx, sizeof(int32_t) * (size_t)C));
  if (o->bbox_voting) MPN_TRY(m->to_voted.ensure(ctx, sizeof(float) * 5 * (size_t)(C - 1) * n_out));
  MPN_CUDA(ctx, cudaMemcpyAsync(m->image_dev.p, image, sizeof(float) * 3 * (size_t)H * W, cudaMemcpyHostToDevice, ctx->stream));
  MPN_CUDA(ctx, cudaMemcpyAsync(m->boxes_dev.p, boxes, sizeof(float) * 4 * (size_t)R, cudaMemcpyHostToDevice, ctx->stream));
  MPN_TRY(mpn_model_trunk_dev(m, (const float *)m->image_dev.p, H, W));
  auto ps = [&](int it) { return (float *)((char *)m->to_pass_scores.p + bs * it); };
  auto pb = [&](int it) { return (float *)((char *)m->to_pass_bboxes.p + bb * it); };
  // pass 1 on the proposals, clamped (:72-78); passes 2..n on nn.SelectBoxes of the previous pass, cached features, NOT clamped (:82-89)
  MPN_TRY(run_detect_pass(m, (const float *)m->boxes_dev.p, R, im_scale, 1, W0, H0, ps(0), pb(0)));
  for (int it = 1; it < n_it; ++it) {
    MPN_TRY(mpn_select_boxes_launch(ctx, ps(it - 1), pb(it - 1), R, C, nullptr, nullptr, (float *)m->to_new_boxes.p));
    MPN_TRY(run_detect_pass(m, (const float *)m->to_new_boxes.p, R, im_scale, 0, 0.f, 0.f, ps(it), pb(it)));
  }
  // joinTable (:99-100); with rbox scores the scores of pass i + 1 go with the boxes of pass i (:91-97)
  const int s0 = o->use_rbox_scores ? 1 : 0, n_blocks = n_it - s0;
  MPN_CUDA(ctx, cudaMemcpyAsync(m->to_scores.p, ps(s0), bs * n_blocks, cudaMemcpyDeviceToDevice, ctx->stream));
  MPN_CUDA(ctx, cudaMemcpyAsync(m->to_bboxes.p, pb(0), bb * n_blocks, cudaMemcpyDeviceToDevice, ctx->stream));
  MPN_TRY(mpn_gather_scored_launch(ctx, (const float *)m->to_scores.p, (const float *)m->to_bboxes.p, (int)n_out, C, o->score_thresh,
                                   (float *)m->to_sb.p, (int32_t *)m->to_src.p, (int32_t *)m->to_counts.p));
  MPN_TRY(mpn_nms_launch(ctx, (const float *)m->to_sb.p, (int)n_out, C - 1, (const int32_t *)m->to_counts.p, (const int32_t *)m->to_src.p,
                         o->nms_thr, (int32_t *)m->to_keep.p, (int32_t *)m->to_keep_counts.p));
  if (o->bbox_voting)
    MPN_TRY(mpn_bbox_vote_batched_launch(ctx, (const float *)m->to_sb.p, (const int32_t *)m->to_counts.p, (const int32_t *)m->to_keep.p,
                                         (const int32_t *)m->to_keep_counts.p, (const float *)m->to_scores.p, (const float *)m->to_bboxes.p, C,
                                         (int)n_out, o->vote_thr, o->vote_score_pow, (float *)m->to_voted.p));
  if (scores) MPN_CUDA(ctx, cudaMemcpyAsync(scores, m->to_scores.p, sizeof(float) * (size_t)n_out * C, cudaMemcpyDeviceToHost, ctx->stream));
  if (bboxes) MPN_CUDA(ctx, cudaMemcpyAsync(bboxes, m->to_bboxes.p, sizeof(float) * (size_t)n_out * 4 * C, cudaMemcpyDeviceToHost, ctx->stream));
  if (keep_idx) MPN_CUDA(ctx, cudaMemcpyAsync(keep_idx, m->to_keep.p, sizeof(int32_t) * (size_t)(C - 1) * n_out, cudaMemcpyDeviceToHost, ctx->stream));
  if (keep_counts) MPN_CUDA(ctx, cudaMemcpyAsync(keep_counts, m->to_keep_counts.p, sizeof(int32_t) * (size_t)(C - 1), cudaMemcpyDeviceToHost, ctx->stream));
  if (voted && o->bbox_voting) MPN_CUDA(ctx, cudaMemcpyAsync(voted, m->to_voted.p, sizeof(float) * 5 * (size_t)(C - 1) * n_out, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_TRY(mpn_ovf_copy_async(ctx, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return mpn_ovf_test(ctx);
}

int mpn_model_set_detection_sink(mpn_model *m, float *records_dev, int64_t capacity, int32_t top_k) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CHECK_ARG(ctx, !records_dev || (capacity > 0 && top_k >= 1 && top_k <= MPN_MAX_DET), "detection sink: capacity > 0 and 1 <= top_k <= MPN_MAX_DET");
  m->sink = records_dev; m->sink_cap = records_dev ? capacity : 0; m->sink_n = 0; m->sink_top_k = records_dev ? top_k : 100;
  return MPN_OK;
}

int mpn_model_detection_sink_count(const mpn_model *m, int64_t *n_records) {
  if (!m || !n_records) return MPN_ERR_ARG;
  *n_records = m->sink_n;
  return MPN_OK;
}

int mpn_model_get_pooled(mpn_model *m, int32_t tower, int64_t r0, int64_t n, float *out, int64_t capacity, int64_t *R_total,
                         int32_t *bins, int32_t *Ctot) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->heads_planned && tower >= 0 && tower < (int)m->tex.size(), "no heads pass yet, or unknown tower");
  const DTensor &t = m->tex[tower].pooled;
  const int64_t row = t.H * t.W * t.C;
  if (R_total) *R_total = t.N;
  if (bins) *bins = (int32_t)(t.H * t.W);
  if (Ctot) *Ctot = (int32_t)t.C;
  if (!out) return MPN_OK;
  MPN_CHECK_ARG(ctx, r0 >= 0 && n > 0 && r0 + n <= t.N && capacity >= n * row, "row range outside the pooled tensor, or buffer too small");
  void *tmp = nullptr;
  MPN_TRY(mpn_scratch(ctx, sizeof(float) * (size_t)(n * row), &tmp));
  MPN_TRY(mpn_join_rows_launch(ctx, t.hi + r0 * row, t.lo + r0 * row, n, row, row, t.fmt, (float *)tmp));
  MPN_CUDA(ctx, cudaMemcpyAsync(out, tmp, sizeof(float) * (size_t)(n * row), cudaMemcpyDeviceToHost, ctx->stream));
  MPN_TRY(mpn_ovf_copy_async(ctx, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return mpn_ovf_test(ctx);
}

int mpn_model_get_trunk_slot(mpn_model *m, int32_t slot, float *out_nchw, int64_t capacity, int32_t *C, int32_t *H,
                             int32_t *W) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->trunk_valid && slot > 0 && m->trunk_slots.count(slot), "unknown trunk slot or no trunk forward yet");
  MPN_CHECK_ARG(ctx, !m->elided_slots.count(slot),
                "trunk slot was fused into the following max pool and never written (mpn_model_set_conv_impl(m, 2) disables the fusion)");
  const DTensor &t = m->trunk_slots[slot];
  const int64_t n = t.N * t.C * t.H * t.W;
  if (C) *C = (int32_t)t.C; if (H) *H = (int32_t)t.H; if (W) *W = (int32_t)t.W;
  if (!out_nchw) return MPN_OK;
  MPN_CHECK_ARG(ctx, capacity >= n, "output buffer too small");
  void *tmp = nullptr;
  MPN_TRY(mpn_scratch(ctx, sizeof(float) * (size_t)n, &tmp));
  MPN_TRY(mpn_nhwc_split_to_nchw_launch(ctx, t, (float *)tmp));
  MPN_CUDA(ctx, cudaMemcpyAsync(out_nchw, tmp, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

int mpn_model_get_slot_planes(mpn_model *m, int32_t tower, int32_t slot, int64_t r0, int64_t n, uint16_t *hi, uint16_t *lo,
                              uint8_t *q8, int32_t *e8, int64_t capacity, int32_t *fmt, int64_t *dims) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  const DTensor *t = nullptr;
  const Fp8Buf *qb = nullptr;        // the slot's e4m3 plane, when an fp8 layer of the current plan reads the slot
  if (tower == -1) {
    MPN_CHECK_ARG(ctx, m->trunk_valid && slot > 0 && m->trunk_slots.count(slot), "unknown trunk slot or no trunk forward yet");
    MPN_CHECK_ARG(ctx, !m->elided_slots.count(slot), "trunk slot was fused into the following max pool and never written");
    t = &m->trunk_slots[slot];
    for (const LayerExec &e : m->trunk_exec)
      if (e.L.kind == MPN_LAYER_CONV && !e.is_direct && e.prob.fp8 && e.L.in_slot == slot) qb = m->trunk_q8[slot].get();
  } else {
    MPN_CHECK_ARG(ctx, m->heads_planned && tower >= 0 && tower < (int)m->tex.size(), "no heads pass yet, or unknown tower");
    mpn_model::TowerExec &X = m->tex[tower];
    MPN_CHECK_ARG(ctx, X.slots.count(slot), "unknown tower slot");
    t = &X.slots[slot];
    auto it = X.q8.find(slot);
    if (it != X.q8.end()) qb = it->second.get();
  }
  const int64_t px = t->H * t->W;        // pixels per sample
  if (fmt) *fmt = t->fmt;
  if (dims) { dims[0] = t->N; dims[1] = t->H; dims[2] = t->W; dims[3] = t->C; }
  if (!hi) return MPN_OK;
  MPN_CHECK_ARG(ctx, lo && r0 >= 0 && n > 0 && r0 + n <= t->N, "rows outside the slot, or lo plane missing");
  MPN_CHECK_ARG(ctx, capacity >= n * px * t->C, "output buffer too small");
  MPN_CHECK_ARG(ctx, !(q8 || e8) || (q8 && e8 && qb), "the current plan keeps no e4m3 plane for this slot");
  // one row per pixel: C values of a ld-strided plane (a concat column slice has ld = the concat width)
  const size_t w = sizeof(uint16_t) * (size_t)t->C, pitch = sizeof(uint16_t) * (size_t)t->ld, rows = (size_t)(n * px);
  const __nv_bfloat16 *src[2] = {t->hi + r0 * px * t->ld, t->lo + r0 * px * t->ld};
  uint16_t *dst[2] = {hi, lo};
  for (int p = 0; p < 2; ++p) {
    if (t->ld == t->C) MPN_CUDA(ctx, cudaMemcpyAsync(dst[p], src[p], w * rows, cudaMemcpyDeviceToHost, ctx->stream));
    else MPN_CUDA(ctx, cudaMemcpy2DAsync(dst[p], w, src[p], pitch, w, rows, cudaMemcpyDeviceToHost, ctx->stream));
  }
  if (q8) {
    MPN_CUDA(ctx, cudaMemcpyAsync(q8, (const uint8_t *)qb->q.p + r0 * px * t->C, (size_t)(n * px * t->C), cudaMemcpyDeviceToHost, ctx->stream));
    MPN_CUDA(ctx, cudaMemcpyAsync(e8, (const int *)qb->e.p + r0, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  }
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

int mpn_model_get_head_outputs(mpn_model *m, float *cls_logits, float *bbox_raw, int64_t *R, int32_t *K) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->heads_planned, "no heads pass yet");
  const int C = m->d.num_classes, nk = (int)m->cls_heads.size();
  if (R) *R = m->hR;
  if (K) *K = nk;
  if (cls_logits)
    MPN_CUDA(ctx, cudaMemcpyAsync(cls_logits, m->cls_logits.p, sizeof(float) * (size_t)nk * m->hR * C, cudaMemcpyDeviceToHost, ctx->stream));
  if (bbox_raw)
    MPN_CUDA(ctx, cudaMemcpyAsync(bbox_raw, m->bbox_raw.p, sizeof(float) * (size_t)m->hR * 4 * C, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

}  // extern "C"

// ================================================================== training: one SGD step of the per-ROI layers, and of the
// trunk from layer trunk_from up when that is > 0 (train.lua:221-370; MultiPathNet's trunk sits under nn.NoBackprop,
// vgg.lua:18-19 freezes conv1_1 .. pool2; see include/mpn_abi.h)

// the number of class heads (K > 1: an integral model); mpn_model_train_step_batch trains head s on threshold set s
int mpn_model_n_cls_heads(const mpn_model *m) { return (int)m->cls_heads.size(); }

// fixed batch norm (mpn_train_spec.n_fixed): a recorded convolution is k x k, k in {1, 3}, stride 1 or 2, pad
// (k - 1) / 2, with or without ReLU and residual, Cout a multiple of 64 (the K blocks of its dgrad GEMM)
static bool fixed_conv_ok(const mpn_layer &L) {
  return L.kind == MPN_LAYER_CONV && L.kh == L.kw && (L.kh == 1 || L.kh == 3) && (L.stride == 1 || L.stride == 2) &&
         L.pad == (L.kh - 1) / 2 && L.weight >= 0 && L.cout > 0 && L.cout % 64 == 0;
}
static const char *const FIXED_CONV_MSG = "training: a fixed-batch-norm layer must be a 1x1 or 3x3 convolution with stride 1 or 2, pad "
                                          "(k - 1) / 2 and a multiple of 64 output channels";
// a layer whose Cin leaves a tail in its last K block (conv_k_pad) runs forward only: no backward GEMM takes the padded
// weight layout. Refused when training begins, for every trained weight (the host-only graph checks do not look at widths)
static const char *const TAIL_MSG = "training: a trained layer must read a multiple of 64 input channels (a Linear after a FLATTEN: "
                                    "channels x pooled area); a layer with a K tail, such as NIN's 96-channel block 1, runs forward only";
static bool recorded(const std::set<int> *rec, const mpn_layer &L) {
  return rec && L.kind == MPN_LAYER_CONV && L.weight >= 0 && rec->count(L.weight);
}
// a tower trained by the graph backward: it holds a recorded layer (fixed batch norm); such a tower ends in an AVGPOOL
static bool graph_tower(const mpn_model_desc *d, const mpn_tower &T, const std::set<int> *rec) {
  for (int i = 0; i < T.n_layers; ++i) if (recorded(rec, d->tower_layers[T.first_layer + i])) return true;
  return false;
}

// host-only: the graph restrictions of a training step. msg: a static description of the first violation. integral: K > 1
// class heads train with the integral loss (mpn_train_spec.integral); without it they are refused, as ever.
// rec: the recorded (fixed-batch-norm) convolutions' weights, null for a training without records.
static int train_check_graph(const mpn_model_desc *d, bool integral, const char **msg, const std::set<int> *rec) {
  *msg = nullptr;
  if (d->n_cls_heads < 1) { *msg = "training: the graph has no class head"; return MPN_ERR_ARG; }
  if (d->n_cls_heads != 1 && !integral) {
    *msg = "training: an integral head (K > 1 class heads) trains only with the integral loss (mpn_train_spec.integral = 1, "
           "Trainer(integral=True))";
    return MPN_ERR_ARG;
  }
  std::set<int> seen;
  auto own = [&](int w) { if (w < 0) return true; return seen.insert(w).second; };
  for (int t = 0; t < d->n_towers; ++t) {
    const mpn_tower &T = d->towers[t];
    const bool graph = graph_tower(d, T, rec);
    for (int i = 0; i < T.n_layers; ++i) {
      const mpn_layer &L = d->tower_layers[T.first_layer + i];
      if (graph && recorded(rec, L)) {
        if (!fixed_conv_ok(L)) { *msg = FIXED_CONV_MSG; return MPN_ERR_ARG; }
        if (!own(L.weight) || !own(L.bias)) { *msg = "training: a parameter tensor is shared between layers"; return MPN_ERR_ARG; }
        continue;
      }
      if (graph && (L.kind == MPN_LAYER_AVGPOOL || L.kind == MPN_LAYER_FLATTEN || i == T.n_layers - 1)) {
        if (L.kind != MPN_LAYER_AVGPOOL || i != T.n_layers - 1 || L.out_slot != T.out_slot) {
          *msg = "training: a tower with fixed-batch-norm layers has no FLATTEN and ends in a global AVGPOOL that the heads read";
          return MPN_ERR_ARG;
        }
        continue;
      }
      if (L.kind == MPN_LAYER_FLATTEN) continue;
      if (L.kind != MPN_LAYER_CONV || L.kh != 1 || L.kw != 1 || L.stride != 1 || L.pad != 0 || L.residual_slot >= 0) {
        *msg = "training: every per-ROI layer must be a 1x1 convolution, FLATTEN or Linear (a ResNet layer4 does not train here)";
        return MPN_ERR_ARG;
      }
      if (!own(L.weight) || !own(L.bias)) { *msg = "training: a parameter tensor is shared between layers"; return MPN_ERR_ARG; }
    }
  }
  // an integral model's K class heads (model_utils.integral's clones) read one column range and have one width
  const mpn_head &c = d->cls_heads[0], &b = d->bbox_head;
  for (int k = 0; k < d->n_cls_heads; ++k) {
    const mpn_head &h = d->cls_heads[k];
    if (h.col_begin != c.col_begin || h.col_len != c.col_len || h.cout != c.cout) {
      *msg = "training: the class heads of an integral model must read the same columns and have the same width";
      return MPN_ERR_ARG;
    }
    if (!own(h.weight) || !own(h.bias)) { *msg = "training: a parameter tensor is shared between layers"; return MPN_ERR_ARG; }
  }
  if (!own(b.weight) || !own(b.bias)) { *msg = "training: a parameter tensor is shared between layers"; return MPN_ERR_ARG; }
  const bool same = c.col_begin == b.col_begin && c.col_len == b.col_len;
  const bool disjoint = c.col_begin + c.col_len <= b.col_begin || b.col_begin + b.col_len <= c.col_begin;
  if (!same && !disjoint) { *msg = "training: the class and bbox heads read partly overlapping columns"; return MPN_ERR_ARG; }
  return MPN_OK;
}

// host-only: the restrictions of training the trunk from layer k (0: frozen, nothing to check). rec: as train_check_graph;
// a range with recorded layers may be a graph (residuals, several readers per slot), else it must be a chain as ever.
static int train_check_trunk_range(const mpn_model_desc *d, int k, const char **msg, const std::set<int> *rec);
static int train_check_trunk(const mpn_model_desc *d, int k, const char **msg, const std::set<int> *rec) {
  *msg = nullptr;
  if (k == 0) return MPN_OK;
  if (train_check_trunk_range(d, k, msg, rec) != MPN_OK) return MPN_ERR_ARG;
  const int n = d->n_trunk_layers;
  const int top = d->trunk_layers[n - 1].out_slot;
  if (d->n_towers != 1) {
    *msg = "training the trunk: the graph must have exactly one tower (MultiPathNet's towers do not train the trunk here)";
    return MPN_ERR_ARG;
  }
  for (int t = 0; t < d->n_towers; ++t) {
    const mpn_tower &T = d->towers[t];
    if (T.n_levels != 1 || T.level_slot[0] != top || T.normalize || T.region != 0) {
      *msg = "training the trunk: every tower must pool its ROIs from the last trunk layer's output alone, without foveal regions or "
             "normalisation (MultiPathNet and ResNet trunks do not train here)";
      return MPN_ERR_ARG;
    }
    if (graph_tower(d, T, rec)) continue;        // the graph backward hands the pooled map its gradient
    const mpn_layer *L0 = T.n_layers >= 2 ? &d->tower_layers[T.first_layer] : nullptr;
    if (!L0 || L0->kind != MPN_LAYER_FLATTEN || L0->in_slot != 0 || L0[1].kind != MPN_LAYER_CONV || L0[1].in_slot != L0->out_slot) {
      *msg = "training the trunk: a tower must start with a FLATTEN of the pooled map and a Linear";
      return MPN_ERR_ARG;
    }
  }
  return MPN_OK;
}

// host-only: MultiPathNet's phase 2 (mpn_train_spec.phase2, utils.vggSetPhase2_outer): the trunk range from k
// trains under train_check_trunk's range rules; every tower level pools a slot that a trained layer writes (at most
// MAX_ROI_BWD_JOBS levels per slot), and a tower's first layer reads the pooled map and is a convolution (conv_mix) or a
// FLATTEN in front of a Linear, whose dX is the pooled map's gradient
static int train_check_phase2(const mpn_model_desc *d, int k, const char **msg) {
  *msg = nullptr;
  if (k == 0) { *msg = "phase 2: phase2_from is 0 (the model has no trunk range that trains in phase 2)"; return MPN_ERR_ARG; }
  if (train_check_trunk_range(d, k, msg, nullptr) != MPN_OK) return MPN_ERR_ARG;
  std::set<int> trained;
  for (int i = k; i < d->n_trunk_layers; ++i) trained.insert(d->trunk_layers[i].out_slot);
  std::map<int, int> jobs;
  for (int t = 0; t < d->n_towers; ++t) {
    const mpn_tower &T = d->towers[t];
    for (int l = 0; l < T.n_levels; ++l) {
      if (!trained.count(T.level_slot[l])) {
        *msg = "phase 2: every tower level must pool a trunk slot that a trained layer (phase2_from and up) writes";
        return MPN_ERR_ARG;
      }
      if (++jobs[T.level_slot[l]] > MAX_ROI_BWD_JOBS) { *msg = "phase 2: more than 8 tower levels pool one trunk slot"; return MPN_ERR_ARG; }
    }
    const mpn_layer *L0 = T.n_layers >= 1 ? &d->tower_layers[T.first_layer] : nullptr;
    bool ok = T.n_levels >= 1 && L0 && L0->in_slot == 0 &&
              (L0->kind == MPN_LAYER_CONV ||
               (L0->kind == MPN_LAYER_FLATTEN && T.n_layers >= 2 && L0[1].kind == MPN_LAYER_CONV && L0[1].in_slot == L0->out_slot));
    for (int i = 1; ok && i < T.n_layers; ++i) ok = d->tower_layers[T.first_layer + i].in_slot != 0;
    if (!ok) {
      *msg = "phase 2: a tower must start with a convolution of the pooled map (conv_mix) or a FLATTEN of it and a Linear, and no "
             "other layer may read the pooled map";
      return MPN_ERR_ARG;
    }
  }
  return MPN_OK;
}

// the layer rules of a trained trunk range (train_check_trunk without its tower rules)
static int train_check_trunk_range(const mpn_model_desc *d, int k, const char **msg, const std::set<int> *rec) {
  const int n = d->n_trunk_layers;
  if (k < 1 || k >= n) { *msg = "training the trunk: trunk_from out of range (layer 0 never trains; 1 <= trunk_from < number of trunk layers)"; return MPN_ERR_ARG; }
  bool graph = false;
  for (int i = k; i < n; ++i) graph |= recorded(rec, d->trunk_layers[i]);
  std::set<int> written;
  for (int i = k; i < n; ++i) {
    const mpn_layer &L = d->trunk_layers[i];
    if (recorded(rec, L) && !(fixed_conv_ok(L) && L.in_slot != 0)) { *msg = FIXED_CONV_MSG; return MPN_ERR_ARG; }
    const bool conv = recorded(rec, L) ||
                      (L.kind == MPN_LAYER_CONV && L.kh == 3 && L.kw == 3 && L.stride == 1 && L.pad == 1 && L.relu && L.residual_slot < 0 &&
                       L.in_slot != 0 && L.weight >= 0);
    const bool pool = L.kind == MPN_LAYER_MAXPOOL && L.kh == 2 && L.kw == 2 && L.stride == 2 && L.pad == 0;
    if (!conv && !pool) {
      *msg = "training the trunk: a trained trunk layer must be a 3x3 / stride 1 / pad 1 convolution with ReLU and no residual, or a 2x2 / "
             "stride 2 / pad 0 max pool (ResNet trunks do not train here)";
      return MPN_ERR_ARG;
    }
    if (graph) {
      for (int s : {L.in_slot, L.residual_slot})
        if (s >= 0 && s != d->trunk_layers[k].in_slot && !written.count(s)) {
          *msg = "training the trunk: a trained layer reads a slot that neither a trained layer below it nor the frozen part's output is";
          return MPN_ERR_ARG;
        }
    }
    if (i > k && ((!graph && L.in_slot != d->trunk_layers[i - 1].out_slot) ||
                  (pool && (L.in_slot != d->trunk_layers[i - 1].out_slot || d->trunk_layers[i - 1].kind != MPN_LAYER_CONV)))) {
      *msg = "training the trunk: the trained layers must form a chain, each reading the previous one's output, a max pool after a convolution";
      return MPN_ERR_ARG;
    }
    if (L.out_slot == d->trunk_layers[k].in_slot || !written.insert(L.out_slot).second) {
      *msg = "training the trunk: a trained layer overwrites a slot the backward reads";
      return MPN_ERR_ARG;
    }
  }
  return MPN_OK;
}

// the fixed-batch-norm records as a set of weight indices: each names a convolution of the graph, once
static int fixed_records(const mpn_model_desc *d, int32_t n, const int32_t *weight, std::set<int> &rec, const char **msg) {
  *msg = nullptr;
  if (n < 0 || (n > 0 && !weight)) { *msg = "fixed batch norm: n < 0 or the weight list is missing"; return MPN_ERR_ARG; }
  std::set<int> convs;
  for (int i = 0; i < d->n_trunk_layers; ++i) if (d->trunk_layers[i].kind == MPN_LAYER_CONV) convs.insert(d->trunk_layers[i].weight);
  for (int i = 0; i < d->n_tower_layers; ++i) if (d->tower_layers[i].kind == MPN_LAYER_CONV) convs.insert(d->tower_layers[i].weight);
  for (int j = 0; j < n; ++j) {
    if (weight[j] < 0 || !convs.count(weight[j]) || !rec.insert(weight[j]).second) {
      *msg = "fixed batch norm: a record names no convolution's weight, or names one twice";
      return MPN_ERR_ARG;
    }
  }
  return MPN_OK;
}

// host-only: every rule of a training under spec s, in the order the header gives; the first refusal goes to msg.
// rec: the records of s (fixed_records)
static int train_check(const mpn_model_desc *d, const mpn_train_spec *s, std::set<int> &rec, const char **msg) {
  if (s->phase2 && s->n_fixed > 0) { *msg = "phase 2: a model with fixed batch norm (spec.fixed_bn) has no phase 2"; return MPN_ERR_ARG; }
  if (fixed_records(d, s->n_fixed, s->fixed_weight, rec, msg) != MPN_OK) return MPN_ERR_ARG;
  const std::set<int> *r = s->n_fixed > 0 ? &rec : nullptr;
  const int rc = s->phase2 ? train_check_phase2(d, s->trunk_from, msg) : train_check_trunk(d, s->trunk_from, msg, r);
  if (rc != MPN_OK) return rc;
  return train_check_graph(d, s->integral != 0, msg, r);
}

static mpn_model_desc model_view(const mpn_model *m) {
  mpn_model_desc d = m->d;
  d.trunk_layers = m->trunk_layers.data(); d.tower_layers = m->tower_layers.data(); d.towers = m->towers.data();
  d.cls_heads = m->cls_heads.data();
  d.n_trunk_layers = (int32_t)m->trunk_layers.size(); d.n_tower_layers = (int32_t)m->tower_layers.size();
  d.n_towers = (int32_t)m->towers.size(); d.n_cls_heads = (int32_t)m->cls_heads.size();
  return d;
}

// the ROI jobs' trunk geometry after the trunk was planned for another image size (the tower plans do not depend on it)
static void refresh_roi_jobs(mpn_model *m) {
  for (int ji = 0; ji < m->jobs.n; ++ji) {
    RoiJob &j = m->jobs.j[ji];
    const mpn_tower &T = m->towers[j.tower];
    int l = 0;
    for (int k = 0; k < ji; ++k) if (m->jobs.j[k].tower == j.tower) ++l;
    const int slot = T.level_slot[l];
    const DTensor &f = m->trunk_slots[slot];
    j.H = (int)f.H; j.W = (int)f.W;
    const mpn_model::Pyramid &P = m->pyramids[slot];
    j.nlev = P.nlev;
    for (int k = 0; k < ROI_MAX_LEVELS; ++k) j.lv[k] = (const float *)P.lv[std::min(k, P.nlev - 1)]->p;
  }
}

static int train_opts_ok(mpn_model *m) {
  MPN_CHECK_ARG(m->ctx, m->ctx->opt_bf16 != 1 && m->ctx->opt_fp8 != 1,
                "training runs the fp32-faithful BF16X3 numerics: switch the \"bf16\" / \"fp8\" options off");
  return MPN_OK;
}

// dW = G^T X (Torch layout [cout][Kin]) and, when dx is set, dX = G W ([rows][Kin] in the layer's input order); G is
// [rows][cout] fp32 (row stride ldg) and already gated. x: the layer's input (split planes, rows x Kin, row stride x.ld);
// flat_c / flat_hw: the FLATTEN in front of a Linear ((h, w, c) input order against the weight's (c, h, w)), 0 otherwise.
// zero columns [c0, c1) of both planes of a row-major [rows][ld] split buffer (the K padding of a GEMM operand); of the
// hi plane only when the buffer has no lo plane (a bf16 training step)
static int zero_cols(mpn_ctx *ctx, SplitBuf &b, int64_t rows, int64_t ld, int64_t c0, int64_t c1) {
  if (c1 <= c0 || rows <= 0) return MPN_OK;
  for (void *p : {b.hi.p, b.lo.p})
    if (p) MPN_CUDA(ctx, cudaMemset2DAsync((char *)p + 2 * c0, (size_t)(2 * ld), 0, (size_t)(2 * (c1 - c0)), (size_t)rows, ctx->stream));
  return MPN_OK;
}

static int train_layer_backward(mpn_model *m, const TrainParam &P, const float *G, int64_t ldg, int64_t rows, const DTensor &x,
                                int flat_c, int flat_hw, float *dx) {
  mpn_ctx *ctx = m->ctx;
  TrainState &T = *m->train;
  const int64_t cout = P.cout, Kin = (int64_t)P.cin * P.kh * P.kw, rp = (rows + 63) / 64 * 64;
  const int perm = flat_hw > 1 ? 2 : 0;
  MPN_TRY(T.opGT.ensure(ctx, (size_t)(cout * rp), !T.bf16));
  MPN_TRY(T.opXT.ensure(ctx, (size_t)(Kin * rp), !T.bf16));
  MPN_TRY(zero_cols(ctx, T.opGT, cout, rp, rows, rp));           // the transposes write every column below `rows`
  MPN_TRY(zero_cols(ctx, T.opXT, Kin, rp, rows, rp));
  auto *gth = (__nv_bfloat16 *)T.opGT.hi.p, *gtl = (__nv_bfloat16 *)T.opGT.lo.p;
  auto *xth = (__nv_bfloat16 *)T.opXT.hi.p, *xtl = (__nv_bfloat16 *)T.opXT.lo.p;
  MPN_TRY(mpn_train_transpose_launch(ctx, G, nullptr, nullptr, ldg, rows, cout, 0, 0, 0, gth, gtl, rp, 0));
  MPN_TRY(mpn_train_transpose_launch(ctx, nullptr, x.hi, x.lo, x.ld, rows, Kin, perm, flat_c, flat_hw, xth, xtl, rp, 0));
  MPN_TRY(mpn_train_gemm(ctx, gth, gtl, cout, rp, rp, xth, xtl, Kin, (float *)P.grad.p, Kin, 0, T.bf16));
  if (!dx) return MPN_OK;
  const int64_t kp = (cout + 63) / 64 * 64;
  MPN_CHECK_ARG(ctx, P.wt_hi && P.wt_ld == kp && P.wt_col0 == 0, "training: a layer with dX has no transposed weight planes");
  MPN_TRY(T.opA.ensure(ctx, (size_t)(rows * kp), !T.bf16));
  MPN_TRY(zero_cols(ctx, T.opA, rows, kp, cout, kp));
  auto *ah = (__nv_bfloat16 *)T.opA.hi.p, *al = (__nv_bfloat16 *)T.opA.lo.p;
  MPN_TRY(mpn_train_gate_split_launch(ctx, const_cast<float *>(G), ldg, rows, cout, nullptr, 1.f, ah, al, kp, 0));
  return mpn_train_gemm(ctx, ah, al, rows, kp, kp, P.wt_hi, P.wt_lo, Kin, dx, Kin, 0, T.bf16);
}

static int tower_graph_backward(mpn_model *m, size_t t);

static int train_backward(mpn_model *m, int64_t R) {
  mpn_ctx *ctx = m->ctx;
  TrainState &T = *m->train;
  const int width = m->concat_width;
  const float p = T.cfg.dropout;
  MPN_TRY(T.dconcat.ensure(ctx, sizeof(float) * (size_t)(R * width)));
  MPN_CUDA(ctx, cudaMemsetAsync(T.dconcat.p, 0, sizeof(float) * (size_t)(R * width), ctx->stream));
  // heads: the selected class head k and the bbox head: dW, db; dX into the concat's columns (one GEMM per head, or one
  // over all heads when they read the same columns). The idle class heads take no gradient (nn.SelectTable).
  const int K = (int)m->cls_heads.size(), k = T.head;
  const mpn_head *hs[2] = {&m->cls_heads[k], &m->d.bbox_head};
  float *gh[2] = {(float *)T.dlogits.p, (float *)T.dbbox.p};
  DTensor concat; concat.hi = (__nv_bfloat16 *)m->concat_buf.hi.p; concat.lo = (__nv_bfloat16 *)m->concat_buf.lo.p;
  concat.N = R; concat.H = concat.W = 1; concat.C = width; concat.ld = width;
  for (int h = 0; h < 2; ++h) {
    DTensor x = concat; x.hi += hs[h]->col_begin; x.lo += hs[h]->col_begin; x.C = hs[h]->col_len;
    MPN_TRY(train_layer_backward(m, T.params[T.param_of[hs[h]->weight]], gh[h], hs[h]->cout, R, x, 0, 0, nullptr));
    if (hs[h]->bias >= 0) MPN_TRY(mpn_train_colsum_launch(ctx, gh[h], hs[h]->cout, R, hs[h]->cout, (float *)T.params[T.param_of[hs[h]->bias]].grad.p));
  }
  const bool same = hs[0]->col_begin == hs[1]->col_begin && hs[0]->col_len == hs[1]->col_len;
  for (int g = 0; g < (same ? 1 : 2); ++g) {
    // same columns: ONE GEMM over the W^T planes [cls_0 .. cls_{K-1} ; bbox] (K0 columns per class head), the idle
    // heads' columns of A zero: their terms are exact zeros
    const int64_t K0 = (hs[0]->cout + 63) / 64 * 64, K1 = (hs[1]->cout + 63) / 64 * 64;
    const int64_t kg = same ? K * K0 + K1 : (g == 0 ? K0 : K1), len = hs[g]->col_len;
    const TrainParam &PW = T.params[T.param_of[same ? m->cls_heads[0].weight : hs[g]->weight]];   // the group's planes start here
    MPN_CHECK_ARG(ctx, PW.wt_hi && PW.wt_ld == kg && PW.wt_col0 == 0, "training: the heads have no transposed weight planes");
    MPN_TRY(T.opA.ensure(ctx, (size_t)(R * kg), !T.bf16));
    auto *ah = (__nv_bfloat16 *)T.opA.hi.p, *al = (__nv_bfloat16 *)T.opA.lo.p;
    for (int j = 0; same && j < K; ++j)
      if (j != k) MPN_TRY(zero_cols(ctx, T.opA, R, kg, j * K0, (j + 1) * K0));
    for (int h = 0; h < 2; ++h) {
      if (!same && h != g) continue;
      const int64_t off = same ? (h == 0 ? k * K0 : K * K0) : 0;
      MPN_TRY(zero_cols(ctx, T.opA, R, kg, off + hs[h]->cout, off + (h == 0 ? K0 : K1)));
      MPN_TRY(mpn_train_gate_split_launch(ctx, gh[h], hs[h]->cout, R, hs[h]->cout, nullptr, 1.f, ah, al, kg, off));
    }
    MPN_TRY(mpn_train_gemm(ctx, ah, al, R, kg, kg, PW.wt_hi, PW.wt_lo, len, (float *)T.dconcat.p + hs[g]->col_begin, width, 0, T.bf16));
  }
  // towers, top down: gate through ReLU (+ dropout), db, dW, and dX while a trained layer lies below
  for (size_t t = 0; t < m->towers.size(); ++t) {
    if (T.graph_tower[t]) { MPN_TRY(tower_graph_backward(m, t)); continue; }
    mpn_model::TowerExec &X = m->tex[t];
    std::vector<int> convs;
    for (size_t li = 0; li < X.layers.size(); ++li) if (X.layers[li].L.kind == MPN_LAYER_CONV) convs.push_back((int)li);
    float *G = (float *)T.dconcat.p + X.col_off;
    int64_t ldg = width;
    for (int j = (int)convs.size() - 1; j >= 0; --j) {
      const LayerExec &e = X.layers[convs[j]];
      const mpn_layer &L = e.L;
      const int64_t rows = R * e.out.H * e.out.W;
      const bool drop = p > 0.f && L.relu && e.out.H == 1 && e.out.W == 1;
      if (L.relu) MPN_TRY(mpn_train_gate_split_launch(ctx, G, ldg, rows, L.cout, &e.out, drop ? 1.f / (1.f - p) : 1.f, nullptr, nullptr, 0, 0));
      if (L.bias >= 0) MPN_TRY(mpn_train_colsum_launch(ctx, G, ldg, rows, L.cout, (float *)T.params[T.param_of[L.bias]].grad.p));
      int fc = 0, fhw = 0;
      DTensor x = e.in;
      for (const LayerExec &f : X.layers)
        if (f.L.kind == MPN_LAYER_FLATTEN && f.L.out_slot == L.in_slot) { fc = (int)f.in.C; fhw = (int)(f.in.H * f.in.W); }
      const TrainParam &P = T.params[T.param_of[L.weight]];
      const int64_t Kin = (int64_t)P.cin * P.kh * P.kw;
      float *dx = nullptr;
      if (j > 0) { MPN_TRY(T.dx[j & 1].ensure(ctx, sizeof(float) * (size_t)(rows * Kin))); dx = (float *)T.dx[j & 1].p; }
      else if (T.trunk_from > 0) {              // the pooled rows' gradient, (h, w, c) order: the trunk backward's input
        MPN_TRY(T.dpooled[t]->ensure(ctx, sizeof(float) * (size_t)(rows * Kin)));
        dx = (float *)T.dpooled[t]->p;
      }
      MPN_TRY(train_layer_backward(m, P, G, ldg, e.in.N * e.in.H * e.in.W, x, fc, fhw, dx));
      G = dx; ldg = (dx && j > 0) ? X.layers[convs[j - 1]].L.cout : 0;
    }
  }
  return MPN_OK;
}

// wgrad of one k x k / stride s / pad q convolution: dW [cout][cin * k * k] (Torch layout) = G^T B^T over the maps'
// output pixels stacked in order, G [pixels][cout] fp32 (gated), xs the maps' inputs (split planes, cin channels, N maps
// each) and ys their outputs (geometry only); ONE GEMM, K = the pixels padded to 64 (only the padding is zeroed), A = G^T,
// B [cin * k * k][pixels] the tap-shifted inputs in Torch (ci, ky, kx) order. bf16: BF16X1, both operands hi planes only
static int conv_wgrad(mpn_ctx *ctx, SplitBuf &opGT, SplitBuf &opTap, const float *G, int64_t cout, const std::vector<DTensor> &xs,
                      const std::vector<DTensor> &ys, int k, int s, int q, float *dw, bool bf16) {
  int64_t P = 0;
  for (const DTensor &y : ys) P += y.N * y.H * y.W;
  const int64_t cin = xs.at(0).C, kk = (int64_t)k * k, kp = (P + 63) / 64 * 64;
  MPN_TRY(opGT.ensure(ctx, (size_t)(cout * kp), !bf16));
  MPN_TRY(opTap.ensure(ctx, (size_t)(cin * kk * kp), !bf16));
  MPN_TRY(zero_cols(ctx, opGT, cout, kp, P, kp));
  MPN_TRY(zero_cols(ctx, opTap, cin * kk, kp, P, kp));
  auto *gth = (__nv_bfloat16 *)opGT.hi.p, *gtl = (__nv_bfloat16 *)opGT.lo.p;
  auto *tph = (__nv_bfloat16 *)opTap.hi.p, *tpl = (__nv_bfloat16 *)opTap.lo.p;
  MPN_TRY(mpn_train_transpose_launch(ctx, G, nullptr, nullptr, cout, P, cout, 0, 0, 0, gth, gtl, kp, 0));
  int64_t off = 0;
  for (size_t i = 0; i < xs.size(); ++i) {
    const DTensor &x = xs[i], &y = ys.at(i);
    MPN_CHECK_ARG(ctx, x.C == cin && x.N == y.N, "wgrad: the images' inputs differ in channels");
    MPN_TRY(mpn_train_tap_transpose_launch(ctx, x, k, s, q, y.H, y.W, tph, tpl, kp, off));
    off += y.N * y.H * y.W;
  }
  return mpn_train_gemm(ctx, gth, gtl, cout, kp, kp, tph, tpl, cin * kk, dw, cin * kk, 1, bf16);
}

// image i's copy of every trunk slot the trunk backward reads, taken after its forward (the trunk reuses one buffer per
// slot for every image); the frozen layers below run exactly as at inference
static int keep_trunk_slots(mpn_model *m, int i) {
  mpn_ctx *ctx = m->ctx;
  TrainState &T = *m->train;
  if ((int)T.img_bufs.size() <= i) { T.img_bufs.resize(i + 1); T.img_slots.resize(i + 1); }
  std::set<int> slots{m->trunk_layers[T.trunk_from].in_slot};
  for (size_t li = T.trunk_from; li < m->trunk_layers.size(); ++li) slots.insert(m->trunk_layers[li].out_slot);
  for (int s : slots) {
    MPN_CHECK_ARG(ctx, !m->elided_slots.count(s), "training the trunk: a slot the backward reads was not written");
    const DTensor &src = m->trunk_slots.at(s);
    MPN_CHECK_ARG(ctx, src.ld == src.C && src.N == 1, "training the trunk: trunk slots must be dense single-image maps");
    const size_t elems = (size_t)(src.H * src.W * src.C);
    auto &b = T.img_bufs[i][s];
    if (!b) b.reset(new SplitBuf());
    MPN_TRY(b->ensure(ctx, elems));
    MPN_CUDA(ctx, cudaMemcpyAsync(b->hi.p, src.hi, 2 * elems, cudaMemcpyDeviceToDevice, ctx->stream));
    MPN_CUDA(ctx, cudaMemcpyAsync(b->lo.p, src.lo, 2 * elems, cudaMemcpyDeviceToDevice, ctx->stream));
    T.img_slots[i][s] = make_split_view(*b, 1, src.H, src.W, src.C);
  }
  return MPN_OK;
}

// One slot of the graph backward (below): its stored maps (the trunk: one per image; a tower: one of N = R ROIs), stacked
// in order, and its gradient: an outside buffer set beforehand (a tower's pooled map) or, from its first contribution to
// the end of its producer's backward, one of T.grad_bufs (buf).
struct GraphSlot { std::vector<DTensor> maps; float *g = nullptr; DevBuf *buf = nullptr; bool written = false; };
static int contribute(mpn_ctx *ctx, TrainState &T, GraphSlot &X, bool stores, bool *store);

// the towers' ROI pooling backward, the first contribution (a store) to every trunk slot a tower level pools, images
// stacked in order: per image, each (tower, level) job's argmax on the image's kept map (its region and scale) and a
// normalised job's (a, b), then per slot ONE gather over the jobs that pool it, in tower order, from the towers' pooled
// rows' gradients (T.dpooled[t], (h, w, c) rows with the levels at their channel offsets)
static int trunk_roi_backward(mpn_model *m, int n_images, const int32_t *rois_per_image, std::map<int, GraphSlot> &S) {
  mpn_ctx *ctx = m->ctx;
  TrainState &T = *m->train;
  const mpn_tower &T0 = m->towers[0];
  const int PW = T0.pooled_w, PH = T0.pooled_h, bins = PW * PH;
  int64_t rmax = 0;
  for (int i = 0; i < n_images; ++i) rmax = std::max<int64_t>(rmax, rois_per_image[i]);
  struct Job { int slot, t, l, ch_off; };
  std::vector<Job> jobs;
  std::vector<int> slots;
  int64_t n_am = 0, n_ab = 0;
  for (size_t t = 0; t < m->towers.size(); ++t) {
    const mpn_tower &Tw = m->towers[t];
    int off = 0;
    for (int l = 0; l < Tw.n_levels; ++l) {
      const int s = Tw.level_slot[l];
      const int64_t C = T.img_slots[0].at(s).C;
      jobs.push_back({s, (int)t, l, off});
      if (std::find(slots.begin(), slots.end(), s) == slots.end()) slots.push_back(s);
      off += (int)C;
      n_am += rmax * bins * C;
      if (Tw.normalize) n_ab += 2 * rmax;
    }
  }
  MPN_TRY(T.roi_argmax.ensure(ctx, sizeof(int32_t) * (size_t)std::max<int64_t>(n_am, 1)));
  if (n_ab > 0) MPN_TRY(T.roi_ab.ensure(ctx, sizeof(double) * (size_t)n_ab));
  for (int s : slots) {
    bool store;
    MPN_TRY(contribute(ctx, T, S.at(s), true, &store));
    MPN_CHECK_ARG(ctx, store, "training the trunk: the ROI backward must be a pooled slot's first contribution");
  }
  std::map<int, int64_t> off_p;
  int64_t off_r = 0;
  for (int i = 0; i < n_images; ++i) {
    const int64_t Ri = rois_per_image[i];
    const float *rois = (const float *)T.rois5.p + off_r * 5;
    std::vector<RoiBwdJob> bj(jobs.size());
    int32_t *am = (int32_t *)T.roi_argmax.p;
    double *ab = (double *)T.roi_ab.p;
    for (size_t k = 0; k < jobs.size(); ++k) {
      const Job &j = jobs[k];
      const mpn_tower &Tw = m->towers[j.t];
      const DTensor &f = T.img_slots[i].at(j.slot);
      const int64_t ctot = m->tex[j.t].ctot;
      RoiBwdJob &b = bj[k];
      b.region = Tw.region; b.scale = Tw.level_scale[j.l];
      b.grad = (const float *)T.dpooled[j.t]->p + off_r * bins * ctot; b.ld = ctot; b.ch_off = j.ch_off;
      b.argmax = am; b.ab = nullptr;
      MPN_TRY(mpn_roi_argmax_nhwc_launch(ctx, f, rois, Ri, PW, PH, b.region, b.scale, m->d.roi_variant, am));
      am += Ri * bins * f.C;
      if (Tw.normalize) { MPN_TRY(mpn_roi_norm_ab_launch(ctx, f, Ri, PW, PH, b, ab)); b.ab = ab; ab += 2 * Ri; }
    }
    for (int s : slots) {
      RoiBwdJobs J{};
      for (size_t k = 0; k < jobs.size(); ++k) if (jobs[k].slot == s) J.j[J.n++] = bj[k];
      const DTensor &f = T.img_slots[i].at(s);
      MPN_TRY(mpn_roi_backward_jobs_launch(ctx, f, rois, Ri, PW, PH, m->d.roi_variant, J, S.at(s).g + off_p[s] * f.C));
      off_p[s] += f.H * f.W;
    }
    off_r += Ri;
  }
  return MPN_OK;
}

// ---- the graph backward: every trained trunk range, and a tower with a record (ResNet blocks). Layers walk in reverse
// order; each reader of a slot contributes to its fp32 gradient in that order (residual first, then dgrad): a fixed
// order, no atomics. The first contribution stores when its kernel writes every element (the ROI backward,
// pool_gate_split, a stride 1 dgrad) and a residual's is a copy; else (col2im, the AVGPOOL's broadcast) the slot is zeroed
// first. Later contributions add. A slot's gradient: GraphSlot, above.

static int64_t map_pixels(const std::vector<DTensor> &v) { int64_t n = 0; for (const DTensor &x : v) n += x.N * x.H * x.W; return n; }

// a contribution to slot X whose kernel writes every element when `stores`: at the first one, X's buffer (the smallest
// free one that fits, else the largest grown, else a new one), zeroed unless the contribution stores; *store: it stores
static int contribute(mpn_ctx *ctx, TrainState &T, GraphSlot &X, bool stores, bool *store) {
  *store = stores && !X.written;
  if (X.written) return MPN_OK;
  X.written = true;
  const size_t bytes = sizeof(float) * (size_t)(map_pixels(X.maps) * X.maps.at(0).C);
  if (!X.g) {
    auto it = T.grad_free.lower_bound(bytes);
    if (it == T.grad_free.end() && !T.grad_free.empty()) --it;
    if (it == T.grad_free.end()) { T.grad_bufs.emplace_back(new DevBuf()); X.buf = T.grad_bufs.back().get(); }
    else { X.buf = it->second; T.grad_free.erase(it); }
    MPN_TRY(X.buf->ensure(ctx, std::max<size_t>(bytes, sizeof(float))));
    X.g = (float *)X.buf->p;
  }
  if (!stores) MPN_CUDA(ctx, cudaMemsetAsync(X.g, 0, bytes, ctx->stream));
  return MPN_OK;
}

// dgrad of a k x k / stride s / pad q convolution into dx (the input maps' gradient, [pixels][cin] fp32, maps stacked in
// order): gs the split planes of the gated output gradient [out pixels][cout]; wt the rotated planes [cin][ky][kx][cout]
// (3x3 / stride 1: per map a 3x3 / pad 1 convolution on the engine, BF16X3, no bias, no ReLU, over N images of H x W:
// the trunk's images one by one, a tower's R ROIs at once) or W'^T [(ky, kx, ci)][cout] (1x1 / stride 1: one GEMM;
// stride 2: one GEMM to the column gradient, then the gather col2im, which adds). Stride 1 stores the product into dx
// when `store`, else adds it from tmp, a workspace. bf16: every product in BF16X1 (gs_lo / wt_lo null)
static int conv_dgrad(mpn_ctx *ctx, DevBuf &tmp, const __nv_bfloat16 *gs_hi, const __nv_bfloat16 *gs_lo, int64_t cout, int64_t cin,
                      int k, int s, int q, const __nv_bfloat16 *wt_hi, const __nv_bfloat16 *wt_lo, const std::vector<DTensor> &xs,
                      const std::vector<DTensor> &ys, float *dx, bool store, bool bf16) {
  const int64_t Po = map_pixels(ys), Pi = map_pixels(xs), kk = (int64_t)k * k;
  if (s == 1) {
    float *out = dx;
    if (!store) { MPN_TRY(tmp.ensure(ctx, sizeof(float) * (size_t)(Pi * cin))); out = (float *)tmp.p; }
    if (k == 1) {
      MPN_TRY(mpn_train_gemm(ctx, gs_hi, gs_lo, Po, cout, cout, wt_hi, wt_lo, cin, out, cin, 0, bf16));
    } else {
      int64_t off = 0;
      for (const DTensor &y : ys) {
        ConvProblem p;
        p.x.hi = const_cast<__nv_bfloat16 *>(gs_hi) + off * cout; p.x.lo = gs_lo ? const_cast<__nv_bfloat16 *>(gs_lo) + off * cout : nullptr;
        p.x.N = y.N; p.x.H = y.H; p.x.W = y.W; p.x.C = cout; p.x.ld = cout;
        p.w_hi = wt_hi; p.w_lo = wt_lo; p.Cout = (int)cin; p.kh = p.kw = 3; p.stride = 1; p.pad = 1; p.bf16 = bf16 ? 1 : 0;
        p.y.f32 = out + off * cin; p.y.N = y.N; p.y.H = y.H; p.y.W = y.W; p.y.C = cin; p.y.ld = cin; p.y_f32_ld = cin;
        ConvPlan pl;
        MPN_TRY(conv_tc_plan(ctx, p, pl));
        MPN_TRY(conv_tc_launch(ctx, p, pl));
        off += y.N * y.H * y.W;
      }
    }
    return store ? MPN_OK : mpn_train_add_launch(ctx, dx, out, Pi * cin);
  }
  MPN_TRY(tmp.ensure(ctx, sizeof(float) * (size_t)(Po * kk * cin)));
  MPN_TRY(mpn_train_gemm(ctx, gs_hi, gs_lo, Po, cout, cout, wt_hi, wt_lo, cin * kk, (float *)tmp.p, cin * kk, 0, bf16));
  int64_t oo = 0, oi = 0;
  for (size_t i = 0; i < xs.size(); ++i) {
    const DTensor &x = xs[i], &y = ys.at(i);
    MPN_TRY(mpn_train_col2im_add_launch(ctx, (const float *)tmp.p + oo * kk * cin, x, k, s, q, y.H, y.W, dx + oi * cin));
    oo += y.N * y.H * y.W; oi += x.N * x.H * x.W;
  }
  return MPN_OK;
}

// Ls: the layers in forward order; no_dx: the slot whose gradient nobody wants (the frozen trunk part's output; a tower's
// pooled map when the trunk is frozen); p: dropout; gtop / ldtop: the gradient of an AVGPOOL's output (the concat's columns);
// more_readers: per slot the readers outside Ls (the tower levels that pool a trunk slot), null for none
static int graph_backward(mpn_model *m, const std::vector<mpn_layer> &Ls, std::map<int, GraphSlot> &S, int no_dx, float p,
                          const float *gtop, int64_t ldtop, const std::map<int, int> *more_readers = nullptr) {
  mpn_ctx *ctx = m->ctx;
  TrainState &T = *m->train;
  auto readers = [&](int s) {
    int r = 0;
    for (const mpn_layer &M : Ls) r += (M.in_slot == s) + (M.residual_slot == s);
    if (more_readers && more_readers->count(s)) r += more_readers->at(s);
    return r;
  };
  for (int li = (int)Ls.size() - 1; li >= 0; --li) {
    const mpn_layer &L = Ls[li];
    GraphSlot &O = S.at(L.out_slot), &I = S.at(L.in_slot);
    bool store;
    if (L.kind == MPN_LAYER_AVGPOOL) {
      MPN_TRY(contribute(ctx, T, I, false, &store));
      for (const DTensor &x : I.maps)
        MPN_TRY(mpn_train_avgpool_backward_launch(ctx, gtop, ldtop, x.N, (int)(x.H * x.W), (int)x.C, I.g));
    } else if (L.kind == MPN_LAYER_MAXPOOL) {         // 2x2 / stride 2 after a ReLU convolution (a VGG layer in the range)
      // pool backward, ReLU gate and split in one kernel; its planes serve the convolution below when the pool is the only
      // reader of its output
      const int64_t C = I.maps[0].C, Pi = map_pixels(I.maps);
      MPN_TRY(T.grad_split.ensure(ctx, (size_t)(Pi * C), !T.bf16));
      MPN_TRY(contribute(ctx, T, I, true, &store));
      if (!store) MPN_TRY(T.dtmp.ensure(ctx, sizeof(float) * (size_t)(Pi * C)));
      float *dst = store ? I.g : (float *)T.dtmp.p;
      auto *gs_hi = (__nv_bfloat16 *)T.grad_split.hi.p, *gs_lo = (__nv_bfloat16 *)T.grad_split.lo.p;
      int64_t oo = 0, oi = 0;
      for (size_t i = 0; i < I.maps.size(); ++i) {
        MPN_CHECK_ARG(ctx, O.maps[i].H == (I.maps[i].H + 1) / 2 && O.maps[i].W == (I.maps[i].W + 1) / 2,
                      "training the trunk: a trained max pool must be ceil-mode at odd sizes");
        MPN_TRY(mpn_train_pool_gate_split_launch(ctx, O.g + oo * C, I.maps[i], dst + oi * C, gs_hi + oi * C, gs_lo ? gs_lo + oi * C : nullptr));
        oo += O.maps[i].H * O.maps[i].W; oi += I.maps[i].H * I.maps[i].W;
      }
      if (!store) MPN_TRY(mpn_train_add_launch(ctx, I.g, dst, Pi * C));
    } else {
      const TrainParam &P = T.params[T.param_of[L.weight]];
      const int64_t cout = L.cout, cin = L.cin, k = L.kh, Po = map_pixels(O.maps);
      MPN_CHECK_ARG(ctx, O.written, "training: a trained layer's output has no reader");
      float *G = O.g;
      // 1. gate (ReLU, dropout on a 1 x 1 map) in place, and the split planes of the gated gradient: already done by the
      //    max pool above when it is this output's only reader
      MPN_TRY(T.grad_split.ensure(ctx, (size_t)(Po * cout), !T.bf16));
      auto *gs_hi = (__nv_bfloat16 *)T.grad_split.hi.p, *gs_lo = (__nv_bfloat16 *)T.grad_split.lo.p;
      const bool pooled = L.relu && li + 1 < (int)Ls.size() && Ls[li + 1].kind == MPN_LAYER_MAXPOOL && readers(L.out_slot) == 1 &&
                          Ls[li + 1].in_slot == L.out_slot;
      int64_t off = 0;
      for (size_t i = 0; !pooled && i < O.maps.size(); ++i) {
        const DTensor &y = O.maps[i];
        const bool drop = p > 0.f && L.relu && y.H == 1 && y.W == 1;
        const int64_t rows = y.N * y.H * y.W;
        MPN_TRY(mpn_train_gate_split_launch(ctx, G + off * cout, cout, rows, cout, L.relu ? &y : nullptr, drop ? 1.f / (1.f - p) : 1.f,
                                            gs_hi + off * cout, gs_lo ? gs_lo + off * cout : nullptr, cout, 0));
        off += rows;
      }
      // 2. the residual slot takes the gated gradient as it is
      if (L.residual_slot >= 0 && L.residual_slot != no_dx) {
        GraphSlot &Rs = S.at(L.residual_slot);
        MPN_TRY(contribute(ctx, T, Rs, true, &store));
        if (store) MPN_CUDA(ctx, cudaMemcpyAsync(Rs.g, G, sizeof(float) * (size_t)(Po * cout), cudaMemcpyDeviceToDevice, ctx->stream));
        else MPN_TRY(mpn_train_add_launch(ctx, Rs.g, G, Po * cout));
      }
      // 3. db (a layer without a record), dW: one GEMM over every output pixel
      if (L.bias >= 0 && T.param_of.count(L.bias)) MPN_TRY(mpn_train_colsum_launch(ctx, G, cout, Po, cout, (float *)T.params[T.param_of[L.bias]].grad.p));
      MPN_TRY(conv_wgrad(ctx, T.opGT, T.opTap, G, cout, I.maps, O.maps, (int)k, L.stride, L.pad, (float *)P.grad.p, T.bf16));
      // 4. dgrad into the input slot
      if (L.in_slot != no_dx) {
        MPN_CHECK_ARG(ctx, P.wt_hi && (P.flip || (P.wt_ld == cout && P.wt_col0 == 0)), "training: a layer with dX has no transposed weight planes");
        MPN_TRY(contribute(ctx, T, I, L.stride == 1, &store));
        MPN_TRY(conv_dgrad(ctx, T.dtmp, gs_hi, gs_lo, cout, cin, (int)k, L.stride, L.pad, P.wt_hi, P.wt_lo, I.maps, O.maps, I.g, store, T.bf16));
      }
    }
    if (O.buf) { T.grad_free.emplace(O.buf->bytes, O.buf); O.buf = nullptr; }   // every reader of O came before its producer
  }
  return MPN_OK;
}

// tower t of a fixed-batch-norm graph: from the concat's columns through its AVGPOOL and blocks; the pooled map's
// gradient (T.dpooled, (h, w, c) rows) when the trunk trains
static int tower_graph_backward(mpn_model *m, size_t t) {
  mpn_ctx *ctx = m->ctx;
  TrainState &T = *m->train;
  mpn_model::TowerExec &X = m->tex[t];
  std::map<int, GraphSlot> S;
  std::vector<mpn_layer> Ls;
  S[0].maps = {X.pooled};
  for (const LayerExec &e : X.layers) { Ls.push_back(e.L); S[e.L.out_slot].maps = {e.out}; }
  const int no_dx = T.trunk_from > 0 ? -1 : 0;
  if (T.trunk_from > 0) {
    MPN_TRY(T.dpooled[t]->ensure(ctx, sizeof(float) * (size_t)(X.pooled.N * X.pooled.H * X.pooled.W * X.pooled.C)));
    S[0].g = (float *)T.dpooled[t]->p;
  }
  return graph_backward(m, Ls, S, no_dx, T.cfg.dropout, (const float *)T.dconcat.p + X.col_off, m->concat_width);
}

// the first trunk layer the backward walks and (*no_dx) the slot whose gradient nobody wants: layer trunk_from and its
// input, or the layer above a max pool at trunk_from and the pool's output (no trained layer lies below the pool)
static int trunk_walk(const mpn_model *m, int trunk_from, int *no_dx) {
  const mpn_layer &L = m->trunk_layers[trunk_from];
  const bool pool = L.kind == MPN_LAYER_MAXPOOL;
  *no_dx = pool ? L.out_slot : L.in_slot;
  return trunk_from + (pool ? 1 : 0);
}

// the trained trunk range on the images' kept slots, from the pooled rows' gradients, which the ROI backward gathers into
// the slots the towers pool (the last one; in MultiPathNet's phase 2 also conv3_3's and conv4_3's). Those levels count as
// readers: a max pool above such a convolution adds its gradient to the ROI backward's, and the convolution gates the sum.
static int trunk_graph_backward(mpn_model *m, int n_images, const int32_t *rois_per_image) {
  TrainState &T = *m->train;
  int no_dx;
  const int k0 = trunk_walk(m, T.trunk_from, &no_dx);
  if (k0 == (int)m->trunk_layers.size()) return MPN_OK;   // the range is one max pool: nothing trains
  std::map<int, GraphSlot> S;
  for (const auto &kv : T.img_slots[0])
    for (int i = 0; i < n_images; ++i) S[kv.first].maps.push_back(T.img_slots[i].at(kv.first));
  MPN_TRY(trunk_roi_backward(m, n_images, rois_per_image, S));
  std::map<int, int> levels;
  for (const mpn_tower &Tw : m->towers)
    for (int l = 0; l < Tw.n_levels; ++l) ++levels[Tw.level_slot[l]];
  std::vector<mpn_layer> Ls(m->trunk_layers.begin() + k0, m->trunk_layers.end());
  return graph_backward(m, Ls, S, no_dx, 0.f, nullptr, 0, &levels);
}

static int train_update(mpn_model *m) {
  mpn_ctx *ctx = m->ctx;
  TrainState &T = *m->train;
  const mpn_train_config &c = T.cfg;
  const int first = T.step == 0 ? 1 : 0;
  // the method's per-step scalars (every tensor shares t = T.step); sgd's rate is clr, lr itself when lr_decay is 0
  const int method = T.optim.method;
  const mpn_optim_step hw = mpn_optim_scalars(T.optim, c.lr, c.weight_decay, T.step), hb = mpn_optim_scalars(T.optim, c.lr, 0.f, T.step);
  for (TrainParam &P : T.params) {
    if (P.idle) continue;                  // a phase-2 trunk tensor before the switch: frozen, as under nn.NoBackprop
    WeightDev &w = *m->weights[P.w];
    // an idle class head still takes the method's step with a zero gradient (Optim.lua updates every module): the
    // no-gradient kernels, which read no gradient buffer
    const float *g = (P.head >= 0 && P.head != T.head) ? nullptr : (const float *)P.grad.p;
    if (P.bias) {
      MPN_TRY(mpn_train_sgd_launch(ctx, method, (float *)w.f32.p, g, (float *)P.buf.p, P.n, hb.lr, c.momentum, c.dampening, 0.f, first,
                                   (float *)P.buf2.p, hb));
      continue;
    }
    // one pass: the master, gradient and buffer are read once; the split planes the training plan reads (same buffers, so
    // its tensor maps stay valid) and the next step's W^T planes are written with the new master; bf16: the hi planes only
    MPN_CHECK_ARG(ctx, m->w_prepared[P.w] == 1 && w.hi.p && w.lo.p, "training: the weight's split planes are not prepared");
    MPN_TRY(mpn_train_sgd_split_launch(ctx, method, (float *)w.f32.p, g, (float *)P.buf.p, P.cout, P.cin, P.kh * P.kw, hw.lr,
                                       c.momentum, c.dampening, c.weight_decay, first, (__nv_bfloat16 *)w.hi.p,
                                       T.bf16 ? nullptr : (__nv_bfloat16 *)w.lo.p,
                                       P.wt_hi, P.wt_lo, P.wt_ld, P.wt_col0, P.flip ? 1 : 0, P.fixed ? (const float *)P.a2.p : nullptr,
                                       (float *)P.buf2.p, hw));
    w.has8 = false;
  }
  return MPN_OK;
}

// MultiPathNet's switch to phase 2 (mpn_model_train_phase2, mpn_model_train_set_state): the idle trunk tensors join, the
// trunk from phase2_from trains, and the next trunk plan materialises the trained convolutions' outputs
static void phase2_switch(mpn_model *m) {
  TrainState &T = *m->train;
  for (TrainParam &P : T.params) P.idle = false;
  T.trunk_from = T.phase2_from;
  T.phase2 = true;
  m->tH = m->tW = 0;
}

// a master written from outside (mpn_model_train_set): every plane derived from it, as train_update leaves them after a
// step, from the same kernel without the step. A plane an inference plan derived (fp16 or e4m3) is dropped and that plan
// redone; so is the concatenated head of MPN_MERGE_HEADS=1. A bf16 training writes its W^T planes (hi only) and leaves
// the forward planes to the next plan, which derives them all from the master.
static int rederive_planes(mpn_model *m, const TrainParam &P) {
  mpn_ctx *ctx = m->ctx;
  WeightDev &w = *m->weights[P.w];
  const int prep = m->w_prepared[P.w];
  if (!P.bias && m->train->bf16) {
    MPN_TRY(mpn_train_split_planes_launch(ctx, (const float *)w.f32.p, P.cout, P.cin, P.kh * P.kw, nullptr, nullptr, P.wt_hi, nullptr, P.wt_ld,
                                          P.wt_col0, P.flip ? 1 : 0));
    m->w_prepared[P.w] = 0; w.has8 = false;
    m->heads_planned = false; m->train->plan = false;
    m->tH = m->tW = 0;
  } else if (!P.bias) {
    const bool split = prep == 1;
    MPN_TRY(mpn_train_split_planes_launch(ctx, (const float *)w.f32.p, P.cout, P.cin, P.kh * P.kw, split ? (__nv_bfloat16 *)w.hi.p : nullptr,
                                          split ? (__nv_bfloat16 *)w.lo.p : nullptr, P.wt_hi, P.wt_lo, P.wt_ld, P.wt_col0, P.flip ? 1 : 0));
    if (prep == 2 || w.has8) {
      if (prep == 2) m->w_prepared[P.w] = 0;
      w.has8 = false;
      m->heads_planned = false;
      m->tH = m->tW = 0;
    }
  }
  const mpn_head &hb = m->d.bbox_head;
  if (m->merged_w >= 0 && (P.head >= 0 || P.w == hb.weight || P.w == hb.bias)) { m->merged_stale = true; m->heads_planned = false; }
  m->trunk_valid = false;
  return MPN_OK;
}

extern "C" {

int mpn_train_check_optim(const mpn_model_desc *d, const mpn_train_spec *s, const mpn_train_optim *o, char *msg, int32_t msg_cap) {
  if (!d || !s || !d->towers || !d->tower_layers || !d->cls_heads || (d->n_trunk_layers > 0 && !d->trunk_layers)) return MPN_ERR_ARG;
  std::set<int> rec;
  const char *why = o ? mpn_optim_refusal(*o) : nullptr;
  const int rc = why ? MPN_ERR_ARG : train_check(d, s, rec, &why);
  if (rc != MPN_OK && msg && msg_cap > 0) snprintf(msg, (size_t)msg_cap, "%s", why);
  return rc;
}

int mpn_train_check(const mpn_model_desc *d, const mpn_train_spec *s, char *msg, int32_t msg_cap) {
  return mpn_train_check_optim(d, s, nullptr, msg, msg_cap);
}

// the trunk range from s->trunk_from trains from the first step, or in phase 2 from mpn_model_train_phase2 on: either way
// its tensors are kept in fp32 here, with their dgrad planes and every tower's first dX planes
int mpn_model_train_begin_optim(mpn_model *m, const mpn_train_config *cfg, const mpn_train_spec *s, const mpn_train_optim *o) {
  if (!m || !cfg || !s || (s->n_fixed > 0 && !s->fixed_scale)) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, !m->train, "training already begun (mpn_model_train_end first)");
  MPN_TRY(train_opts_ok(m));
  const mpn_model_desc d = model_view(m);
  const char *why = o ? mpn_optim_refusal(*o) : nullptr;
  if (why) return mpn_fail(ctx, MPN_ERR_ARG, why);
  std::set<int> recs;
  if (train_check(&d, s, recs, &why) != MPN_OK) return mpn_fail(ctx, MPN_ERR_ARG, why);
  const std::set<int> *rec = s->n_fixed > 0 ? &recs : nullptr;
  const int from = s->trunk_from;                 // the trunk range (0: none)
  const bool phase2 = s->phase2 != 0;
  MPN_CHECK_ARG(ctx, cfg->lr >= 0.f && cfg->momentum >= 0.f && cfg->dampening >= 0.f && cfg->dampening <= 1.f && cfg->weight_decay >= 0.f &&
                     cfg->dropout >= 0.f && cfg->dropout < 1.f && cfg->bbox_regression >= 0.f && std::isfinite(cfg->lr),
                "training config out of range (lr, momentum, weight decay, bbox weight >= 0; 0 <= dampening <= 1; 0 <= dropout < 1)");
  const char *envm = getenv("MPN_MERGE_HEADS");
  MPN_CHECK_ARG(ctx, !(envm && envm[0] == '1'), "training does not run with MPN_MERGE_HEADS=1 (merged head planes are an inference experiment)");
  std::unique_ptr<TrainState> T(new TrainState());
  T->cfg = *cfg;
  if (o) T->optim = *o;
  const bool sgd = T->optim.method == MPN_OPTIM_SGD;
  const bool two = T->optim.method == MPN_OPTIM_ADAM || T->optim.method == MPN_OPTIM_ADAMAX;
  T->bf16 = ctx->opt_train_bf16 == 1;
  T->trunk_from = phase2 ? 0 : from;
  T->phase2_from = phase2 ? from : 0;
  for (size_t t = 0; t < m->towers.size(); ++t) T->dpooled.emplace_back(new DevBuf());
  if (rec) T->fixed = recs;
  for (const mpn_tower &Tw : m->towers) T->graph_tower.push_back(graph_tower(&d, Tw, rec));
  // flat: a Linear over a FLATTENed (kh, kw, cin) map, whose K is the whole vector
  auto add = [&](int w, int cout, int cin, int kh, int kw, bool bias, bool flat = false) -> int {
    if (w < 0) return MPN_OK;
    MPN_CHECK_ARG(ctx, w < (int)m->weights.size(), "layer weight index out of range");
    MPN_CHECK_ARG(ctx, m->w_prepared[w] == 0 && m->weights[w]->f32.p,
                  "training needs the fp32 weights: begin it before the model's first heads / detect call (and, when the trunk trains, "
                  "before its first trunk call), or rebuild the model");
    MPN_CHECK_ARG(ctx, bias || (flat ? (int64_t)cin * kh * kw : (int64_t)cin) % 64 == 0, TAIL_MSG);
    TrainParam P; P.w = w; P.n = m->weights[w]->n; P.bias = bias; P.cout = cout; P.cin = cin; P.kh = kh; P.kw = kw;
    MPN_CHECK_ARG(ctx, P.n == (bias ? (int64_t)cout : (int64_t)cout * cin * kh * kw), "parameter size does not match its layer");
    T->param_of[w] = (int)T->params.size();
    T->params.push_back(std::move(P));
    return MPN_OK;
  };
  for (const mpn_tower &Tw : m->towers) {
    int fc = 0, fh = 0, fw = 0, flat_slot = -1;
    // the FLATTEN's input geometry: the pooled map (slot 0) or a 1x1 convolution's output, both pooled_h x pooled_w
    std::map<int, int> ch; ch[0] = 0;
    for (int i = 0; i < Tw.n_layers; ++i) {
      const mpn_layer &L = m->tower_layers[Tw.first_layer + i];
      if (L.kind == MPN_LAYER_FLATTEN) {
        fh = Tw.pooled_h; fw = Tw.pooled_w; flat_slot = L.out_slot;
        fc = ch.count(L.in_slot) && ch[L.in_slot] > 0 ? ch[L.in_slot] : -1;
        continue;
      }
      ch[L.out_slot] = L.cout;
      if (L.in_slot == flat_slot) {
        if (fc < 0) fc = L.cin / (fh * fw);          // FLATTEN of the pooled map: its channels follow from the Linear
        MPN_CHECK_ARG(ctx, fc * fh * fw == L.cin, "Linear after FLATTEN: input size mismatch");
        MPN_TRY(add(L.weight, L.cout, fc, fh, fw, false, /*flat=*/true));
      } else {
        MPN_TRY(add(L.weight, L.cout, L.cin, L.kh, L.kw, false));
      }
      if (!T->fixed.count(L.weight)) MPN_TRY(add(L.bias, L.cout, 0, 0, 0, true));   // a recorded layer's bias is a constant
    }
  }
  for (size_t k = 0; k < m->cls_heads.size(); ++k) {        // every class head of an integral model, then the bbox head
    const mpn_head &h = m->cls_heads[k];
    MPN_TRY(add(h.weight, h.cout, h.col_len, 1, 1, false));
    MPN_TRY(add(h.bias, h.cout, 0, 0, 0, true));
    for (int w : {h.weight, h.bias}) if (w >= 0) T->params[T->param_of[w]].head = (int)k;
  }
  MPN_TRY(add(m->d.bbox_head.weight, m->d.bbox_head.cout, m->d.bbox_head.col_len, 1, 1, false));
  MPN_TRY(add(m->d.bbox_head.bias, m->d.bbox_head.cout, 0, 0, 0, true));
  for (int li = from; from > 0 && li < (int)m->trunk_layers.size(); ++li) {
    const mpn_layer &L = m->trunk_layers[li];
    if (L.kind != MPN_LAYER_CONV) continue;
    MPN_TRY(add(L.weight, L.cout, L.cin, L.kh, L.kw, false));
    if (!T->fixed.count(L.weight)) MPN_TRY(add(L.bias, L.cout, 0, 0, 0, true));
    for (int w : {L.weight, L.bias}) if (T->param_of.count(w)) T->params[T->param_of[w]].idle = phase2;
  }
  for (TrainParam &P : T->params) {
    MPN_TRY(P.grad.ensure(ctx, sizeof(float) * (size_t)P.n));
    MPN_TRY(P.buf.ensure(ctx, sizeof(float) * (size_t)P.n));
    MPN_CUDA(ctx, cudaMemsetAsync(P.grad.p, 0, sizeof(float) * (size_t)P.n, ctx->stream));
    MPN_CUDA(ctx, cudaMemsetAsync(P.buf.p, 0, sizeof(float) * (size_t)P.n, ctx->stream));
    if (!two) continue;
    MPN_TRY(P.buf2.ensure(ctx, sizeof(float) * (size_t)P.n));
    MPN_CUDA(ctx, cudaMemsetAsync(P.buf2.p, 0, sizeof(float) * (size_t)P.n, ctx->stream));
  }
  // a recorded layer's a^2 per output channel (fp32), the factor of its gradient in sgd's update, or a itself for the
  // W-space rule of the other methods (mpn_optim_elem_fixed); the scales of layers that do not train (a frozen trunk)
  // are not needed
  std::vector<std::vector<float>> a2_host(s->n_fixed);
  for (int j = 0; j < s->n_fixed; ++j) {
    if (!T->param_of.count(s->fixed_weight[j])) continue;
    TrainParam &P = T->params[T->param_of[s->fixed_weight[j]]];
    MPN_CHECK_ARG(ctx, s->fixed_scale[j], "fixed batch norm: a scale array is missing");
    a2_host[j].resize(P.cout);
    for (int c = 0; c < P.cout; ++c) {
      const float a = s->fixed_scale[j][c];
      MPN_CHECK_ARG(ctx, std::isfinite(a), "fixed batch norm: a scale is not finite");
      MPN_CHECK_ARG(ctx, sgd || a != 0.f, "fixed batch norm: a scale of 0 under an optim method other than sgd (W = W' / a)");
      a2_host[j][c] = sgd ? a * a : a;
    }
    P.fixed = true;
    MPN_TRY(P.a2.ensure(ctx, sizeof(float) * (size_t)P.cout));
    MPN_CUDA(ctx, cudaMemcpyAsync(P.a2.p, a2_host[j].data(), sizeof(float) * (size_t)P.cout, cudaMemcpyHostToDevice, ctx->stream));
  }
  // W^T planes of every layer whose dX is needed: every head (one buffer [cls_0 .. cls_{K-1} ; bbox] when they read the
  // same columns, else one per class head and one for the bbox head) and every tower
  // convolution above the tower's first; built here from the masters, then rewritten by each update
  auto make_wt = [&](std::vector<int> ws) -> int {
    int64_t ld = 0;
    for (int w : ws) ld += (T->params[T->param_of[w]].cout + 63) / 64 * 64;
    const TrainParam &P0 = T->params[T->param_of[ws[0]]];
    const int64_t Kin = (int64_t)P0.cin * P0.kh * P0.kw;
    T->wt_bufs.emplace_back(new SplitBuf());
    SplitBuf &b = *T->wt_bufs.back();
    MPN_TRY(b.ensure(ctx, (size_t)(Kin * ld), !T->bf16));
    MPN_CUDA(ctx, cudaMemsetAsync(b.hi.p, 0, 2 * (size_t)(Kin * ld), ctx->stream));
    if (b.lo.p) MPN_CUDA(ctx, cudaMemsetAsync(b.lo.p, 0, 2 * (size_t)(Kin * ld), ctx->stream));
    int64_t col = 0;
    for (int w : ws) {
      TrainParam &P = T->params[T->param_of[w]];
      P.wt_hi = (__nv_bfloat16 *)b.hi.p; P.wt_lo = (__nv_bfloat16 *)b.lo.p; P.wt_ld = ld; P.wt_col0 = col;
      const int fhw = P.kh * P.kw;
      MPN_TRY(mpn_train_transpose_launch(ctx, (const float *)m->weights[w]->f32.p, nullptr, nullptr, Kin, P.cout, Kin, fhw > 1 ? 1 : 0, P.cin,
                                         fhw, P.wt_hi, P.wt_lo, ld, col));
      col += (P.cout + 63) / 64 * 64;
    }
    return MPN_OK;
  };
  {
    const mpn_head &hc = m->cls_heads[0], &hb = m->d.bbox_head;
    if (hc.col_begin == hb.col_begin && hc.col_len == hb.col_len) {
      std::vector<int> ws;
      for (const mpn_head &h : m->cls_heads) ws.push_back(h.weight);
      ws.push_back(hb.weight);
      MPN_TRY(make_wt(ws));
    } else {
      for (const mpn_head &h : m->cls_heads) MPN_TRY(make_wt({h.weight}));
      MPN_TRY(make_wt({hb.weight}));
    }
    // the dgrad planes of a 3x3 / stride 1 convolution: [Cin][ky][kx][Cout], rotated by 180 degrees
    auto make_flip = [&](int w) -> int {
      TrainParam &P = T->params[T->param_of[w]];
      T->wt_bufs.emplace_back(new SplitBuf());
      SplitBuf &b = *T->wt_bufs.back();
      MPN_TRY(b.ensure(ctx, (size_t)P.n, !T->bf16));
      P.wt_hi = (__nv_bfloat16 *)b.hi.p; P.wt_lo = (__nv_bfloat16 *)b.lo.p; P.wt_ld = P.cout; P.wt_col0 = 0; P.flip = true;
      return mpn_train_transpose_launch(ctx, (const float *)m->weights[w]->f32.p, nullptr, nullptr, (int64_t)P.cin * 9, P.cout,
                                        (int64_t)P.cin * 9, 3, P.cin, 9, P.wt_hi, P.wt_lo, P.wt_ld, 0);
    };
    // graph backward: every convolution whose input gradient is wanted (its input is not the pooled map of a frozen trunk,
    // nor the frozen trunk part's output): the rotated planes for 3x3 / stride 1, else W^T [(ky, kx, ci)][Cout] for one GEMM
    auto graph_planes = [&](const mpn_layer &L, int no_dx_slot) -> int {
      if (L.kind != MPN_LAYER_CONV || L.in_slot == no_dx_slot) return MPN_OK;
      return (L.kh == 3 && L.stride == 1) ? make_flip(L.weight) : make_wt({L.weight});
    };
    for (size_t t = 0; t < m->towers.size(); ++t) {
      const mpn_tower &Tw = m->towers[t];
      if (T->graph_tower[t]) {
        for (int i = 0; i < Tw.n_layers; ++i) MPN_TRY(graph_planes(m->tower_layers[Tw.first_layer + i], from > 0 ? -1 : 0));
        continue;
      }
      bool below = from > 0;                   // a trained trunk below the tower: its first layer has a dX too
      for (int i = 0; i < Tw.n_layers; ++i) {
        const mpn_layer &L = m->tower_layers[Tw.first_layer + i];
        if (L.kind != MPN_LAYER_CONV) continue;
        if (below) MPN_TRY(make_wt({L.weight}));
        below = true;
      }
    }
    if (from > 0) {                            // phase 2's planes too, from the masters phase 1 leaves unchanged
      int no_dx;
      for (int li = trunk_walk(m, from, &no_dx); li < (int)m->trunk_layers.size(); ++li) MPN_TRY(graph_planes(m->trunk_layers[li], no_dx));
      if (!phase2) m->tH = m->tW = 0;          // the next trunk plan materialises the trained convolutions' outputs
    }
  }
  for (cudaEvent_t &e : T->ev) MPN_CUDA(ctx, cudaEventCreate(&e));
  m->train = std::move(T);
  m->heads_planned = false;
  return MPN_OK;
}

int mpn_model_train_begin(mpn_model *m, const mpn_train_config *cfg, const mpn_train_spec *s) {
  return mpn_model_train_begin_optim(m, cfg, s, nullptr);
}

int mpn_model_train_step_dev(mpn_model *m, int32_t n_images, const float *const *images_dev, const int32_t *image_hw,
                             const int32_t *rois_per_image, const float *boxes_dev, const int32_t *labels_dev,
                             const float *bbox_targets_dev, float *losses_dev) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train, "no training begun (mpn_model_train_begin)");
  MPN_TRY(train_opts_ok(m));
  TrainState &T = *m->train;
  MPN_CHECK_ARG(ctx, n_images >= 1 && images_dev && image_hw && rois_per_image && boxes_dev && labels_dev && bbox_targets_dev && losses_dev,
                "training step: an argument is missing");
  int64_t R = 0;
  for (int i = 0; i < n_images; ++i) {
    MPN_CHECK_ARG(ctx, images_dev[i] && image_hw[2 * i] > 0 && image_hw[2 * i + 1] > 0 && image_hw[2 * i] <= m->d.max_h &&
                       image_hw[2 * i + 1] <= m->d.max_w, "training step: an image is missing or larger than max_h x max_w");
    MPN_CHECK_ARG(ctx, rois_per_image[i] >= 0, "training step: negative ROI count");
    R += rois_per_image[i];
  }
  MPN_CHECK_ARG(ctx, R > 0 && R <= m->d.max_rois, "training step: R out of range (0 < R <= max_rois)");
  const int C = m->d.num_classes;
  struct PlanScheme {                  // the step's trunk and heads plans take the training's numerics
    mpn_model *m;
    PlanScheme(mpn_model *m_, bool bf16) : m(m_) { m->plan_train_bf16 = bf16; }
    ~PlanScheme() { m->plan_train_bf16 = false; }
  } scheme(m, T.bf16);
  MPN_TRY(ensure_trunk(m, image_hw[0], image_hw[1]));
  // the per-image trunk plans below leave heads_planned unset; the tower plans depend on R and the channel counts only
  if (!T.plan || m->hR != R || m->tex.empty()) {
    if (!T.plan) forget_derived_planes(m);
    m->plan_split_only = true;
    const int rc = plan_heads(m, R);
    m->plan_split_only = false;
    MPN_TRY(rc);
    T.plan = true;
  }
  MPN_TRY(T.rois5.ensure(ctx, sizeof(float) * 5 * (size_t)R));
  MPN_TRY(T.dlogits.ensure(ctx, sizeof(float) * (size_t)(R * C)));
  MPN_TRY(T.dbbox.ensure(ctx, sizeof(float) * (size_t)(R * 4 * C)));
  MPN_CUDA(ctx, cudaEventRecord(T.ev[0], ctx->stream));
  MPN_TRY(mpn_train_rois5_launch(ctx, boxes_dev, R, (float *)T.rois5.p));
  // trunk per image, then its ROIs into rows [off, off + R_i) of the pooled tensors
  const mpn_tower &T0 = m->towers[0];
  const int64_t bins = (int64_t)T0.pooled_h * T0.pooled_w;
  int64_t off = 0;
  for (int i = 0; i < n_images; ++i) {
    MPN_TRY(ensure_trunk(m, image_hw[2 * i], image_hw[2 * i + 1]));
    refresh_roi_jobs(m);
    m->heads_planned = true;                       // the tower plans do not depend on the image size
    MPN_TRY(run_trunk(m, images_dev[i]));
    const int64_t Ri = rois_per_image[i];
    if (Ri > 0) {
      RoiJobs J = m->jobs;
      for (int k = 0; k < J.n; ++k) { J.j[k].out_hi += off * bins * J.j[k].out_ld; J.j[k].out_lo += off * bins * J.j[k].out_ld; }
      MPN_TRY(mpn_roi_pool_fused_launch(ctx, J, (const float *)T.rois5.p + off * 5, Ri, T0.pooled_w, T0.pooled_h, m->d.roi_variant));
    }
    off += Ri;
    if (T.trunk_from > 0) MPN_TRY(keep_trunk_slots(m, i));
  }
  MPN_CUDA(ctx, cudaEventRecord(T.ev[1], ctx->stream));
  MPN_TRY(run_towers_heads(m, R, &T));
  MPN_TRY(mpn_train_criteria_launch(ctx, (const float *)m->cls_logits.p + (size_t)T.head * R * C, (const float *)m->bbox_raw.p, labels_dev,
                                    bbox_targets_dev, (int)R, C,
                                    T.cfg.bbox_regression, (float *)T.dlogits.p, (float *)T.dbbox.p, losses_dev));
  MPN_CUDA(ctx, cudaEventRecord(T.ev[2], ctx->stream));
  MPN_TRY(train_backward(m, R));
  if (T.trunk_from > 0) MPN_TRY(trunk_graph_backward(m, n_images, rois_per_image));
  MPN_CUDA(ctx, cudaEventRecord(T.ev[3], ctx->stream));
  MPN_TRY(train_update(m));
  MPN_CUDA(ctx, cudaEventRecord(T.ev[4], ctx->stream));
  T.last_R = R; T.last_images = n_images; T.last_head = T.head;
  ++T.step;
  // the cached trunk features are the minibatch's last image: heads / detect without a new trunk call must not pool from it
  m->trunk_valid = false;
  return MPN_OK;
}

int mpn_model_train_phase_ms(mpn_model *m, float *ms) {
  if (!m || !ms) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train && m->train->step > 0, "no training step yet");
  TrainState &T = *m->train;
  MPN_CUDA(ctx, cudaEventSynchronize(T.ev[4]));
  for (int k = 0; k < 4; ++k) MPN_CUDA(ctx, cudaEventElapsedTime(&ms[k], T.ev[k], T.ev[k + 1]));
  return MPN_OK;
}

int mpn_model_train_step(mpn_model *m, int32_t n_images, const float *const *images, const int32_t *image_hw, const int32_t *rois_per_image,
                         const float *boxes, const int32_t *labels, const float *bbox_targets, float *losses) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train, "no training begun (mpn_model_train_begin)");
  MPN_CHECK_ARG(ctx, n_images >= 1 && images && image_hw && rois_per_image && boxes && labels && bbox_targets && losses,
                "training step: an argument is missing");
  TrainState &T = *m->train;
  const int C = m->d.num_classes;
  int64_t R = 0;
  for (int i = 0; i < n_images; ++i) {
    MPN_CHECK_ARG(ctx, images[i] && image_hw[2 * i] > 0 && image_hw[2 * i + 1] > 0 && image_hw[2 * i] <= m->d.max_h &&
                       image_hw[2 * i + 1] <= m->d.max_w, "training step: an image is missing or larger than max_h x max_w");
    MPN_CHECK_ARG(ctx, rois_per_image[i] >= 0, "training step: negative ROI count");
    R += rois_per_image[i];
  }
  MPN_CHECK_ARG(ctx, R > 0 && R <= m->d.max_rois, "training step: R out of range (0 < R <= max_rois)");
  for (int64_t r = 0; r < R; ++r) MPN_CHECK_ARG(ctx, labels[r] >= 1 && labels[r] <= C, "training step: a label is outside 1..num_classes");
  if ((int)T.images.size() < n_images) T.images.resize(n_images);
  std::vector<const float *> ptrs(n_images);
  for (int i = 0; i < n_images; ++i) {
    const size_t b = sizeof(float) * 3 * (size_t)image_hw[2 * i] * image_hw[2 * i + 1];
    MPN_TRY(T.images[i].ensure(ctx, b));
    MPN_CUDA(ctx, cudaMemcpyAsync(T.images[i].p, images[i], b, cudaMemcpyHostToDevice, ctx->stream));
    ptrs[i] = (const float *)T.images[i].p;
  }
  MPN_TRY(T.boxes.ensure(ctx, sizeof(float) * 4 * (size_t)R));
  MPN_TRY(T.labels.ensure(ctx, sizeof(int32_t) * (size_t)R));
  MPN_TRY(T.targets.ensure(ctx, sizeof(float) * 4 * (size_t)(R * C)));
  MPN_TRY(T.losses.ensure(ctx, sizeof(float) * 4));
  MPN_CUDA(ctx, cudaMemcpyAsync(T.boxes.p, boxes, sizeof(float) * 4 * (size_t)R, cudaMemcpyHostToDevice, ctx->stream));
  MPN_CUDA(ctx, cudaMemcpyAsync(T.labels.p, labels, sizeof(int32_t) * (size_t)R, cudaMemcpyHostToDevice, ctx->stream));
  MPN_CUDA(ctx, cudaMemcpyAsync(T.targets.p, bbox_targets, sizeof(float) * 4 * (size_t)(R * C), cudaMemcpyHostToDevice, ctx->stream));
  MPN_TRY(mpn_model_train_step_dev(m, n_images, ptrs.data(), image_hw, rois_per_image, (const float *)T.boxes.p, (const int32_t *)T.labels.p,
                                   (const float *)T.targets.p, (float *)T.losses.p));
  MPN_CUDA(ctx, cudaMemcpyAsync(losses, T.losses.p, sizeof(float) * 3, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_TRY(mpn_ovf_copy_async(ctx, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return mpn_ovf_test(ctx);
}

int mpn_model_train_select_head(mpn_model *m, int32_t k) {
  if (!m) return MPN_ERR_ARG;
  MPN_CHECK_ARG(m->ctx, m->train, "no training begun (mpn_model_train_begin)");
  const int K = (int)m->cls_heads.size();
  if (k < 0 || k >= K)
    return mpn_fail(m->ctx, MPN_ERR_ARG, "train_select_head: class head " + std::to_string(k) + " out of range 0.." + std::to_string(K - 1));
  m->train->head = k;
  return MPN_OK;
}

int mpn_model_train_set_lr(mpn_model *m, float lr) {
  if (!m) return MPN_ERR_ARG;
  MPN_CHECK_ARG(m->ctx, m->train, "no training begun (mpn_model_train_begin)");
  MPN_CHECK_ARG(m->ctx, lr >= 0.f && std::isfinite(lr), "lr must be finite and >= 0");
  m->train->cfg.lr = lr;
  return MPN_OK;
}

int mpn_model_train_decay(mpn_model *m, float factor) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train, "no training begun (mpn_model_train_begin)");
  MPN_CHECK_ARG(ctx, factor >= 0.f && std::isfinite(factor), "decay factor must be finite and >= 0");
  m->train->cfg.lr *= factor;
  if (m->train->optim.method != MPN_OPTIM_SGD) return MPN_OK;     // train.lua scales u.dfdx, which only sgd's state has
  for (TrainParam &P : m->train->params) MPN_TRY(mpn_train_scale_launch(ctx, (float *)P.buf.p, P.n, factor));
  return MPN_OK;
}

int mpn_model_train_phase2(mpn_model *m, float lr) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train, "no training begun (mpn_model_train_begin)");
  TrainState &T = *m->train;
  MPN_CHECK_ARG(ctx, T.phase2_from > 0, "phase 2: training did not begin with mpn_train_spec.phase2 = 1");
  MPN_CHECK_ARG(ctx, !T.phase2, "phase 2: the switch was already made");
  MPN_CHECK_ARG(ctx, lr < 0.f || std::isfinite(lr), "phase 2: lr must be finite (< 0 keeps the rate and the buffers)");
  if (lr >= 0.f) {                                // train.lua:243-257: the new rate, every momentum buffer (u.dfdx) zeroed
    T.cfg.lr = lr;
    if (T.optim.method == MPN_OPTIM_SGD)          // the other methods' state is not u.dfdx: it is kept
      for (TrainParam &P : T.params) MPN_CUDA(ctx, cudaMemsetAsync(P.buf.p, 0, sizeof(float) * (size_t)P.n, ctx->stream));
  }
  phase2_switch(m);                               // the trunk tensors join with zero state
  return MPN_OK;
}

int mpn_model_train_get(mpn_model *m, int32_t weight, int32_t what, float *out, int64_t capacity) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train, "no training begun (mpn_model_train_begin)");
  MPN_CHECK_ARG(ctx, m->train->param_of.count(weight), "not a trainable parameter tensor");
  MPN_CHECK_ARG(ctx, what >= 0 && what <= 3, "what: 0 weight, 1 gradient of the last step, 2 momentum buffer (first state), 3 second state");
  const TrainParam &P = m->train->params[m->train->param_of[weight]];
  MPN_CHECK_ARG(ctx, what != 3 || P.buf2.p, "what 3: the optim method has no second state (adam and adamax have one)");
  MPN_CHECK_ARG(ctx, out && capacity >= P.n, "output buffer missing or too small");
  if (what == 1 && P.head >= 0 && P.head != m->train->last_head) {    // an idle head's gradient is zero (nn.SelectTable)
    std::fill(out, out + P.n, 0.f);
    return MPN_OK;
  }
  const void *src = what == 0 ? m->weights[weight]->f32.p : (what == 1 ? P.grad.p : (what == 2 ? P.buf.p : P.buf2.p));
  MPN_CUDA(ctx, cudaMemcpyAsync(out, src, sizeof(float) * (size_t)P.n, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

int mpn_model_train_set(mpn_model *m, int32_t weight, int32_t what, const float *src, int64_t n) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train, "no training begun (mpn_model_train_begin)");
  TrainState &T = *m->train;
  MPN_CHECK_ARG(ctx, T.param_of.count(weight), "train_set: weight " + std::to_string(weight) + " is not a trained tensor");
  MPN_CHECK_ARG(ctx, what == 0 || what == 2 || what == 3, "train_set: what: 0 weight, 2 momentum buffer");
  const TrainParam &P = T.params[T.param_of[weight]];
  MPN_CHECK_ARG(ctx, what != 3 || P.buf2.p, "train_set: what 3: the optim method has no second state (adam and adamax have one)");
  MPN_CHECK_ARG(ctx, src && n == P.n, "train_set: weight " + std::to_string(weight) + " has " + std::to_string(P.n) + " elements, got " +
                                          std::to_string(n));
  void *dst = what == 0 ? m->weights[weight]->f32.p : (what == 2 ? P.buf.p : P.buf2.p);
  MPN_CUDA(ctx, cudaMemcpyAsync(dst, src, sizeof(float) * (size_t)n, cudaMemcpyHostToDevice, ctx->stream));
  if (what == 0) MPN_TRY(rederive_planes(m, P));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

int mpn_model_train_get_state(mpn_model *m, mpn_train_state *out) {
  if (!m || !out) return MPN_ERR_ARG;
  MPN_CHECK_ARG(m->ctx, m->train, "no training begun (mpn_model_train_begin)");
  const TrainState &T = *m->train;
  out->step = T.step; out->lr = T.cfg.lr; out->head = T.head; out->last_head = T.last_head; out->phase2 = T.phase2 ? 1 : 0;
  return MPN_OK;
}

int mpn_model_train_set_state(mpn_model *m, const mpn_train_state *s) {
  if (!m || !s) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CHECK_ARG(ctx, m->train, "no training begun (mpn_model_train_begin)");
  TrainState &T = *m->train;
  const int K = (int)m->cls_heads.size();
  MPN_CHECK_ARG(ctx, s->step >= 0 && s->step <= (int64_t)UINT32_MAX, "train_set_state: step out of range 0..2^32-1");
  MPN_CHECK_ARG(ctx, s->lr >= 0.f && std::isfinite(s->lr), "train_set_state: lr must be finite and >= 0");
  MPN_CHECK_ARG(ctx, s->head >= 0 && s->head < K && s->last_head >= 0 && s->last_head < K,
                "train_set_state: class head out of range 0.." + std::to_string(K - 1));
  MPN_CHECK_ARG(ctx, s->phase2 == 0 || s->phase2 == 1, "train_set_state: phase2 is 0 or 1");
  MPN_CHECK_ARG(ctx, !s->phase2 || T.phase2_from > 0, "train_set_state: phase 2 on a training that did not begin with mpn_train_spec.phase2 = 1");
  MPN_CHECK_ARG(ctx, s->phase2 || !T.phase2, "train_set_state: the switch to phase 2 was already made and cannot be undone");
  if (s->phase2 && !T.phase2) phase2_switch(m);   // the buffers stay: the checkpoint's are set next
  T.step = (uint32_t)s->step; T.cfg.lr = s->lr; T.head = s->head; T.last_head = s->last_head;
  return MPN_OK;
}

int mpn_model_train_dropout_mask(mpn_model *m, int32_t tower, int32_t layer, uint8_t *out, int64_t capacity, int64_t *n_out) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train && m->train->step > 0, "no training step yet");
  MPN_CHECK_ARG(ctx, tower >= 0 && tower < (int)m->towers.size(), "unknown tower");
  const mpn_tower &Tw = m->towers[tower];
  MPN_CHECK_ARG(ctx, layer >= 0 && layer < Tw.n_layers && m->tower_layers[Tw.first_layer + layer].kind == MPN_LAYER_CONV, "not a layer of the tower");
  const int64_t n = m->train->last_R * m->tower_layers[Tw.first_layer + layer].cout;
  if (n_out) *n_out = n;
  if (!out) return MPN_OK;
  MPN_CHECK_ARG(ctx, capacity >= n, "output buffer too small");
  MPN_CHECK_ARG(ctx, m->train->cfg.dropout > 0.f, "dropout is off (p = 0): every element is kept");
  void *tmp = nullptr;
  MPN_TRY(mpn_scratch(ctx, (size_t)n, &tmp));
  MPN_TRY(mpn_train_dropout_mask_launch(ctx, n, m->train->cfg.seed, m->train->step - 1, tower, layer, m->train->cfg.dropout, (uint8_t *)tmp));
  MPN_CUDA(ctx, cudaMemcpyAsync(out, tmp, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

int mpn_model_train_relu_gate(mpn_model *m, int32_t tower, int32_t layer, uint8_t *out, int64_t capacity, int64_t *n_out) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train && m->train->step > 0 && m->train->plan, "no training step since the last inference call");
  MPN_CHECK_ARG(ctx, tower >= 0 && tower < (int)m->tex.size(), "unknown tower");
  const auto &layers = m->tex[tower].layers;
  MPN_CHECK_ARG(ctx, layer >= 0 && layer < (int)layers.size() && layers[layer].L.kind == MPN_LAYER_CONV && layers[layer].L.relu,
                "not a ReLU layer of the tower");
  const DTensor &y = layers[layer].out;
  const int64_t rows = y.N * y.H * y.W, n = rows * y.C;
  if (n_out) *n_out = n;
  if (!out) return MPN_OK;
  MPN_CHECK_ARG(ctx, capacity >= n, "output buffer too small");
  void *tmp = nullptr;
  MPN_TRY(mpn_scratch(ctx, (size_t)n, &tmp));
  MPN_TRY(mpn_train_gate_mask_launch(ctx, y, rows, y.C, (uint8_t *)tmp));
  MPN_CUDA(ctx, cudaMemcpyAsync(out, tmp, (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

int mpn_model_train_outputs(mpn_model *m, float *cls_logits, float *bbox_deltas) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train && m->train->step > 0 && m->train->plan, "no training step since the last inference call");
  const int64_t R = m->train->last_R, C = m->d.num_classes;
  const float *logits = (const float *)m->cls_logits.p + (size_t)m->train->last_head * R * C;      // the trained head's
  if (cls_logits) MPN_CUDA(ctx, cudaMemcpyAsync(cls_logits, logits, sizeof(float) * (size_t)(R * C), cudaMemcpyDeviceToHost, ctx->stream));
  if (bbox_deltas) MPN_CUDA(ctx, cudaMemcpyAsync(bbox_deltas, m->bbox_raw.p, sizeof(float) * (size_t)(R * 4 * C), cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

int mpn_model_train_trunk_slot(mpn_model *m, int32_t image, int32_t slot, float *out_nchw, int64_t capacity, int32_t *C, int32_t *H,
                               int32_t *W) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, m->train && m->train->step > 0 && m->train->trunk_from > 0, "no training step of the trunk yet");
  const TrainState &T = *m->train;
  MPN_CHECK_ARG(ctx, image >= 0 && image < T.last_images && T.img_slots[image].count(slot), "image or trunk slot not kept by the last step");
  const DTensor &t = T.img_slots[image].at(slot);
  const int64_t n = t.C * t.H * t.W;
  if (C) *C = (int32_t)t.C; if (H) *H = (int32_t)t.H; if (W) *W = (int32_t)t.W;
  if (!out_nchw) return MPN_OK;
  MPN_CHECK_ARG(ctx, capacity >= n, "output buffer too small");
  void *tmp = nullptr;
  MPN_TRY(mpn_scratch(ctx, sizeof(float) * (size_t)n, &tmp));
  MPN_TRY(mpn_nhwc_split_to_nchw_launch(ctx, t, (float *)tmp));
  MPN_CUDA(ctx, cudaMemcpyAsync(out_nchw, tmp, sizeof(float) * (size_t)n, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

// ---- test hooks of the trunk-training kernels, on host buffers (synchronous)
static int upload(mpn_ctx *ctx, DevBuf &b, const void *src, size_t bytes) {
  MPN_TRY(b.ensure(ctx, bytes + 256));
  MPN_CUDA(ctx, cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, ctx->stream));
  return MPN_OK;
}
static DTensor planes_view(DevBuf &hi, DevBuf &lo, int64_t H, int64_t W, int64_t C) {
  DTensor t; t.hi = (__nv_bfloat16 *)hi.p; t.lo = (__nv_bfloat16 *)lo.p; t.N = 1; t.H = H; t.W = W; t.C = C; t.ld = C;
  return t;
}
static int download(mpn_ctx *ctx, void *dst, const DevBuf &b, size_t bytes) {
  MPN_CUDA(ctx, cudaMemcpyAsync(dst, b.p, bytes, cudaMemcpyDeviceToHost, ctx->stream));
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  return MPN_OK;
}

int mpn_debug_roi_backward_nhwc(mpn_ctx *ctx, const uint16_t *hi, const uint16_t *lo, int32_t H, int32_t W, int32_t C, const float *rois,
                                int64_t R, int32_t PW, int32_t PH, float scale, int32_t variant, const float *grad_out, float *grad) {
  if (!ctx) return MPN_ERR_ARG;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, hi && lo && rois && grad_out && grad && H > 0 && W > 0 && C > 0 && R >= 0 && PW > 0 && PH > 0 && (variant == 1 || variant == 2),
                "roi backward hook: bad arguments");
  const size_t cells = (size_t)H * W, bins = (size_t)PW * PH;
  DevBuf h, l, r, go, am, out;
  MPN_TRY(upload(ctx, h, hi, 2 * cells * C)); MPN_TRY(upload(ctx, l, lo, 2 * cells * C));
  MPN_TRY(upload(ctx, r, rois, sizeof(float) * 5 * (size_t)R)); MPN_TRY(upload(ctx, go, grad_out, sizeof(float) * (size_t)R * bins * C));
  MPN_TRY(am.ensure(ctx, sizeof(int32_t) * ((size_t)R * bins * C + 1))); MPN_TRY(out.ensure(ctx, sizeof(float) * cells * C));
  MPN_TRY(mpn_roi_backward_nhwc_launch(ctx, planes_view(h, l, H, W, C), (const float *)r.p, R, PW, PH, scale, variant, (const float *)go.p,
                                       (int32_t *)am.p, (float *)out.p));
  return download(ctx, grad, out, sizeof(float) * cells * C);
}

int mpn_debug_roi_backward_jobs(mpn_ctx *ctx, const uint16_t *hi, const uint16_t *lo, int32_t H, int32_t W, int32_t C, const float *rois,
                                int64_t R, int32_t PW, int32_t PH, int32_t variant, int32_t n_jobs, const int32_t *region, const float *scale,
                                const int32_t *normalize, const int64_t *ld, const int32_t *ch_off, const float *const *grad_out, float *grad,
                                double *ab, int32_t *argmax) {
  if (!ctx) return MPN_ERR_ARG;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, hi && lo && rois && grad && region && scale && normalize && ld && ch_off && grad_out && H > 0 && W > 0 && C > 0 && R >= 0 &&
                     PW > 0 && PH > 0 && (variant == 1 || variant == 2) && n_jobs >= 1 && n_jobs <= MAX_ROI_BWD_JOBS,
                "roi backward jobs hook: bad arguments");
  const size_t cells = (size_t)H * W, bins = (size_t)PW * PH;
  DevBuf h, l, r, out, am, abd;
  std::vector<DevBuf> go(n_jobs);
  MPN_TRY(upload(ctx, h, hi, 2 * cells * C)); MPN_TRY(upload(ctx, l, lo, 2 * cells * C));
  MPN_TRY(upload(ctx, r, rois, sizeof(float) * 5 * (size_t)R));
  MPN_TRY(am.ensure(ctx, sizeof(int32_t) * ((size_t)n_jobs * R * bins * C + 1))); MPN_TRY(out.ensure(ctx, sizeof(float) * cells * C));
  MPN_TRY(abd.ensure(ctx, sizeof(double) * (2 * (size_t)n_jobs * R + 1)));
  MPN_CUDA(ctx, cudaMemsetAsync(abd.p, 0, sizeof(double) * (2 * (size_t)n_jobs * R + 1), ctx->stream));
  const DTensor f = planes_view(h, l, H, W, C);
  RoiBwdJobs J{};
  J.n = n_jobs;
  for (int k = 0; k < n_jobs; ++k) {
    MPN_CHECK_ARG(ctx, grad_out[k] && region[k] >= 0 && region[k] <= 3 && ch_off[k] >= 0 && ld[k] >= ch_off[k] + C,
                  "roi backward jobs hook: a job's region, gradient or channel range is bad");
    MPN_TRY(upload(ctx, go[k], grad_out[k], sizeof(float) * (size_t)R * bins * (size_t)ld[k]));
    RoiBwdJob &b = J.j[k];
    b.region = region[k]; b.scale = scale[k]; b.grad = (const float *)go[k].p; b.ld = ld[k]; b.ch_off = ch_off[k];
    b.argmax = (const int32_t *)am.p + (size_t)k * R * bins * C; b.ab = nullptr;
    MPN_TRY(mpn_roi_argmax_nhwc_launch(ctx, f, (const float *)r.p, R, PW, PH, b.region, b.scale, variant, const_cast<int32_t *>(b.argmax)));
    if (normalize[k]) {
      double *abk = (double *)abd.p + 2 * (size_t)k * R;
      MPN_TRY(mpn_roi_norm_ab_launch(ctx, f, R, PW, PH, b, abk));
      b.ab = abk;
    }
  }
  MPN_TRY(mpn_roi_backward_jobs_launch(ctx, f, (const float *)r.p, R, PW, PH, variant, J, (float *)out.p));
  if (ab) MPN_TRY(download(ctx, ab, abd, sizeof(double) * 2 * (size_t)n_jobs * R));
  if (argmax) MPN_TRY(download(ctx, argmax, am, sizeof(int32_t) * (size_t)n_jobs * R * bins * C));
  return download(ctx, grad, out, sizeof(float) * cells * C);
}

int mpn_debug_pool_backward(mpn_ctx *ctx, const uint16_t *y_hi, const uint16_t *y_lo, int32_t H, int32_t W, int32_t C, const float *grad_pool,
                            float *grad) {
  if (!ctx) return MPN_ERR_ARG;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, y_hi && y_lo && grad_pool && grad && H > 0 && W > 0 && C > 0, "pool backward hook: bad arguments");
  const size_t n = (size_t)H * W * C, np = (size_t)((H + 1) / 2) * ((W + 1) / 2) * C;
  DevBuf h, l, gp, out, ah, al;
  MPN_TRY(upload(ctx, h, y_hi, 2 * n)); MPN_TRY(upload(ctx, l, y_lo, 2 * n)); MPN_TRY(upload(ctx, gp, grad_pool, sizeof(float) * np));
  // "train_bf16" on: the hi-only form of a bf16 training step
  MPN_TRY(out.ensure(ctx, sizeof(float) * n)); MPN_TRY(ah.ensure(ctx, 2 * n));
  if (ctx->opt_train_bf16 != 1) MPN_TRY(al.ensure(ctx, 2 * n));
  MPN_TRY(mpn_train_pool_gate_split_launch(ctx, (const float *)gp.p, planes_view(h, l, H, W, C), (float *)out.p, (__nv_bfloat16 *)ah.p,
                                           (__nv_bfloat16 *)al.p));
  return download(ctx, grad, out, sizeof(float) * n);
}

int mpn_debug_conv_backward(mpn_ctx *ctx, int32_t n_images, const int32_t *image_hw, int32_t cin, int32_t cout, int32_t k, int32_t stride,
                            const uint16_t *x_hi, const uint16_t *x_lo, const float *g, const float *w, float *dw, float *dx) {
  if (!ctx) return MPN_ERR_ARG;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, n_images >= 1 && image_hw && x_hi && x_lo && g && w && dw && dx && cin > 0 && cin % 8 == 0 && cout > 0 && cout % 64 == 0 &&
                     (k == 1 || k == 3) && (stride == 1 || stride == 2),
                "conv backward hook: bad arguments (cin a multiple of 8, cout of 64, k 1 or 3, stride 1 or 2)");
  const int q = (k - 1) / 2;
  std::vector<DTensor> xs, ys;
  int64_t Pi = 0, Po = 0;
  for (int i = 0; i < n_images; ++i) {
    DTensor x; x.N = 1; x.H = image_hw[2 * i]; x.W = image_hw[2 * i + 1]; x.C = cin; x.ld = cin;
    MPN_CHECK_ARG(ctx, x.H > 0 && x.W > 0, "conv backward hook: empty image");
    DTensor y; y.N = 1; y.H = (x.H + 2 * q - k) / stride + 1; y.W = (x.W + 2 * q - k) / stride + 1; y.C = cout; y.ld = cout;
    xs.push_back(x); ys.push_back(y);
    Pi += x.H * x.W; Po += y.H * y.W;
  }
  const int64_t kk = (int64_t)k * k;
  const size_t nw = (size_t)cout * cin * kk;
  DevBuf xh, xl, gd, wd, dwd, dxd, tmp;
  SplitBuf gs, wt, opGT, opTap;
  MPN_TRY(upload(ctx, xh, x_hi, 2 * (size_t)Pi * cin)); MPN_TRY(upload(ctx, xl, x_lo, 2 * (size_t)Pi * cin));
  MPN_TRY(upload(ctx, gd, g, sizeof(float) * (size_t)Po * cout)); MPN_TRY(upload(ctx, wd, w, sizeof(float) * nw));
  const bool bf16 = ctx->opt_train_bf16 == 1;          // the operands and GEMMs of a bf16 training step
  MPN_TRY(gs.ensure(ctx, (size_t)Po * cout, !bf16)); MPN_TRY(wt.ensure(ctx, nw, !bf16));
  MPN_TRY(dwd.ensure(ctx, sizeof(float) * nw)); MPN_TRY(dxd.ensure(ctx, sizeof(float) * (size_t)Pi * cin));
  // dx as the first contribution to a slot: stride 1 stores, the col2im of stride 2 adds to zeros
  if (stride == 2) MPN_CUDA(ctx, cudaMemsetAsync(dxd.p, 0, sizeof(float) * (size_t)Pi * cin, ctx->stream));
  // the operands as the step makes them: the gradient's split planes, the weight planes from the fp32 weight (make_flip /
  // make_wt of mpn_model_train_begin)
  MPN_TRY(mpn_train_gate_split_launch(ctx, (float *)gd.p, cout, Po, cout, nullptr, 1.f, (__nv_bfloat16 *)gs.hi.p, (__nv_bfloat16 *)gs.lo.p, cout, 0));
  const bool flip = k == 3 && stride == 1;
  MPN_TRY(mpn_train_transpose_launch(ctx, (const float *)wd.p, nullptr, nullptr, (int64_t)cin * kk, cout, (int64_t)cin * kk,
                                     flip ? 3 : (k > 1 ? 1 : 0), cin, (int)kk, (__nv_bfloat16 *)wt.hi.p, (__nv_bfloat16 *)wt.lo.p, cout, 0));
  int64_t off = 0;
  for (DTensor &x : xs) {
    x.hi = (__nv_bfloat16 *)xh.p + off * cin; x.lo = (__nv_bfloat16 *)xl.p + off * cin;
    off += x.H * x.W;
  }
  MPN_TRY(conv_wgrad(ctx, opGT, opTap, (const float *)gd.p, cout, xs, ys, k, stride, q, (float *)dwd.p, bf16));
  MPN_TRY(conv_dgrad(ctx, tmp, (const __nv_bfloat16 *)gs.hi.p, (const __nv_bfloat16 *)gs.lo.p, cout, cin, k, stride, q,
                     (const __nv_bfloat16 *)wt.hi.p, (const __nv_bfloat16 *)wt.lo.p, xs, ys, (float *)dxd.p, stride == 1, bf16));
  MPN_TRY(download(ctx, dw, dwd, sizeof(float) * nw));
  return download(ctx, dx, dxd, sizeof(float) * (size_t)Pi * cin);
}

int mpn_model_train_end(mpn_model *m) {
  if (!m) return MPN_ERR_ARG;
  mpn_ctx *ctx = m->ctx;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  if (!m->train) return MPN_OK;
  MPN_CUDA(ctx, cudaStreamSynchronize(ctx->stream));
  forget_derived_planes(m);                         // the next plan derives from the trained masters, then frees them
  m->train.reset();
  m->heads_planned = false;
  return MPN_OK;
}

}  // extern "C"

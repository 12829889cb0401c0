// conv_gemm.cuh — shared declarations for the convolution / GEMM engines.
#pragma once
#include "common.cuh"
#include <cuda.h>   // CUtensorMap type only; the encode entry point is fetched at run time

// One convolution (or Linear = 1x1 conv on a 1x1 map) in the internal NHWC split-bf16
// representation. y[n,ho,wo,co] = sum_{kh,kw,ci} x[n, ho*s+kh-p, wo*s+kw-p, ci] * w[co,(kh,kw,ci)]
//                                 + bias[co] (+ residual) (ReLU)
// fp32 output of a split-K GEMM scattered by column range (several small heads computed by ONE GEMM): the reduce pass
// writes column c in [c0, c1) of segment s to ptr[pixel * ld + (c - c0)]
struct OutSeg { int c0, c1; float *ptr; long long ld; };
struct OutScatter { int n = 0; OutSeg seg[8]; };

// Operand scheme of the wgmma engine (a template parameter of its kernel):
//   BF16X3: A and B as split-bf16 hi / lo planes, A_lo*B_hi + A_hi*B_lo + A_hi*B_hi per k16 — the fp32-faithful default;
//   FP16X2: A as fp16 hi / lo planes, B as ONE scaled fp16 plane, A_lo*B + A_hi*B (fc6 / fc7 "w16");
//   BF16X1: the opt-in bf16 inference mode (mpn_ctx_set_option "bf16"): only the hi planes are loaded, A_hi*B_hi per k16.
//   FP8X1:  the opt-in fp8 inference mode (option "fp8"): A and B as ONE e4m3 plane each (fp8_e4m3.cuh), A8*B8 per k32;
//           the epilogue multiplies the accumulator by 2^-(e_a[sample] + e_w[channel]).
// Every scheme writes the same output formats (split planes, fp32, split-K partials, fused pool).
enum class OperandScheme : int { BF16X3 = 0, FP16X2 = 1, BF16X1 = 2, FP8X1 = 3 };

struct ConvProblem {
  DTensor x;                       // input  (split planes)
  const __nv_bfloat16 *w_hi = nullptr, *w_lo = nullptr;   // [Cout][kh*kw*conv_k_pad(Cin)], K order (kh,kw,ci)
  const float *bias = nullptr;     // [Cout] or null
  int Cout = 0, kh = 1, kw = 1, stride = 1, pad = 0;
  int pad_w = -1;                  // horizontal pad when it differs from the vertical `pad` (1 x n / n x 1 kernels); -1: = pad
  int relu = 0;
  DTensor res;                     // optional residual (split planes), same geometry as y
  DTensor y;                       // output: split planes (hi/lo) and/or f32; y.ld / f32_ld = pixel strides
  int64_t y_f32_ld = 0;
  DTensor pool;                    // optional: 2x2/2 ceil max pool of y written by the epilogue (3x3 / stride 1 plans only)
  int pool_only = 0;               // 1: y itself is not written (nobody else reads it)
  // 1: rows are independent samples (per-ROI layers): the plan may depend on (Cout, K) only where it affects rounding —
  // the N tile and the split-K count — so a row's result does not change with the number of rows in
  // the call (chunked forward == full forward, bit for bit: modules/test.lua:85-98, ImageDetect.lua:126-133)
  int m_invariant = 0;
  // "w16" numerics for the big per-ROI Linears (fc6 / fc7): the weight as ONE fp16 plane scaled by a power of two
  // (w16[co][k] = rn_fp16(w * scale), w16_inv_scale = 1 / scale), the activation still hi + lo bf16: two tensor-core
  // products per MAC (A_hi x W + A_lo x W) instead of three; the epilogue multiplies the accumulator by w16_inv_scale.
  const void *w16 = nullptr; float w16_inv_scale = 1.f;
  // 1: bf16 inference numerics — the hi planes of x and w only (rn_bf16 of the fp32 values), ONE product per MAC;
  // the lo planes are not read. Not combinable with w16. conv_ref_launch honours it too.
  int bf16 = 0;
  // fp8 inference numerics (fp8 = 1): x8 = e4m3 plane [pixel][x.C] (dense) of 2^x8_exp[sample] * x.hi, one exponent per
  // sample (x.H * x.W pixels: the image in the trunk, the ROI in per-ROI layers); w8 = e4m3 plane [Cout][kh*kw*Cin] of
  // 2^w8_exp[co] * w_hi (w8_exp readable up to Cout rounded up to 128). Not combinable with w16 or bf16; conv_ref_launch
  // reads the same operands.
  int fp8 = 0;
  const uint8_t *x8 = nullptr; const int *x8_exp = nullptr;
  const uint8_t *w8 = nullptr; const int *w8_exp = nullptr;
  OutScatter scatter;             // n > 0: split-K plans only (conv_tc_launch rejects it otherwise)
  // 1: a trunk weight gradient (flat GEMM, K = the minibatch's pixels): when K >= 16384 the planner splits K into as many
  // parts as fill the SMs. Only the training step's wgrad sets it, so no other GEMM's plan or summation order changes.
  int wide_k_split = 0;
  // 1: a per-ROI Linear without a bias — the first factor of an SVD-compressed fc6 / fc7 (models.svd_compress,
  // utils.SVDlinear's nn.LinearNB): deep K, narrow N. The planner splits its K so that the units of a 1000-ROI call fill
  // the SMs; the split count is a function of (K, Cout, SM count), so a row's result still does not depend on R.
  // Only such layers set it, so no other layer's plan changes.
  int fill_split = 0;
};

inline int conv_pad_w(const ConvProblem &p) { return p.pad_w < 0 ? p.pad : p.pad_w; }

// Group g of G of a grouped convolution (CaffeNet's conv2, conv4, conv5) as an engine problem of its own. p is the whole
// layer: x and y its input and output, w_hi / w_lo Torch's Cout x Cin/G x kh x kw laid out [Cout][kh][kw][conv_k_pad(Cin/G)],
// bias Cout. The group reads the channel view [g Cin/G, (g+1) Cin/G) of x (the A map's channel extent is the view's C and its
// strides come from ld, so the TMA zero-fills past the group's last channel: a K tail as any other), writes the channel
// view [g Cout/G, (g+1) Cout/G) of y, and takes its Cout/G contiguous weight rows and biases. Cin/G and Cout/G are
// multiples of 8, so each view starts on 16 bytes.
inline ConvProblem conv_group(const ConvProblem &p, int G, int g) {
  ConvProblem q = p;
  const int64_t ci = p.x.C / G, co = p.Cout / G, row = (int64_t)p.kh * p.kw * conv_k_pad(ci);
  q.x.hi += g * ci; q.x.lo += g * ci; q.x.C = ci;
  q.y.hi += g * co; q.y.lo += g * co; q.y.C = co;
  q.Cout = (int)co;
  q.w_hi += g * co * row; q.w_lo += g * co * row;
  if (q.bias) q.bias += g * co;
  return q;
}

// Plan = tile decomposition + TMA descriptors for one ConvProblem on the wgmma path.
struct ConvPlan {
  CUtensorMap tmA_hi, tmA_lo, tmB_hi, tmB_lo;
  int BN = 0;                      // 64 / 128 / 256
  int tn = 0, th = 0, tw = 0;      // 128 output pixels per M tile = tn*th*tw
  int tiles_img = 0, tiles_h = 0, tiles_w = 0, tiles_n = 0;
  int splitk = 1, kb_per_split = 0; // split-K over K blocks for tiny GEMMs (deterministic two-pass reduce)
  int mode = 0;                    // 0 generic implicit GEMM, 1 = 3x3/s1/p1 with 16 x 8 patches (fused 2x2 pooling possible)
  int flat = 0;                    // 1: 1x1/s1/p0 => pixels treated as one flat axis
  OperandScheme ops = OperandScheme::BF16X3;   // FP16X2 when ConvProblem::w16 is set, BF16X1 / FP8X1 when ConvProblem::bf16 / fp8 is
  int valid = 0;
};

int conv_tc_plan(mpn_ctx *ctx, const ConvProblem &p, ConvPlan &plan);
int conv_tc_launch(mpn_ctx *ctx, const ConvProblem &p, const ConvPlan &plan);
int conv_ref_launch(mpn_ctx *ctx, const ConvProblem &p);           // CUDA-core fp32 check kernel
// first-layer direct conv: x is NCHW fp32 (N x Cin x H x W), w fp32 [Cout][Cin][kh][kw] (Torch layout)
int conv_direct_nchw_launch(mpn_ctx *ctx, const float *x_nchw, int N, int Cin, int H, int W, const float *w,
                            const float *bias, int Cout, int kh, int kw, int stride, int pad, int relu,
                            DTensor &y, const float *w_host = nullptr, const float *bias_host = nullptr);
// first layer (3x3/1/1, Cin 3, Cout 64) on the tensor cores: x NCHW fp32, w fp32 [64][27] (Torch layout), y NHWC split planes
int conv1_tc_launch(mpn_ctx *ctx, const float *x_nchw, int N, int H, int W, const float *w_dev, const float *bias_dev, int relu,
                    DTensor &y);
double conv_flops(const ConvProblem &p);
// fp8 numerics (fp8.cu): the e4m3 plane of the hi plane of x (dense, [pixel][x.C]) and its per-sample exponents
// (x.N samples of x.H * x.W pixels); a sample without a valid scale raises the ctx's flag (bit 2, mpn_ovf_test fails)
int mpn_fp8_quantize_launch(mpn_ctx *ctx, const DTensor &x, uint8_t *q8, int *exps);
// a weight's hi plane [rows][K] -> e4m3 plane + per-row exponents (rows up to `rows_pad` get exponent 0)
int mpn_fp8_weight_launch(mpn_ctx *ctx, const __nv_bfloat16 *w_hi, int64_t rows, int64_t K, int64_t rows_pad, uint8_t *q8, int *exps);

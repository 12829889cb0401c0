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

struct ConvProblem {
  DTensor x;                       // input  (split planes)
  const __nv_bfloat16 *w_hi = nullptr, *w_lo = nullptr;   // [Cout][kh*kw*Cin], K order (kh,kw,ci)
  const float *bias = nullptr;     // [Cout] or null
  int Cout = 0, kh = 1, kw = 1, stride = 1, pad = 0;
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
  OutScatter scatter;              // n > 0: split-K plans only (conv_tc_launch rejects it otherwise)
};

// Plan = tile decomposition + TMA descriptors for one ConvProblem on the wgmma path.
struct ConvPlan {
  CUtensorMap tmA_hi, tmA_lo, tmB_hi, tmB_lo;
  int BN = 0;                      // 64 / 128 / 256
  int tn = 0, th = 0, tw = 0;      // 128 output pixels per M tile = tn*th*tw
  int tiles_img = 0, tiles_h = 0, tiles_w = 0, tiles_n = 0;
  int splitk = 1, kb_per_split = 0; // split-K over K blocks for tiny GEMMs (deterministic two-pass reduce)
  int mode = 0;                    // 0 generic implicit GEMM, 1 = 3x3/s1/p1 with 16 x 8 patches (fused 2x2 pooling possible)
  int flat = 0;                    // 1: 1x1/s1/p0 => pixels treated as one flat axis
  int w16 = 0;                     // 1: B operand = one fp16 plane (ConvProblem::w16), 2 MMAs per k16
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

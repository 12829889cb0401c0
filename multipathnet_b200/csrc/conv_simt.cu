// conv_simt.cu — CUDA-core convolution kernels (sm_90a).
//  * conv_direct_nchw_kernel: the FIRST trunk layer (Cin=3: VGG conv1_1 K=27, ResNet conv1
//    7x7/s2 K=147). K is too small for a 64-wide tensor-core K block, the layer is ~0.6 % of
//    the trunk FLOPs and HBM-write-bound; it reads the NCHW fp32 image exactly as
//    ImageDetect hands it over (ImageDetect.lua:167-169) and emits NHWC split-bf16 planes.
//  * conv_ref_kernel: a deliberately plain one-thread-per-output fp32 kernel over the same
//    split-bf16 operands as the wgmma engine. Verification/debug only (mpn_model_set_conv_impl
//    = 1, mpn_*_check impl=1): it lets tests separate "tensor-core engine bug" from "graph bug". In the bf16 numerics
//    (ConvProblem::bf16) it reads only the hi planes, the operand rounding of the engine's BF16X1 kernels; in the fp8
//    numerics (ConvProblem::fp8) the same e4m3 planes and exponents as the engine's FP8X1 kernels.
#include "conv_gemm.cuh"
#include "fp8_e4m3.cuh"
#include <stdlib.h>

namespace {

constexpr int DC_CO = 16;   // output channels per thread

__global__ void __launch_bounds__(256)
conv_direct_nchw_kernel(const float *__restrict__ x, int N, int Cin, int H, int W, const float *__restrict__ w,
                        const float *__restrict__ bias, int Cout, int kh, int kw, int stride, int pad, int relu,
                        int Ho, int Wo, __nv_bfloat16 *__restrict__ oh, __nv_bfloat16 *__restrict__ ol,
                        long long ld) {
  // s_w[k][16]: the block's 16 output channels contiguous per filter element, so one broadcast
  // LDS.128 feeds 4 FMAs (a [co][k] layout costs one LDS per FMA and is LSU-issue-bound: 197 us -> ~30 us)
  extern __shared__ float4 s_w4[];
  float *s_w = reinterpret_cast<float *>(s_w4);
  const int K = Cin * kh * kw;
  const int co0 = blockIdx.y * DC_CO;
  for (int i = threadIdx.x; i < DC_CO * K; i += blockDim.x) {
    const int k = i / DC_CO, c = i - k * DC_CO;
    const int co = co0 + c;
    s_w[i] = (co < Cout) ? w[(size_t)co * K + k] : 0.f;
  }
  __syncthreads();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)N * Ho * Wo) return;
  const int wo = (int)(pix % Wo), ho = (int)((pix / Wo) % Ho), n = (int)(pix / ((long long)Wo * Ho));
  float acc[DC_CO];
#pragma unroll
  for (int c = 0; c < DC_CO; ++c) acc[c] = 0.f;
  for (int ci = 0; ci < Cin; ++ci)
    for (int r = 0; r < kh; ++r) {
      const int hi = ho * stride + r - pad;
      if (hi < 0 || hi >= H) continue;
      const float *xrow = x + (((size_t)n * Cin + ci) * H + hi) * W;
      for (int q = 0; q < kw; ++q) {
        const int wi = wo * stride + q - pad;
        if (wi < 0 || wi >= W) continue;
        const float v = __ldg(xrow + wi);
        const float4 *wk = s_w4 + ((ci * kh + r) * kw + q) * (DC_CO / 4);
#pragma unroll
        for (int c4 = 0; c4 < DC_CO / 4; ++c4) {
          const float4 ww = wk[c4];
          acc[4 * c4 + 0] = fmaf(v, ww.x, acc[4 * c4 + 0]);
          acc[4 * c4 + 1] = fmaf(v, ww.y, acc[4 * c4 + 1]);
          acc[4 * c4 + 2] = fmaf(v, ww.z, acc[4 * c4 + 2]);
          acc[4 * c4 + 3] = fmaf(v, ww.w, acc[4 * c4 + 3]);
        }
      }
    }
#pragma unroll
  for (int g = 0; g < DC_CO / 8; ++g) {
    const int c = co0 + g * 8;
    if (c >= Cout) break;
    uint32_t ph[4], pl[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float f0 = acc[g * 8 + 2 * t] + (bias ? __ldg(bias + c + 2 * t) : 0.f);
      float f1 = acc[g * 8 + 2 * t + 1] + (bias ? __ldg(bias + c + 2 * t + 1) : 0.f);
      if (relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
      __nv_bfloat16 h0, l0, h1, l1;
      split_bf16(f0, h0, l0); split_bf16(f1, h1, l1);
      ph[t] = pack_bf16x2(h0, h1); pl[t] = pack_bf16x2(l0, l1);
    }
    *reinterpret_cast<uint4 *>(oh + pix * ld + c) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
    *reinterpret_cast<uint4 *>(ol + pix * ld + c) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
  }
}

// VGG conv1_1 specialisation: 3x3 / s1 / p1 / Cin=3, fully unrolled (27 taps): per tap 1 predicated LDG, 4 broadcast
// LDS.128 and 16 FMAs, no loop or index arithmetic. Same smem weight layout and epilogue as the generic kernel.
__global__ void __launch_bounds__(256)
conv_direct_3x3c3_kernel(const float *__restrict__ x, int N, int H, int W, const float *__restrict__ w,
                         const float *__restrict__ bias, int Cout, int relu, __nv_bfloat16 *__restrict__ oh,
                         __nv_bfloat16 *__restrict__ ol, long long ld) {
  __shared__ float4 s_w4[27 * (DC_CO / 4)];
  float *s_w = reinterpret_cast<float *>(s_w4);
  const int co0 = blockIdx.y * DC_CO;
  for (int i = threadIdx.x; i < DC_CO * 27; i += blockDim.x) {
    const int k = i / DC_CO, c = i - k * DC_CO;
    s_w[i] = (co0 + c < Cout) ? w[(size_t)(co0 + c) * 27 + k] : 0.f;
  }
  __syncthreads();
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)N * H * W) return;
  const int wo = (int)(pix % W), ho = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
  float acc[DC_CO];
#pragma unroll
  for (int c = 0; c < DC_CO; ++c) acc[c] = 0.f;
  const float *xn = x + (size_t)n * 3 * H * W;
#pragma unroll
  for (int ci = 0; ci < 3; ++ci)
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hi = ho + r - 1;
      const bool hok = (hi >= 0) && (hi < H);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int wi = wo + q - 1;
        const bool ok = hok && (wi >= 0) && (wi < W);
        const float v = ok ? __ldg(xn + ((size_t)ci * H + hi) * W + wi) : 0.f;
        const float4 *wk = s_w4 + ((ci * 3 + r) * 3 + q) * (DC_CO / 4);
#pragma unroll
        for (int c4 = 0; c4 < DC_CO / 4; ++c4) {
          const float4 ww = wk[c4];
          acc[4 * c4 + 0] = fmaf(v, ww.x, acc[4 * c4 + 0]);
          acc[4 * c4 + 1] = fmaf(v, ww.y, acc[4 * c4 + 1]);
          acc[4 * c4 + 2] = fmaf(v, ww.z, acc[4 * c4 + 2]);
          acc[4 * c4 + 3] = fmaf(v, ww.w, acc[4 * c4 + 3]);
        }
      }
    }
#pragma unroll
  for (int g = 0; g < DC_CO / 8; ++g) {
    const int c = co0 + g * 8;
    if (c >= Cout) break;
    uint32_t ph[4], pl[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      float f0 = acc[g * 8 + 2 * t] + (bias ? __ldg(bias + c + 2 * t) : 0.f);
      float f1 = acc[g * 8 + 2 * t + 1] + (bias ? __ldg(bias + c + 2 * t + 1) : 0.f);
      if (relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
      __nv_bfloat16 h0, l0, h1, l1;
      split_bf16(f0, h0, l0); split_bf16(f1, h1, l1);
      ph[t] = pack_bf16x2(h0, h1); pl[t] = pack_bf16x2(l0, l1);
    }
    *reinterpret_cast<uint4 *>(oh + pix * ld + c) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
    *reinterpret_cast<uint4 *>(ol + pix * ld + c) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
  }
}

// VGG conv1_1, second specialisation (Cout = 64): the whole 64 x 27 filter bank + bias travels as a __grid_constant__
// kernel parameter (7 KB, constant bank), so every FMA takes its weight as an immediate constant operand: no LDS at
// all (the smem-broadcast version is LSU-bound at ~110 us; this one is FMA-bound). One thread = one pixel x 64 channels.
struct Conv1Params { float w[64 * 27]; float b[64]; };

__global__ void __launch_bounds__(128)
conv_direct_3x3c3_o64_kernel(const float *__restrict__ x, int N, int H, int W, const __grid_constant__ Conv1Params cp,
                             int relu, __nv_bfloat16 *__restrict__ oh, __nv_bfloat16 *__restrict__ ol, long long ld) {
  const long long pix = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (pix >= (long long)N * H * W) return;
  const int wo = (int)(pix % W), ho = (int)((pix / W) % H), n = (int)(pix / ((long long)W * H));
  const float *xn = x + (size_t)n * 3 * H * W;
  float in[27];
#pragma unroll
  for (int ci = 0; ci < 3; ++ci)
#pragma unroll
    for (int r = 0; r < 3; ++r) {
      const int hi = ho + r - 1;
      const bool hok = (hi >= 0) && (hi < H);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int wi = wo + q - 1;
        const bool ok = hok && (wi >= 0) && (wi < W);
        in[(ci * 3 + r) * 3 + q] = ok ? __ldg(xn + ((size_t)ci * H + hi) * W + wi) : 0.f;
      }
    }
#pragma unroll
  for (int g = 0; g < 8; ++g) {                       // 8 output channels at a time -> one 16-byte store per plane
    float f[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      float a = cp.b[g * 8 + e];
#pragma unroll
      for (int k = 0; k < 27; ++k) a = fmaf(in[k], cp.w[(g * 8 + e) * 27 + k], a);
      f[e] = relu ? fmaxf(a, 0.f) : a;
    }
    uint32_t ph[4], pl[4];
#pragma unroll
    for (int t = 0; t < 4; ++t) {
      __nv_bfloat16 h0, l0, h1, l1;
      split_bf16(f[2 * t], h0, l0); split_bf16(f[2 * t + 1], h1, l1);
      ph[t] = pack_bf16x2(h0, h1); pl[t] = pack_bf16x2(l0, l1);
    }
    *reinterpret_cast<uint4 *>(oh + pix * ld + g * 8) = make_uint4(ph[0], ph[1], ph[2], ph[3]);
    *reinterpret_cast<uint4 *>(ol + pix * ld + g * 8) = make_uint4(pl[0], pl[1], pl[2], pl[3]);
  }
}

struct RefParams {
  const __nv_bfloat16 *xh, *xl; long long xld; int N, H, W, Cin;
  const __nv_bfloat16 *wh, *wl;
  const __half *w16; float w16_inv;        // "w16" layers: one scaled fp16 weight plane instead of wh / wl
  int xfmt, ofmt; unsigned *ovf;           // plane formats of the input / output (0 = bf16 split, 1 = fp16 split)
  int bf16;                                // 1: operands = the hi planes only (bf16 numerics)
  const float *bias; int Cout, kh, kw, stride, pad, pad_w, relu, Ho, Wo;
  const __nv_bfloat16 *rh, *rl; long long rld;
  __nv_bfloat16 *oh, *ol; long long old_;
  float *of; long long ofld;
  const uint8_t *x8, *w8; const int *x8e, *w8e;   // fp8 numerics: e4m3 planes (x8 dense, ld = Cin) and exponents, or null
};

__global__ void __launch_bounds__(256) conv_ref_kernel(const RefParams p) {
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  const long long total = (long long)p.N * p.Ho * p.Wo * p.Cout;
  if (idx >= total) return;
  const int co = (int)(idx % p.Cout); const long long pix = idx / p.Cout;
  const int wo = (int)(pix % p.Wo), ho = (int)((pix / p.Wo) % p.Ho), n = (int)(pix / ((long long)p.Wo * p.Ho));
  float acc = 0.f;
  const long long Cp = conv_k_pad(p.Cin);           // a tap's channels in the weight layout (ConvProblem::w_hi)
  const long long Ktot = (long long)p.kh * p.kw * Cp;
  for (int r = 0; r < p.kh; ++r) {
    const int hi = ho * p.stride + r - p.pad;
    if (hi < 0 || hi >= p.H) continue;
    for (int q = 0; q < p.kw; ++q) {
      const int wi = wo * p.stride + q - p.pad_w;
      if (wi < 0 || wi >= p.W) continue;
      const long long xo = (((long long)n * p.H + hi) * p.W + wi) * p.xld;
      const long long wo_ = (long long)co * Ktot + (long long)(r * p.kw + q) * Cp;
      if (p.x8) {
        const long long xo8 = (((long long)n * p.H + hi) * p.W + wi) * p.Cin;
        for (int ci = 0; ci < p.Cin; ++ci)
          acc = fmaf(mpn_fp8::e4m3_value(p.x8[xo8 + ci]), mpn_fp8::e4m3_value(p.w8[wo_ + ci]), acc);
        continue;
      }
      for (int ci = 0; ci < p.Cin; ++ci) {
        const float a = p.bf16 ? __bfloat162float(p.xh[xo + ci])
                               : join_planes(p.xfmt, __bfloat16_as_ushort(p.xh[xo + ci]), __bfloat16_as_ushort(p.xl[xo + ci]));
        const float b = p.w16 ? __half2float(p.w16[wo_ + ci])
                              : (p.bf16 ? __bfloat162float(p.wh[wo_ + ci]) : join_bf16(p.wh[wo_ + ci], p.wl[wo_ + ci]));
        acc = fmaf(a, b, acc);
      }
    }
  }
  if (p.w16) acc *= p.w16_inv;
  if (p.x8) acc *= mpn_fp8::pow2(-(p.x8e[n] + p.w8e[co]));
  if (p.bias) acc += p.bias[co];
  if (p.rh) acc += join_bf16(p.rh[pix * p.rld + co], p.rl[pix * p.rld + co]);
  if (p.relu) acc = fmaxf(acc, 0.f);
  if (p.oh) {
    uint32_t h2, l2;
    split_x2(p.ofmt, acc, 0.f, h2, l2, p.ovf);
    p.oh[pix * p.old_ + co] = __ushort_as_bfloat16((unsigned short)(h2 & 0xffffu)); p.ol[pix * p.old_ + co] = __ushort_as_bfloat16((unsigned short)(l2 & 0xffffu));
  }
  if (p.of) p.of[pix * p.ofld + co] = acc;
}

}  // namespace

int conv_direct_nchw_launch(mpn_ctx *ctx, const float *x_nchw, int N, int Cin, int H, int W, const float *w,
                            const float *bias, int Cout, int kh, int kw, int stride, int pad, int relu, DTensor &y,
                            const float *w_host, const float *bias_host) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_CONV_DIRECT);
  MPN_CHECK_ARG(ctx, Cout % 8 == 0, "conv_direct: Cout must be a multiple of 8");
  const long long pixels = (long long)N * y.H * y.W;
  if (pixels <= 0) return MPN_OK;
  const size_t smem = sizeof(float) * DC_CO * Cin * kh * kw;
  MPN_CHECK_ARG(ctx, smem <= 48 * 1024, "conv_direct: filter too large");
  dim3 grid((unsigned)((pixels + 255) / 256), (unsigned)((Cout + DC_CO - 1) / DC_CO));
  if (Cin == 3 && kh == 3 && kw == 3 && stride == 1 && pad == 1 && Cout == 64 && y.ld == 64 && bias) {
    const char *e = getenv("MPN_CONV1_TC");           // debug knob: 0 = CUDA-core kernels below
    if (!(e && e[0] == '0')) return conv1_tc_launch(ctx, x_nchw, N, H, W, w, bias, relu, y);
  }
  if (Cin == 3 && kh == 3 && kw == 3 && stride == 1 && pad == 1 && Cout == 64 && w_host && y.ld % 8 == 0) {
    Conv1Params cp;
    memcpy(cp.w, w_host, sizeof(cp.w));
    if (bias_host) memcpy(cp.b, bias_host, sizeof(cp.b)); else memset(cp.b, 0, sizeof(cp.b));
    conv_direct_3x3c3_o64_kernel<<<(unsigned)((pixels + 127) / 128), 128, 0, ctx->stream>>>(x_nchw, N, H, W, cp, relu, y.hi, y.lo, y.ld);
    MPN_LAUNCHED(ctx);
    return MPN_OK;
  }
  if (Cin == 3 && kh == 3 && kw == 3 && stride == 1 && pad == 1) {
    conv_direct_3x3c3_kernel<<<grid, 256, 0, ctx->stream>>>(x_nchw, N, H, W, w, bias, Cout, relu, y.hi, y.lo, y.ld);
    MPN_LAUNCHED(ctx);
    return MPN_OK;
  }
  conv_direct_nchw_kernel<<<grid, 256, smem, ctx->stream>>>(x_nchw, N, Cin, H, W, w, bias, Cout, kh, kw, stride, pad,
                                                          relu, (int)y.H, (int)y.W, y.hi, y.lo, y.ld);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int conv_ref_launch(mpn_ctx *ctx, const ConvProblem &p) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_CONV_TC);
  RefParams r;
  r.xh = p.x.hi; r.xl = p.x.lo; r.xld = p.x.ld; r.N = (int)p.x.N; r.H = (int)p.x.H; r.W = (int)p.x.W; r.Cin = (int)p.x.C;
  r.wh = p.w_hi; r.wl = p.w_lo; r.w16 = (const __half *)p.w16; r.w16_inv = p.w16_inv_scale;
  MPN_CHECK_ARG(ctx, !(p.bf16 && (p.w16 || p.x.fmt)), "conv_ref: the bf16 numerics read split-bf16 operands");
  r.xfmt = p.x.fmt; r.ofmt = p.y.fmt; r.ovf = nullptr; r.bf16 = p.bf16;
  if (p.y.fmt) MPN_TRY(mpn_ovf_flag(ctx, &r.ovf));
  r.bias = p.bias; r.Cout = p.Cout; r.kh = p.kh; r.kw = p.kw; r.stride = p.stride;
  r.pad = p.pad; r.pad_w = conv_pad_w(p); r.relu = p.relu; r.Ho = (int)p.y.H; r.Wo = (int)p.y.W;
  r.rh = p.res.hi; r.rl = p.res.lo; r.rld = p.res.ld;
  r.oh = p.y.hi; r.ol = p.y.lo; r.old_ = p.y.ld; r.of = p.y.f32; r.ofld = p.y_f32_ld;
  MPN_CHECK_ARG(ctx, !p.fp8 || (p.x8 && p.x8_exp && p.w8 && p.w8_exp && !p.w16 && !p.bf16 && !p.x.fmt),
                "conv_ref: the fp8 numerics read e4m3 planes and exponents of split-bf16 operands");
  r.x8 = p.fp8 ? p.x8 : nullptr; r.w8 = p.w8; r.x8e = p.x8_exp; r.w8e = p.w8_exp;
  const long long total = (long long)r.N * r.Ho * r.Wo * r.Cout;
  if (total <= 0) return MPN_OK;
  conv_ref_kernel<<<(unsigned)((total + 255) / 256), 256, 0, ctx->stream>>>(r);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

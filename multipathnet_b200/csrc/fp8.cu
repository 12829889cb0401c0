// fp8.cu — the operand quantizers of the opt-in fp8 inference numerics (mpn_ctx_set_option "fp8"; the rule is in
// fp8_e4m3.cuh):
//  * activations: for every slot an fp8 layer reads, once per forward pass, one e4m3 plane [pixel][C] of 2^e * hi and one
//    exponent per sample (the image in the trunk, the ROI in per-ROI layers). Two launches: per-(sample, block) maxima of
//    |hi|, then every block re-reduces its sample's maxima (a max: any order gives the same bits), derives e and
//    quantizes its share of the sample. Profile category "fp8_quantize".
//  * weights: one block per output channel: max |hi| over the channel's row, its exponent, its e4m3 row.
// A group without a valid scale (non-finite max, or beyond 448 * 2^60) raises the value 2 in the ctx's flag and is written as
// zeros; the next host-synchronous entry point fails (mpn_ovf_test).
#include "conv_gemm.cuh"
#include "fp8_e4m3.cuh"

namespace {

constexpr int QT = 256;                    // threads per quantizer block

// max of the |bf16| bit patterns of 8 packed values (for non-negative values the bit order is the value order; NaN > inf)
__device__ __forceinline__ unsigned absmax8(uint4 v) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  unsigned m = 0;
#pragma unroll
  for (int i = 0; i < 4; ++i) m = max(m, max(w[i] & 0x7fffu, (w[i] >> 16) & 0x7fffu));
  return m;
}

__device__ __forceinline__ unsigned block_max(unsigned m, unsigned *red) {
  m = __reduce_max_sync(0xffffffffu, m);
  if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
  __syncthreads();
  if (threadIdx.x < 32) {
    unsigned x = threadIdx.x < QT / 32 ? red[threadIdx.x] : 0u;
    x = __reduce_max_sync(0xffffffffu, x);
    if (threadIdx.x == 0) red[0] = x;
  }
  __syncthreads();
  return red[0];
}

// e and the multiplier of a group from its bf16 |max| bits; invalid groups: flag, multiplier 0 (all codes 0)
__device__ __forceinline__ float group_scale(unsigned mbits, int &e, unsigned *flag) {
  const float amax = __uint_as_float(mbits << 16);
  e = mpn_fp8::scale_exponent(amax);
  if (!mpn_fp8::scale_ok(amax, e)) { atomicOr(flag, 2u); return 0.f; }
  return mpn_fp8::pow2(e);
}

// 8 bf16 (packed) * sc -> 8 e4m3 codes (packed, element 0 in the low byte)
__device__ __forceinline__ uint2 quant8(uint4 v, float sc) {
  const uint32_t w[4] = {v.x, v.y, v.z, v.w};
  uint32_t o[2] = {0u, 0u};
#pragma unroll
  for (int i = 0; i < 8; ++i) {
    const uint32_t b = (i & 1) ? (w[i >> 1] & 0xffff0000u) : (w[i >> 1] << 16);
    o[i >> 2] |= (uint32_t)mpn_fp8::e4m3_rn(__uint_as_float(b) * sc) << (8 * (i & 3));
  }
  return make_uint2(o[0], o[1]);
}

struct QParams {
  const __nv_bfloat16 *hi; long long ld; int C8; long long pps;   // pps: pixels per sample
  int nb; unsigned *part;                                          // nb blocks per sample; part[sample * nb + block]
  uint8_t *q8; int *exps; unsigned *flag;
};

__global__ void __launch_bounds__(QT) fp8_amax_kernel(const QParams p) {
  MPN_PDL_SYNC();
  __shared__ unsigned red[QT / 32];
  const long long n = blockIdx.y, chunks = p.pps * p.C8;
  unsigned m = 0;
  for (long long j = (long long)blockIdx.x * QT + threadIdx.x; j < chunks; j += (long long)p.nb * QT) {
    const long long pix = n * p.pps + j / p.C8; const int c = (int)(j % p.C8) * 8;
    m = max(m, absmax8(*reinterpret_cast<const uint4 *>(p.hi + pix * p.ld + c)));
  }
  m = block_max(m, red);
  if (threadIdx.x == 0) p.part[n * p.nb + blockIdx.x] = m;
}

__global__ void __launch_bounds__(QT) fp8_quant_kernel(const QParams p) {
  MPN_PDL_SYNC();
  __shared__ unsigned red[QT / 32];
  __shared__ float s_sc;
  const long long n = blockIdx.y, chunks = p.pps * p.C8;
  unsigned m = 0;
  for (int i = threadIdx.x; i < p.nb; i += QT) m = max(m, p.part[n * p.nb + i]);
  m = block_max(m, red);
  if (threadIdx.x == 0) {
    int e;
    s_sc = group_scale(m, e, p.flag);
    if (blockIdx.x == 0) p.exps[n] = e;
  }
  __syncthreads();
  const float sc = s_sc;
  for (long long j = (long long)blockIdx.x * QT + threadIdx.x; j < chunks; j += (long long)p.nb * QT) {
    const long long pix = n * p.pps + j / p.C8; const int c = (int)(j % p.C8) * 8;
    *reinterpret_cast<uint2 *>(p.q8 + pix * (long long)p.C8 * 8 + c) = quant8(*reinterpret_cast<const uint4 *>(p.hi + pix * p.ld + c), sc);
  }
}

// one block per row (rows_pad of them: rows past `rows` only write exponent 0)
__global__ void __launch_bounds__(QT) fp8_weight_kernel(const __nv_bfloat16 *hi, long long rows, long long K, uint8_t *q8, int *exps, unsigned *flag) {
  MPN_PDL_SYNC();
  __shared__ unsigned red[QT / 32];
  __shared__ float s_sc;
  const long long r = blockIdx.x;
  if (r >= rows) { if (threadIdx.x == 0) exps[r] = 0; return; }
  const __nv_bfloat16 *row = hi + r * K;
  unsigned m = 0;
  for (long long k = threadIdx.x * 8ll; k < K; k += QT * 8ll) m = max(m, absmax8(*reinterpret_cast<const uint4 *>(row + k)));
  m = block_max(m, red);
  if (threadIdx.x == 0) { int e; s_sc = group_scale(m, e, flag); exps[r] = e; }
  __syncthreads();
  const float sc = s_sc;
  for (long long k = threadIdx.x * 8ll; k < K; k += QT * 8ll)
    *reinterpret_cast<uint2 *>(q8 + r * K + k) = quant8(*reinterpret_cast<const uint4 *>(row + k), sc);
}

}  // namespace

int mpn_fp8_quantize_launch(mpn_ctx *ctx, const DTensor &x, uint8_t *q8, int *exps) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_FP8_QUANT);
  MPN_CHECK_ARG(ctx, x.hi && x.fmt == 0 && x.C % 8 == 0 && x.ld % 8 == 0 && q8 && exps, "fp8 quantize: bf16 planes with C, ld multiples of 8");
  MPN_CHECK_ARG(ctx, x.N > 0 && x.N < 65536, "fp8 quantize: 1 <= samples < 65536");
  QParams p;
  p.hi = x.hi; p.ld = x.ld; p.C8 = (int)(x.C / 8); p.pps = x.H * x.W;
  const long long chunks = p.pps * p.C8;
  p.nb = (int)std::min<long long>(std::max<long long>((chunks + QT * 8 - 1) / (QT * 8), 1), 512);
  p.q8 = q8; p.exps = exps;
  MPN_TRY(mpn_ovf_flag(ctx, &p.flag));
  MPN_TRY(mpn_scratch4(ctx, sizeof(unsigned) * (size_t)x.N * p.nb, (void **)&p.part));
  const dim3 grid((unsigned)p.nb, (unsigned)x.N);
  MPN_CUDA(ctx, mpn_launch_pdl(ctx, fp8_amax_kernel, grid, dim3(QT), 0, p));
  MPN_LAUNCHED(ctx);
  MPN_CUDA(ctx, mpn_launch_pdl(ctx, fp8_quant_kernel, grid, dim3(QT), 0, p));
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_fp8_weight_launch(mpn_ctx *ctx, const __nv_bfloat16 *w_hi, int64_t rows, int64_t K, int64_t rows_pad, uint8_t *q8, int *exps) {
  MPN_CHECK_ARG(ctx, w_hi && q8 && exps && rows > 0 && K > 0 && K % 8 == 0 && rows_pad >= rows && rows_pad < (1ll << 31),
                "fp8 weight: bf16 rows with K a multiple of 8");
  unsigned *flag = nullptr;
  MPN_TRY(mpn_ovf_flag(ctx, &flag));
  MPN_CUDA(ctx, mpn_launch_pdl(ctx, fp8_weight_kernel, dim3((unsigned)rows_pad), dim3(QT), 0, w_hi, (long long)rows, (long long)K, q8, exps, flag));
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// Host-only view of the operand rule (no GPU), the code the quantizers run: h = n_samples x sample_elems fp32 values
// (bf16 hi-plane values in the product), per sample e = the scale exponent of max |h| and q = rn_e4m3(2^e * h).
// MPN_ERR_ARG when a sample has no valid scale.
extern "C" int mpn_debug_fp8(const float *h, int64_t n_samples, int64_t sample_elems, int32_t *e_out, uint8_t *q_out) {
  if (!h || !e_out || !q_out || n_samples <= 0 || sample_elems <= 0) return MPN_ERR_ARG;
  for (int64_t n = 0; n < n_samples; ++n) {
    const float *x = h + n * sample_elems;
    float amax = 0.f;
    for (int64_t i = 0; i < sample_elems; ++i) {
      const float a = fabsf(x[i]);
      if (amax == amax && !(a <= amax)) amax = a;   // a NaN, once taken, sticks
    }
    const int e = mpn_fp8::scale_exponent(amax);
    if (!mpn_fp8::scale_ok(amax, e)) return MPN_ERR_ARG;
    e_out[n] = e;
    const float sc = mpn_fp8::pow2(e);
    for (int64_t i = 0; i < sample_elems; ++i) q_out[n * sample_elems + i] = mpn_fp8::e4m3_rn(x[i] * sc);
  }
  return MPN_OK;
}

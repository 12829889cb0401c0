// train.cu — the kernels of the training step (mpn_model_train_step, model.cu): the two criteria, dropout and the ReLU /
// dropout gate of the backward, the transposes that make K-major split planes for the backward GEMMs, the bias column
// sums and the update under each optim method (with a no-gradient variant for the idle heads of an integral model); for a
// training trunk the max-pool backward and the tap-shifted operand of the 3x3 weight gradient. The GEMMs themselves run
// on the wgmma engine (gemm_tc.cu). The element rules live in train_rule.cuh; every reduction here runs in a fixed order, without
// floating-point atomics, so two runs give the same bits.
#include "conv_gemm.cuh"
#include <algorithm>
#include <cfloat>
#include "train_rule.cuh"

namespace {

constexpr int CRIT_THREADS = 256;
constexpr unsigned TRAIN_FLAG_LABEL = 4u;   // bit 2 of the ctx's device flag: a label outside 1..C reached the criteria

// one CTA: thread t takes rows t, t + 256, ... in order, then a fixed tree over the 256 partial sums
__global__ void __launch_bounds__(CRIT_THREADS) criteria_kernel(const float *__restrict__ x, const float *__restrict__ d,
                                                                const int32_t *__restrict__ labels, const float *__restrict__ t,
                                                                int R, int64_t R_norm, int C, float bbox_w, float *__restrict__ gx,
                                                                float *__restrict__ gd, float *__restrict__ losses, unsigned *flag) {
  __shared__ double s_ce[CRIT_THREADS], s_sl[CRIT_THREADS];
  const double inv_R = 1.0 / (double)R_norm;           // R_norm: the minibatch's rows, of which these R are a shard
  double ce = 0.0, sl = 0.0;
  for (int r = threadIdx.x; r < R; r += CRIT_THREADS) {
    const int lab = labels[r];
    float *gxr = gx + (size_t)r * C, *gdr = gd + (size_t)r * 4 * C;
    if (lab < 1 || lab > C) {                              // refused by the host entry; the device entry reports it
      atomicOr(flag, TRAIN_FLAG_LABEL);
      for (int j = 0; j < C; ++j) gxr[j] = 0.f;
      for (int j = 0; j < 4 * C; ++j) gdr[j] = 0.f;
      continue;
    }
    double a, b;
    mpn_criteria_row(x + (size_t)r * C, d + (size_t)r * 4 * C, t + (size_t)r * 4 * C, lab, C, inv_R, (double)bbox_w, gxr, gdr, &a, &b);
    ce += a; sl += b;
  }
  s_ce[threadIdx.x] = ce; s_sl[threadIdx.x] = sl;
  __syncthreads();
  for (int s = CRIT_THREADS / 2; s > 0; s >>= 1) {
    if ((int)threadIdx.x < s) { s_ce[threadIdx.x] += s_ce[threadIdx.x + s]; s_sl[threadIdx.x] += s_sl[threadIdx.x + s]; }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    const double c = s_ce[0] * inv_R, b = s_sl[0] * inv_R;
    losses[0] = (float)(c + (double)bbox_w * b); losses[1] = (float)c; losses[2] = (float)b;
  }
}

// R x 4 boxes of one image -> R x 5 ROI rows with batch index 1 (the trunk holds one image)
__global__ void rois5_kernel(const float *__restrict__ boxes, int64_t R, float *__restrict__ rois) {
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  rois[r * 5] = 1.f;
  for (int k = 0; k < 4; ++k) rois[r * 5 + 1 + k] = boxes[r * 4 + k];
}

// in place on split planes [rows][cols] (pixel stride ld): v = keep ? v * scale : 0, re-split. elem0: the Philox element
// of the first one (row0 * cols for a shard whose first row is the minibatch's row row0)
__global__ void dropout_kernel(__nv_bfloat16 *hi, __nv_bfloat16 *lo, int64_t ld, int64_t rows, int64_t cols, uint64_t seed,
                               uint32_t step, int tower, int layer, uint32_t thr, float scale, uint64_t elem0) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int64_t r = i / cols, c = i - r * cols, o = r * ld + c;
  const float v = join_bf16(hi[o], lo[o]);
  const float y = mpn_dropout_keep(seed, step, tower, layer, elem0 + (uint64_t)i, thr) ? v * scale : 0.f;
  __nv_bfloat16 h, l; split_bf16(y, h, l);
  hi[o] = h; lo[o] = l;
}

__global__ void dropout_mask_kernel(int64_t n, uint64_t seed, uint32_t step, int tower, int layer, uint32_t thr, uint64_t elem0,
                                    uint8_t *out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = (uint8_t)mpn_dropout_keep(seed, step, tower, layer, elem0 + (uint64_t)i, thr);
}

// the sum of K replicas' gradient pieces, element by element in replica order ((s0 + s1) + s2) + ..., into dst (which may
// be s0); float4 where every pointer is 16-byte aligned, the tail one element at a time
struct ReplicaSrc { const float *p[MPN_MAX_REPLICAS]; };
__global__ void __launch_bounds__(256) replica_sum_kernel(float *dst, const __grid_constant__ ReplicaSrc src, int k, int64_t n, int vec) {
  const int64_t stride = (int64_t)gridDim.x * blockDim.x;
  int64_t i0 = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const int64_t n4 = vec ? n / 4 : 0;
  for (int64_t i = i0; i < n4; i += stride) {
    float4 s = reinterpret_cast<const float4 *>(src.p[0])[i];
    for (int r = 1; r < k; ++r) {
      const float4 v = reinterpret_cast<const float4 *>(src.p[r])[i];
      s.x += v.x; s.y += v.y; s.z += v.z; s.w += v.w;
    }
    reinterpret_cast<float4 *>(dst)[i] = s;
  }
  for (int64_t i = 4 * n4 + i0; i < n; i += stride) {
    float s = src.p[0][i];
    for (int r = 1; r < k; ++r) s += src.p[r][i];
    dst[i] = s;
  }
}

// the backward gate of a stored ReLU (+ dropout) output: y > 0
__global__ void gate_mask_kernel(const __nv_bfloat16 *__restrict__ hi, const __nv_bfloat16 *__restrict__ lo, int64_t ld, int64_t rows,
                                 int64_t cols, uint8_t *__restrict__ out) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int64_t r = i / cols, c = i - r * cols;
  out[i] = join_bf16(hi[r * ld + c], lo[r * ld + c]) > 0.f ? 1 : 0;
}

// the backward through ReLU (+ dropout) of a layer whose stored output is y: G = y > 0 ? G * scale : 0, in place (y null:
// no gate); the gated G also goes to the row-major split planes A [rows][a_col0 + c] (A null: not wanted). LO false:
// the hi plane only, rn_bf16(G) (a bf16 training step: its GEMMs read no lo plane)
template <bool LO = true>
__global__ void gate_split_kernel(float *G, int64_t ldg, int64_t rows, int64_t cols, const __nv_bfloat16 *__restrict__ y_hi,
                                  const __nv_bfloat16 *__restrict__ y_lo, int64_t ldy, float scale, __nv_bfloat16 *a_hi,
                                  __nv_bfloat16 *a_lo, int64_t lda, int64_t a_col0) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * cols) return;
  const int64_t r = i / cols, c = i - r * cols;
  float g = G[r * ldg + c];
  if (y_hi) {
    g = join_bf16(y_hi[r * ldy + c], y_lo[r * ldy + c]) > 0.f ? g * scale : 0.f;
    G[r * ldg + c] = g;
  }
  if (a_hi) {
    __nv_bfloat16 h, l; split_bf16(g, h, l);
    a_hi[r * lda + a_col0 + c] = h;
    if (LO) a_lo[r * lda + a_col0 + c] = l;
  }
}

// source [rows][cols] (fp32, or split planes when src_hi is set; pixel stride lds) -> K-major split planes: element
// (r, k) goes to dst[perm(k)][dst_col0 + r] (row stride ldd). perm: 0 identity; 1 source columns in (c, p) order, p over
// the fhw pixels of a flattened map, to destination rows (p, c); 2 the reverse; 3 (c, p) to (c, fhw - 1 - p): a 3x3
// convolution's weight rotated by 180 degrees, the dgrad weight planes [Cin][ky][kx][Cout]. 32 x 32 tiles through shared memory.
// LO false: the hi plane only, rn_bf16 of an fp32 source and a copy of a split source's hi plane (its lo plane not read)
template <bool LO = true>
__global__ void transpose_split_kernel(const float *__restrict__ src, const __nv_bfloat16 *__restrict__ src_hi,
                                       const __nv_bfloat16 *__restrict__ src_lo, int64_t lds, int64_t rows, int64_t cols,
                                       int perm, int fc, int fhw, __nv_bfloat16 *__restrict__ dst_hi,
                                       __nv_bfloat16 *__restrict__ dst_lo, int64_t ldd, int64_t dst_col0) {
  __shared__ float tile[32][33];
  const int64_t r0 = (int64_t)blockIdx.y * 32, k0 = (int64_t)blockIdx.x * 32;
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int64_t r = r0 + j, k = k0 + threadIdx.x;
    float v = 0.f;
    if (r < rows && k < cols)
      v = src_hi ? (LO ? join_bf16(src_hi[r * lds + k], src_lo[r * lds + k]) : __bfloat162float(src_hi[r * lds + k])) : src[r * lds + k];
    tile[j][threadIdx.x] = v;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int64_t k = k0 + j, r = r0 + threadIdx.x;
    if (k >= cols || r >= rows) continue;
    int64_t dk = k;
    if (perm == 1) dk = (k % fhw) * fc + k / fhw;
    else if (perm == 2) dk = (k % fc) * fhw + k / fc;
    else if (perm == 3) dk = (k / fhw) * fhw + (fhw - 1 - k % fhw);
    __nv_bfloat16 h, l; split_bf16(tile[threadIdx.x][j], h, l);
    dst_hi[dk * ldd + dst_col0 + r] = h;
    if (LO) dst_lo[dk * ldd + dst_col0 + r] = l;
  }
}

// column sums of G [rows][cols]: chunk b of 256 rows -> partial[b][c] in row order, then the chunks in order
constexpr int COLSUM_ROWS = 256;
__global__ void colsum_partial_kernel(const float *__restrict__ G, int64_t ldg, int64_t rows, int64_t cols, float *__restrict__ part) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  const int64_t r0 = (int64_t)blockIdx.y * COLSUM_ROWS, r1 = min(rows, r0 + COLSUM_ROWS);
  float s = 0.f;
  for (int64_t r = r0; r < r1; ++r) s += G[r * ldg + c];
  part[(int64_t)blockIdx.y * cols + c] = s;
}
__global__ void colsum_final_kernel(const float *__restrict__ part, int nchunks, int64_t cols, float *__restrict__ out) {
  const int64_t c = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= cols) return;
  float s = 0.f;
  for (int b = 0; b < nchunks; ++b) s += part[(int64_t)b * cols + c];
  out[c] = s;
}

// HAS_G false: the update of a tensor that took no gradient this step (an idle head of an integral model: nn.SelectTable
// hands the heads it did not select a zero gradInput, and optim.sgd still steps them): g is 0 and is not read.
// M: the optim method (MPN_OPTIM_*). sgd reads lr .. first; the others read h, and buf2 (adam / adamax's second state).
constexpr bool two_states(int M) { return M == MPN_OPTIM_ADAM || M == MPN_OPTIM_ADAMAX; }
template <bool HAS_G, int M = MPN_OPTIM_SGD>
__global__ void sgd_kernel(float *__restrict__ w, const float *__restrict__ g, float *__restrict__ buf, int64_t n, float lr,
                           float momentum, float dampening, float wd, int first, float *__restrict__ buf2, mpn_optim_step h) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  float wi = w[i], bi = buf[i];
  if constexpr (M == MPN_OPTIM_SGD) {
    mpn_sgd_elem(wi, HAS_G ? g[i] : 0.f, bi, lr, momentum, dampening, wd, first);
  } else {
    float b2 = two_states(M) ? buf2[i] : 0.f;
    mpn_optim_elem<M>(wi, HAS_G ? g[i] : 0.f, bi, b2, h);
    if (two_states(M)) buf2[i] = b2;
  }
  w[i] = wi; buf[i] = bi;
}

// optim.sgd fused with the re-split of the updated weight: masters, gradient and momentum buffer are read once, and the
// split planes the forward reads ([o][(p, c)]: the engine's K order) and, when wt_hi is set, the K-major transposed planes
// the next step's dX GEMM reads ([(p, c)][wt_col0 + o], row stride ldwt) are written from the same registers. One CTA per
// UPD_ROWS output rows x cb input channels x every pixel p of a FLATTEN'd map (fhw = 1 for a 1x1 convolution or Linear):
// the Torch-layout reads w[o][c * fhw + p] are contiguous runs of cb * fhw floats, the split writes runs of cb channels,
// the transposed writes runs of UPD_ROWS rows. HAS_G false: the no-gradient update (sgd_kernel), g not read. rs (null:
// none): a factor per output row on the gradient, a^2 of a fixed-batch-norm layer (optim.sgd on W = W' / a, restated on W').
// UPDATE false: no step at all (mpn_model_train_set): w is read, buf and g are not touched, and the planes are rewritten
// from w by the same stores; hi null skips the forward's split planes (a weight no plan has prepared yet). LO false: the
// hi planes only (a bf16 training step); the forward planes' lo half is left as it is, and the next inference plan
// derives it again from the master (forget_derived_planes, model.cu). M: the optim method, as sgd_kernel; for the methods
// other than sgd, rs holds a itself and the update is mpn_optim_elem_fixed's W-space rule.
constexpr int UPD_ROWS = 16;
template <bool HAS_G, bool UPDATE = true, bool LO = true, int M = MPN_OPTIM_SGD>
__global__ void __launch_bounds__(256) sgd_split_kernel(float *__restrict__ w, const float *__restrict__ g, float *__restrict__ buf,
                                                        int cout, int fc, int fhw, int cb, float lr, float momentum, float dampening,
                                                        float wd, int first, __nv_bfloat16 *__restrict__ hi, __nv_bfloat16 *__restrict__ lo,
                                                        __nv_bfloat16 *__restrict__ wt_hi, __nv_bfloat16 *__restrict__ wt_lo, int64_t ldwt,
                                                        int64_t wt_col0, int wt_flip, const float *__restrict__ rs,
                                                        float *__restrict__ buf2, mpn_optim_step h) {
  extern __shared__ float s_w[];                       // [UPD_ROWS][cb * fhw], Torch order within a row
  const int o0 = blockIdx.y * UPD_ROWS, c0 = blockIdx.x * cb;
  const int no = min(UPD_ROWS, cout - o0), nc = min(cb, fc - c0), span = nc * fhw;
  const int64_t K = (int64_t)fc * fhw;
  for (int i = threadIdx.x; i < no * span; i += blockDim.x) {
    const int o = i / span, j = i - o * span;
    const int64_t idx = (int64_t)(o0 + o) * K + (int64_t)c0 * fhw + j;
    float wi = w[idx];
    if (UPDATE) {
      float bi = buf[idx];
      if constexpr (M == MPN_OPTIM_SGD) {
        mpn_sgd_elem(wi, HAS_G ? (rs ? rs[o0 + o] * g[idx] : g[idx]) : 0.f, bi, lr, momentum, dampening, wd, first);
      } else {
        float b2 = two_states(M) ? buf2[idx] : 0.f;
        const float gi = HAS_G ? g[idx] : 0.f;
        if (rs) mpn_optim_elem_fixed<M>(wi, gi, rs[o0 + o], bi, b2, h);
        else mpn_optim_elem<M>(wi, gi, bi, b2, h);
        if (two_states(M)) buf2[idx] = b2;
      }
      w[idx] = wi; buf[idx] = bi;
    }
    s_w[o * span + j] = wi;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < no * span && (UPDATE || hi); i += blockDim.x) {          // split planes, channel fastest
    const int o = i / span, j = i - o * span, p = j / nc, c = j - p * nc;
    __nv_bfloat16 h, l; split_bf16(s_w[o * span + c * fhw + p], h, l);
    const int64_t e = (int64_t)(o0 + o) * K + (int64_t)p * fc + c0 + c;
    hi[e] = h;
    if (LO) lo[e] = l;
  }
  if (!wt_hi) return;
  for (int i = threadIdx.x; i < no * span; i += blockDim.x) {          // transposed planes, output row fastest
    const int pc = i / no, o = i - pc * no, p = pc / nc, c = pc - p * nc;
    __nv_bfloat16 h, l; split_bf16(s_w[o * span + c * fhw + p], h, l);
    const int64_t e = (wt_flip ? ((int64_t)(c0 + c) * fhw + (fhw - 1 - p)) : ((int64_t)p * fc + c0 + c)) * ldwt + wt_col0 + o0 + o;
    wt_hi[e] = h;
    if (LO) wt_lo[e] = l;
  }
}

// the backward of a 2x2 / stride 2 / pad 0 ceil-mode max pool fused with the ReLU gate of the convolution below it and the
// split of the next dgrad's operand. y: the convolution's stored output (H x W x C split planes, pixel stride ldy); gp:
// the pool output's gradient ((H + 1) / 2 x (W + 1) / 2 x C fp32). A cell gets its window's gradient if it is the
// window's first maximum in row-major order on hi + lo (windows clipped at odd sizes), else 0; then 0 where y <= 0.
// Each cell lies in one window: a gather, no atomics. G: H x W x C fp32; a_hi / a_lo: the same as split planes (LO
// false: a_hi only). The max and the gate read y's hi + lo in either form.
template <bool LO = true>
__global__ void pool_gate_split_kernel(const float *__restrict__ gp, int H, int W, int C, const __nv_bfloat16 *__restrict__ y_hi,
                                       const __nv_bfloat16 *__restrict__ y_lo, int64_t ldy, float *__restrict__ G,
                                       __nv_bfloat16 *__restrict__ a_hi, __nv_bfloat16 *__restrict__ a_lo) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)H * W * C) return;
  const int64_t p = i / C;
  const int c = (int)(i - p * C), h = (int)(p / W), w = (int)(p - (int64_t)h * W), oh = h >> 1, ow = w >> 1;
  float m = -FLT_MAX; int64_t mi = -1;
  for (int yy = 2 * oh; yy < min(2 * oh + 2, H); ++yy)
    for (int xx = 2 * ow; xx < min(2 * ow + 2, W); ++xx) {
      const int64_t q = (int64_t)yy * W + xx;
      const float v = join_bf16(y_hi[q * ldy + c], y_lo[q * ldy + c]);
      if (v > m) { m = v; mi = q; }
    }
  const float g = (mi == p && join_bf16(y_hi[p * ldy + c], y_lo[p * ldy + c]) > 0.f) ? gp[((int64_t)oh * ((W + 1) / 2) + ow) * C + c] : 0.f;
  G[i] = g;
  __nv_bfloat16 hh, ll; split_bf16(g, hh, ll);
  a_hi[i] = hh;
  if (LO) a_lo[i] = ll;
}

// the B operand of a kh x kw / stride s / pad (ph, pw) convolution's weight gradient dW[co][ci][ky][kx] = sum_p G[p][co]
// X[tap(p)][ci] (output pixel p = (n, oh, ow) reads input cell (oh * s + ky - ph, ow * s + kx - pw) of map n, tap = ky * kw
// + kx, 0 outside the map): K-major planes B[ci * kh * kw + tap][col0 + p] from N maps X (N x H x W x Cin split planes,
// pixel stride ldx) with Ho x Wo outputs each, so that the GEMM's N order is the weight's Torch order. 32 pixels x 32 channels
// per tile through shared memory; the planes are copied, not re-split. LO false: the hi planes only (x_lo not read).
template <bool LO = true>
__global__ void tap_transpose_kernel(const __nv_bfloat16 *__restrict__ x_hi, const __nv_bfloat16 *__restrict__ x_lo, int N, int H,
                                     int W, int Cin, int64_t ldx, int kh, int kw, int s, int ph, int pw, int Ho, int Wo,
                                     __nv_bfloat16 *__restrict__ b_hi, __nv_bfloat16 *__restrict__ b_lo, int64_t ldb, int64_t col0) {
  __shared__ __nv_bfloat16 th[32][34], tl[LO ? 32 : 1][34];
  const int tap = blockIdx.z, ky = tap / kw, kx = tap % kw;
  const int64_t Po = (int64_t)Ho * Wo, P = (int64_t)N * Po, p0 = (int64_t)blockIdx.x * 32;
  const int c0 = blockIdx.y * 32;
  const __nv_bfloat16 z = __ushort_as_bfloat16((unsigned short)0);
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int64_t p = p0 + j;
    const int c = c0 + threadIdx.x;
    __nv_bfloat16 a = z, b = z;
    if (p < P && c < Cin) {
      const int64_t n = p / Po, po = p - n * Po;
      const int h = (int)(po / Wo) * s + ky - ph, w = (int)(po % Wo) * s + kx - pw;
      if (h >= 0 && h < H && w >= 0 && w < W) {
        const int64_t o = ((n * H + h) * W + w) * ldx + c;
        a = x_hi[o];
        if constexpr (LO) b = x_lo[o];
      }
    }
    th[j][threadIdx.x] = a;
    if constexpr (LO) tl[j][threadIdx.x] = b;
  }
  __syncthreads();
  for (int j = threadIdx.y; j < 32; j += blockDim.y) {
    const int c = c0 + j;
    const int64_t p = p0 + threadIdx.x;
    if (c >= Cin || p >= P) continue;
    const int64_t e = ((int64_t)c * kh * kw + tap) * ldb + col0 + p;
    b_hi[e] = th[threadIdx.x][j];
    if constexpr (LO) b_lo[e] = tl[threadIdx.x][j];
  }
}

// the dgrad of a stride-2 convolution from its column gradient: dcol [N x Ho x Wo][k * k * Cin] fp32 (column (ky * k + kx)
// * Cin + ci, the product G . W' of the dgrad GEMM) -> dx [N x H x W][Cin] += the sum over the taps that read the cell,
// in (ky, kx) order from +0 (at most 4 of them for 3x3 / pad 1, 1 for 1x1 / pad 0). A gather: no atomics.
__global__ void col2im_add_kernel(const float *__restrict__ dcol, int N, int H, int W, int Cin, int k, int s, int q, int Ho, int Wo,
                                  float *__restrict__ dx) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)N * H * W * Cin) return;
  const int64_t cell = i / Cin;
  const int ci = (int)(i - cell * Cin);
  const int64_t n = cell / ((int64_t)H * W);
  const int hw = (int)(cell - n * H * W), h = hw / W, w = hw - (hw / W) * W;
  float acc = 0.f;
  for (int ky = 0; ky < k; ++ky) {
    const int th = h + q - ky;
    if (th < 0 || th % s != 0 || th / s >= Ho) continue;
    for (int kx = 0; kx < k; ++kx) {
      const int tw = w + q - kx;
      if (tw < 0 || tw % s != 0 || tw / s >= Wo) continue;
      acc += dcol[((n * Ho + th / s) * Wo + tw / s) * ((int64_t)k * k * Cin) + (ky * k + kx) * Cin + ci];
    }
  }
  dx[i] += acc;
}

// the backward of a k x k / stride s / pad p windowed average pool (avgpool_win_kernel, elementwise.cu): each input cell
// of N maps H x W x C sums g / count over the windows that contain it, in (ky, kx) order from +0, count being the divisor
// the forward used (the window clipped to the padded map, or, exclude_pad, to the image). gp: the output's gradient, N x
// Ho x Wo rows of row stride ldgp; dx [N x H x W][C] fp32 = the sum (store) or += it. A gather: no atomics.
__global__ void avgpool_win_backward_kernel(const float *__restrict__ gp, int64_t ldgp, int N, int H, int W, int C, int k, int s, int p,
                                            int exclude_pad, int Ho, int Wo, float *__restrict__ dx, int store) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= (int64_t)N * H * W * C) return;
  const int64_t cell = i / C;
  const int c = (int)(i - cell * C);
  const int64_t n = cell / ((int64_t)H * W);
  const int hw = (int)(cell - n * H * W), h = hw / W, w = hw - (hw / W) * W;
  float acc = 0.f;
  for (int ky = 0; ky < k; ++ky) {
    const int th = h + p - ky;
    if (th < 0 || th % s != 0 || th / s >= Ho) continue;
    const int ho = th / s;
    for (int kx = 0; kx < k; ++kx) {
      const int tw = w + p - kx;
      if (tw < 0 || tw % s != 0 || tw / s >= Wo) continue;
      const int wo = tw / s;
      int h0 = ho * s - p, w0 = wo * s - p;
      int h1 = min(h0 + k, H + p), w1 = min(w0 + k, W + p);
      int count = (h1 - h0) * (w1 - w0);
      if (exclude_pad) { h0 = max(h0, 0); w0 = max(w0, 0); h1 = min(h1, H); w1 = min(w1, W); count = (h1 - h0) * (w1 - w0); }
      acc += gp[((n * Ho + ho) * Wo + wo) * ldgp + c] / (float)max(count, 1);
    }
  }
  dx[i] = store ? acc : dx[i] + acc;
}

// the backward of a global average pool: G [rows x hw][C] += gp[r][c] / hw (gp row stride ldgp: the tower's columns of
// the concat gradient)
__global__ void avgpool_backward_kernel(const float *__restrict__ gp, int64_t ldgp, int64_t rows, int hw, int C, float inv,
                                        float *__restrict__ G) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= rows * hw * C) return;
  const int64_t p = i / C, r = p / hw;
  const int c = (int)(i - p * C);
  G[i] += gp[r * ldgp + c] * inv;
}

__global__ void add_kernel(float *__restrict__ dst, const float *__restrict__ src, int64_t n) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) dst[i] += src[i];
}

__global__ void scale_kernel(float *__restrict__ x, int64_t n, float f) {
  const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) x[i] *= f;
}

unsigned nblk(int64_t n, int t) { return (unsigned)((n + t - 1) / t); }

}  // namespace

int mpn_train_criteria_launch(mpn_ctx *ctx, const float *x, const float *d, const int32_t *labels, const float *t, int R, int64_t R_norm,
                              int C, float bbox_w, float *gx, float *gd, float *losses) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  unsigned *flag = nullptr;
  MPN_TRY(mpn_ovf_flag(ctx, &flag));
  criteria_kernel<<<1, CRIT_THREADS, 0, ctx->stream>>>(x, d, labels, t, R, R_norm, C, bbox_w, gx, gd, losses, flag);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_rois5_launch(mpn_ctx *ctx, const float *boxes, int64_t R, float *rois) {
  if (R <= 0) return MPN_OK;
  rois5_kernel<<<nblk(R, 128), 128, 0, ctx->stream>>>(boxes, R, rois);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_dropout_launch(mpn_ctx *ctx, const DTensor &x, int64_t rows, int64_t cols, uint64_t seed, uint32_t step, int tower,
                             int layer, float p, uint64_t elem0) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  const int64_t n = rows * cols;
  if (n <= 0) return MPN_OK;
  dropout_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(x.hi, x.lo, x.ld, rows, cols, seed, step, tower, layer,
                                                        mpn_dropout_threshold(p), 1.f / (1.f - p), elem0);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_dropout_mask_launch(mpn_ctx *ctx, int64_t n, uint64_t seed, uint32_t step, int tower, int layer, float p, uint64_t elem0,
                                  uint8_t *out) {
  if (n <= 0) return MPN_OK;
  dropout_mask_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(n, seed, step, tower, layer, mpn_dropout_threshold(p), elem0, out);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_replica_sum_launch(mpn_ctx *ctx, float *dst, const float *const *src, int k, int64_t n) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  MPN_CHECK_ARG(ctx, k >= 1 && k <= MPN_MAX_REPLICAS, "replica sum: 1..MPN_MAX_REPLICAS sources");
  if (n <= 0) return MPN_OK;
  ReplicaSrc s{};
  bool vec = ((uintptr_t)dst & 15) == 0;
  for (int r = 0; r < k; ++r) { s.p[r] = src[r]; vec = vec && ((uintptr_t)src[r] & 15) == 0; }
  const unsigned grid = (unsigned)std::min<int64_t>(nblk(vec ? (n + 3) / 4 : n, 256), (int64_t)ctx->sm_count * 8);
  replica_sum_kernel<<<grid, 256, 0, ctx->stream>>>(dst, s, k, n, vec ? 1 : 0);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_gate_mask_launch(mpn_ctx *ctx, const DTensor &y, int64_t rows, int64_t cols, uint8_t *out) {
  if (rows * cols <= 0) return MPN_OK;
  gate_mask_kernel<<<nblk(rows * cols, 256), 256, 0, ctx->stream>>>(y.hi, y.lo, y.ld, rows, cols, out);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_gate_split_launch(mpn_ctx *ctx, float *G, int64_t ldg, int64_t rows, int64_t cols, const DTensor *y, float scale,
                                __nv_bfloat16 *a_hi, __nv_bfloat16 *a_lo, int64_t lda, int64_t a_col0) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  const int64_t n = rows * cols;
  if (n <= 0 || (!y && !a_hi)) return MPN_OK;
  if (a_hi && !a_lo)
    gate_split_kernel<false><<<nblk(n, 256), 256, 0, ctx->stream>>>(G, ldg, rows, cols, y ? y->hi : nullptr, y ? y->lo : nullptr,
                                                                    y ? y->ld : 0, scale, a_hi, nullptr, lda, a_col0);
  else
    gate_split_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(G, ldg, rows, cols, y ? y->hi : nullptr, y ? y->lo : nullptr, y ? y->ld : 0,
                                                             scale, a_hi, a_lo, lda, a_col0);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_transpose_launch(mpn_ctx *ctx, const float *src, const __nv_bfloat16 *src_hi, const __nv_bfloat16 *src_lo, int64_t lds,
                               int64_t rows, int64_t cols, int perm, int fc, int fhw, __nv_bfloat16 *dst_hi, __nv_bfloat16 *dst_lo,
                               int64_t ldd, int64_t dst_col0) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  if (rows <= 0 || cols <= 0) return MPN_OK;
  MPN_CHECK_ARG(ctx, (cols + 31) / 32 < (1ll << 31) && (rows + 31) / 32 < 65536, "transpose: matrix too large");
  dim3 grid((unsigned)((cols + 31) / 32), (unsigned)((rows + 31) / 32));
  if (!dst_lo)
    transpose_split_kernel<false><<<grid, dim3(32, 8), 0, ctx->stream>>>(src, src_hi, nullptr, lds, rows, cols, perm, fc, fhw, dst_hi,
                                                                         nullptr, ldd, dst_col0);
  else
    transpose_split_kernel<<<grid, dim3(32, 8), 0, ctx->stream>>>(src, src_hi, src_lo, lds, rows, cols, perm, fc, fhw, dst_hi, dst_lo,
                                                                  ldd, dst_col0);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_colsum_launch(mpn_ctx *ctx, const float *G, int64_t ldg, int64_t rows, int64_t cols, float *out) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  if (cols <= 0) return MPN_OK;
  const int64_t nch = (rows + COLSUM_ROWS - 1) / COLSUM_ROWS;
  MPN_CHECK_ARG(ctx, nch >= 1 && nch < 65536, "colsum: row count out of range");
  float *part = nullptr;
  MPN_TRY(mpn_scratch(ctx, sizeof(float) * (size_t)(nch * cols), (void **)&part));
  colsum_partial_kernel<<<dim3(nblk(cols, 128), (unsigned)nch), 128, 0, ctx->stream>>>(G, ldg, rows, cols, part);
  MPN_LAUNCHED(ctx);
  colsum_final_kernel<<<nblk(cols, 128), 128, 0, ctx->stream>>>(part, (int)nch, cols, out);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// M: the optim method; h its per-step scalars (mpn_optim_scalars), buf2 its second state (adam / adamax)
template <int M>
static void sgd_go(mpn_ctx *ctx, float *w, const float *g, float *buf, int64_t n, float lr, float momentum, float dampening, float wd, int first,
                   float *buf2, const mpn_optim_step &h) {
  if (g) sgd_kernel<true, M><<<nblk(n, 256), 256, 0, ctx->stream>>>(w, g, buf, n, lr, momentum, dampening, wd, first, buf2, h);
  else sgd_kernel<false, M><<<nblk(n, 256), 256, 0, ctx->stream>>>(w, nullptr, buf, n, lr, momentum, dampening, wd, first, buf2, h);
}

int mpn_train_sgd_launch(mpn_ctx *ctx, int method, float *w, const float *g, float *buf, int64_t n, float lr, float momentum, float dampening,
                         float wd, int first, float *buf2, const mpn_optim_step &h) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  if (n <= 0) return MPN_OK;
  switch (method) {
    case MPN_OPTIM_SGD: sgd_go<MPN_OPTIM_SGD>(ctx, w, g, buf, n, lr, momentum, dampening, wd, first, buf2, h); break;
    case MPN_OPTIM_ADAM: sgd_go<MPN_OPTIM_ADAM>(ctx, w, g, buf, n, lr, momentum, dampening, wd, first, buf2, h); break;
    case MPN_OPTIM_ADAMAX: sgd_go<MPN_OPTIM_ADAMAX>(ctx, w, g, buf, n, lr, momentum, dampening, wd, first, buf2, h); break;
    case MPN_OPTIM_ADAGRAD: sgd_go<MPN_OPTIM_ADAGRAD>(ctx, w, g, buf, n, lr, momentum, dampening, wd, first, buf2, h); break;
    case MPN_OPTIM_RMSPROP: sgd_go<MPN_OPTIM_RMSPROP>(ctx, w, g, buf, n, lr, momentum, dampening, wd, first, buf2, h); break;
    default: return mpn_fail(ctx, MPN_ERR_ARG, "update: optim method out of range");
  }
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// the update instantiations of method M may take more than 48 KB of dynamic shared memory
template <int M>
static int split_smem_attrs(mpn_ctx *ctx) {
  const int bytes = (int)(sizeof(float) * UPD_ROWS * 1568);
  MPN_CUDA(ctx, cudaFuncSetAttribute(sgd_split_kernel<true, true, true, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  MPN_CUDA(ctx, cudaFuncSetAttribute(sgd_split_kernel<false, true, true, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  MPN_CUDA(ctx, cudaFuncSetAttribute(sgd_split_kernel<true, true, false, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  MPN_CUDA(ctx, cudaFuncSetAttribute(sgd_split_kernel<false, true, false, M>, cudaFuncAttributeMaxDynamicSharedMemorySize, bytes));
  return MPN_OK;
}

// sgd_split_kernel's tiling of a cout x (fc * fhw) weight: cb input channels per CTA, its shared memory and grid
static int sgd_split_geometry(mpn_ctx *ctx, int cout, int fc, int fhw, int *cb, size_t *smem, dim3 *grid) {
  MPN_CHECK_ARG(ctx, cout > 0 && fc > 0 && fhw > 0 && fhw <= 1568, "sgd_split: bad weight geometry");
  *cb = std::max(1, std::min(512, 1568 / fhw));
  *smem = sizeof(float) * UPD_ROWS * *cb * fhw;
  if (*smem > 48 * 1024 && !ctx->tc_attr_set[30]) {
    MPN_TRY(split_smem_attrs<MPN_OPTIM_SGD>(ctx));
    MPN_CUDA(ctx, cudaFuncSetAttribute(sgd_split_kernel<false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(sizeof(float) * UPD_ROWS * 1568)));
    MPN_CUDA(ctx, cudaFuncSetAttribute(sgd_split_kernel<false, false, false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       (int)(sizeof(float) * UPD_ROWS * 1568)));
    MPN_TRY(split_smem_attrs<MPN_OPTIM_ADAM>(ctx));
    MPN_TRY(split_smem_attrs<MPN_OPTIM_ADAMAX>(ctx));
    MPN_TRY(split_smem_attrs<MPN_OPTIM_ADAGRAD>(ctx));
    MPN_TRY(split_smem_attrs<MPN_OPTIM_RMSPROP>(ctx));
    ctx->tc_attr_set[30] = 1;
  }
  *grid = dim3((unsigned)((fc + *cb - 1) / *cb), (unsigned)((cout + UPD_ROWS - 1) / UPD_ROWS));
  return MPN_OK;
}

// the planes an update writes, rewritten from the masters w as they stand (no step): sgd_split_kernel<false, false>.
// hi / lo null: only the W^T planes (the weight's split planes are not prepared yet). lo and wt_lo null: the hi planes
// only (a bf16 training)
int mpn_train_split_planes_launch(mpn_ctx *ctx, const float *w, int cout, int fc, int fhw, __nv_bfloat16 *hi, __nv_bfloat16 *lo,
                                  __nv_bfloat16 *wt_hi, __nv_bfloat16 *wt_lo, int64_t ldwt, int64_t wt_col0, int wt_flip) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  int cb; size_t smem; dim3 grid;
  MPN_TRY(sgd_split_geometry(ctx, cout, fc, fhw, &cb, &smem, &grid));
  if (!hi && !wt_hi) return MPN_OK;
  const mpn_optim_step h = {};
  if (!lo && !wt_lo)
    sgd_split_kernel<false, false, false><<<grid, 256, smem, ctx->stream>>>(const_cast<float *>(w), nullptr, nullptr, cout, fc, fhw, cb, 0.f,
                                                                            0.f, 0.f, 0.f, 0, hi, nullptr, wt_hi, nullptr, ldwt, wt_col0,
                                                                            wt_flip, nullptr, nullptr, h);
  else
    sgd_split_kernel<false, false><<<grid, 256, smem, ctx->stream>>>(const_cast<float *>(w), nullptr, nullptr, cout, fc, fhw, cb, 0.f, 0.f,
                                                                     0.f, 0.f, 0, hi, lo, wt_hi, wt_lo, ldwt, wt_col0, wt_flip, nullptr,
                                                                     nullptr, h);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

template <int M>
static void sgd_split_go(mpn_ctx *ctx, dim3 grid, size_t smem, int cb, float *w, const float *g, float *buf, int cout, int fc, int fhw, float lr,
                         float momentum, float dampening, float wd, int first, __nv_bfloat16 *hi, __nv_bfloat16 *lo, __nv_bfloat16 *wt_hi,
                         __nv_bfloat16 *wt_lo, int64_t ldwt, int64_t wt_col0, int wt_flip, const float *row_scale, float *buf2,
                         const mpn_optim_step &h) {
  if (!lo && !wt_lo) {
    if (g)
      sgd_split_kernel<true, true, false, M><<<grid, 256, smem, ctx->stream>>>(w, g, buf, cout, fc, fhw, cb, lr, momentum, dampening, wd, first,
                                                                               hi, nullptr, wt_hi, nullptr, ldwt, wt_col0, wt_flip, row_scale,
                                                                               buf2, h);
    else
      sgd_split_kernel<false, true, false, M><<<grid, 256, smem, ctx->stream>>>(w, nullptr, buf, cout, fc, fhw, cb, lr, momentum, dampening, wd,
                                                                                first, hi, nullptr, wt_hi, nullptr, ldwt, wt_col0, wt_flip,
                                                                                nullptr, buf2, h);
  } else if (g)
    sgd_split_kernel<true, true, true, M><<<grid, 256, smem, ctx->stream>>>(w, g, buf, cout, fc, fhw, cb, lr, momentum, dampening, wd, first, hi,
                                                                            lo, wt_hi, wt_lo, ldwt, wt_col0, wt_flip, row_scale, buf2, h);
  else
    sgd_split_kernel<false, true, true, M><<<grid, 256, smem, ctx->stream>>>(w, nullptr, buf, cout, fc, fhw, cb, lr, momentum, dampening, wd,
                                                                             first, hi, lo, wt_hi, wt_lo, ldwt, wt_col0, wt_flip, nullptr, buf2, h);
}

// g null: the no-gradient variant; lo and wt_lo null: the hi planes only (a bf16 training). row_scale: a fixed-batch-norm
// weight's a^2 per output row under sgd, a under the other methods
int mpn_train_sgd_split_launch(mpn_ctx *ctx, int method, float *w, const float *g, float *buf, int cout, int fc, int fhw, float lr, float momentum,
                               float dampening, float wd, int first, __nv_bfloat16 *hi, __nv_bfloat16 *lo, __nv_bfloat16 *wt_hi,
                               __nv_bfloat16 *wt_lo, int64_t ldwt, int64_t wt_col0, int wt_flip, const float *row_scale, float *buf2,
                               const mpn_optim_step &h) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  int cb; size_t smem; dim3 grid;
  MPN_TRY(sgd_split_geometry(ctx, cout, fc, fhw, &cb, &smem, &grid));
#define MPN_SPLIT_GO(M) sgd_split_go<M>(ctx, grid, smem, cb, w, g, buf, cout, fc, fhw, lr, momentum, dampening, wd, first, hi, lo, wt_hi, wt_lo, \
                                        ldwt, wt_col0, wt_flip, row_scale, buf2, h)
  switch (method) {
    case MPN_OPTIM_SGD: MPN_SPLIT_GO(MPN_OPTIM_SGD); break;
    case MPN_OPTIM_ADAM: MPN_SPLIT_GO(MPN_OPTIM_ADAM); break;
    case MPN_OPTIM_ADAMAX: MPN_SPLIT_GO(MPN_OPTIM_ADAMAX); break;
    case MPN_OPTIM_ADAGRAD: MPN_SPLIT_GO(MPN_OPTIM_ADAGRAD); break;
    case MPN_OPTIM_RMSPROP: MPN_SPLIT_GO(MPN_OPTIM_RMSPROP); break;
    default: return mpn_fail(ctx, MPN_ERR_ARG, "update: optim method out of range");
  }
#undef MPN_SPLIT_GO
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_pool_gate_split_launch(mpn_ctx *ctx, const float *gp, const DTensor &y, float *G, __nv_bfloat16 *a_hi, __nv_bfloat16 *a_lo) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  const int64_t n = y.H * y.W * y.C;
  if (n <= 0) return MPN_OK;
  if (!a_lo) pool_gate_split_kernel<false><<<nblk(n, 256), 256, 0, ctx->stream>>>(gp, (int)y.H, (int)y.W, (int)y.C, y.hi, y.lo, y.ld, G, a_hi, nullptr);
  else pool_gate_split_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(gp, (int)y.H, (int)y.W, (int)y.C, y.hi, y.lo, y.ld, G, a_hi, a_lo);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// x: N maps; kh x kw / stride s / pad (ph, pw) with Ho x Wo outputs per map (3x3 / 1 / 1 and Ho x Wo = H x W: the
// trunk's 3x3 layers; 1 x n / n x 1 with a pad per axis: Inception-v3's)
int mpn_train_tap_transpose_launch(mpn_ctx *ctx, const DTensor &x, int kh, int kw, int s, int ph, int pw, int64_t Ho, int64_t Wo,
                                   __nv_bfloat16 *b_hi, __nv_bfloat16 *b_lo, int64_t ldb, int64_t col0) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  const int64_t P = x.N * Ho * Wo;
  if (P <= 0) return MPN_OK;
  MPN_CHECK_ARG(ctx, (P + 31) / 32 < (1ll << 31) && (x.C + 31) / 32 < 65536 && kh >= 1 && kw >= 1 && kh * kw <= 49, "tap transpose: map too large");
  const dim3 grid((unsigned)((P + 31) / 32), (unsigned)((x.C + 31) / 32), (unsigned)(kh * kw));
  if (!b_lo)
    tap_transpose_kernel<false><<<grid, dim3(32, 8), 0, ctx->stream>>>(x.hi, nullptr, (int)x.N, (int)x.H, (int)x.W, (int)x.C, x.ld, kh, kw, s,
                                                                       ph, pw, (int)Ho, (int)Wo, b_hi, nullptr, ldb, col0);
  else
    tap_transpose_kernel<<<grid, dim3(32, 8), 0, ctx->stream>>>(x.hi, x.lo, (int)x.N, (int)x.H, (int)x.W, (int)x.C, x.ld, kh, kw, s, ph, pw,
                                                                 (int)Ho, (int)Wo, b_hi, b_lo, ldb, col0);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// x: the input geometry (N maps of H x W x Cin); dcol: N x Ho x Wo rows of k * k * Cin; dx += the gathered sums
int mpn_train_col2im_add_launch(mpn_ctx *ctx, const float *dcol, const DTensor &x, int k, int s, int q, int64_t Ho, int64_t Wo, float *dx) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  const int64_t n = x.N * x.H * x.W * x.C;
  if (n <= 0) return MPN_OK;
  col2im_add_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(dcol, (int)x.N, (int)x.H, (int)x.W, (int)x.C, k, s, q, (int)Ho, (int)Wo, dx);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// x: the pool's input geometry (N maps of H x W x C); gp: its output's gradient (Ho x Wo per map, row stride ldgp)
int mpn_train_avgpool_win_backward_launch(mpn_ctx *ctx, const float *gp, int64_t ldgp, const DTensor &x, int k, int s, int p, int exclude_pad,
                                          int64_t Ho, int64_t Wo, float *dx, int store) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  const int64_t n = x.N * x.H * x.W * x.C;
  if (n <= 0) return MPN_OK;
  avgpool_win_backward_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(gp, ldgp, (int)x.N, (int)x.H, (int)x.W, (int)x.C, k, s, p, exclude_pad,
                                                                      (int)Ho, (int)Wo, dx, store);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_avgpool_backward_launch(mpn_ctx *ctx, const float *gp, int64_t ldgp, int64_t rows, int hw, int C, float *G) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  const int64_t n = rows * hw * C;
  if (n <= 0) return MPN_OK;
  avgpool_backward_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(gp, ldgp, rows, hw, C, 1.f / (float)hw, G);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_add_launch(mpn_ctx *ctx, float *dst, const float *src, int64_t n) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  if (n <= 0) return MPN_OK;
  add_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(dst, src, n);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_train_scale_launch(mpn_ctx *ctx, float *x, int64_t n, float f) {
  if (n <= 0) return MPN_OK;
  scale_kernel<<<nblk(n, 256), 256, 0, ctx->stream>>>(x, n, f);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// out[M][N] (fp32, row stride ldo) = A[M][K] . B[N][K]^T on the wgmma engine: A and B split planes, K a multiple of 64,
// A's row stride lda and B dense. A Linear is a 1x1 convolution over M flat pixels. wide_k_split: a weight gradient over
// pixels (ConvProblem::wide_k_split). bf16: BF16X1 on the hi planes (a bf16 training step; a_lo / b_lo may be null),
// else BF16X3.
int mpn_train_gemm(mpn_ctx *ctx, const __nv_bfloat16 *a_hi, const __nv_bfloat16 *a_lo, int64_t M, int64_t K, int64_t lda,
                   const __nv_bfloat16 *b_hi, const __nv_bfloat16 *b_lo, int64_t N, float *out, int64_t ldo, int wide_k_split, int bf16) {
  // the engine reads B rows conv_k_pad(K) apart: a K off the 64 grid would need a padded B, which no caller builds
  MPN_CHECK_ARG(ctx, K % 64 == 0, "train_gemm: K must be a multiple of 64 (B is dense)");
  ConvProblem p;
  p.wide_k_split = wide_k_split;
  p.bf16 = bf16;
  p.x.hi = const_cast<__nv_bfloat16 *>(a_hi); p.x.lo = const_cast<__nv_bfloat16 *>(a_lo);
  p.x.N = M; p.x.H = 1; p.x.W = 1; p.x.C = K; p.x.ld = lda;
  p.w_hi = b_hi; p.w_lo = b_lo; p.Cout = (int)N;
  p.y.f32 = out; p.y.N = M; p.y.H = 1; p.y.W = 1; p.y.C = N; p.y.ld = ldo; p.y_f32_ld = ldo;
  ConvPlan pl;
  MPN_TRY(conv_tc_plan(ctx, p, pl));
  return conv_tc_launch(ctx, p, pl);
}

// the host view of the update kernels' element loop (mpn_debug_optim)
template <int M>
static void debug_optim(float *w, const float *g, float *s1, float *s2, const float *a, int64_t n, const mpn_optim_step &h) {
  for (int64_t i = 0; i < n; ++i) {
    float b2 = two_states(M) ? s2[i] : 0.f;
    const float gi = g ? g[i] : 0.f;
    if (a) mpn_optim_elem_fixed<M>(w[i], gi, a[i], s1[i], b2, h);
    else mpn_optim_elem<M>(w[i], gi, s1[i], b2, h);
    if (two_states(M)) s2[i] = b2;
  }
}

// ---- host-only views of the element rules (no GPU): what the CPU suite restates
extern "C" {

int mpn_debug_dropout(uint64_t seed, uint32_t step, int32_t tower, int32_t layer, uint64_t elem0, int64_t n, float p, uint8_t *out) {
  if (!out || n < 0 || !(p >= 0.f && p < 1.f) || tower < 0 || tower > 65535 || layer < 0 || layer > 65535) return MPN_ERR_ARG;
  const uint32_t thr = mpn_dropout_threshold(p);
  for (int64_t i = 0; i < n; ++i) out[i] = (uint8_t)mpn_dropout_keep(seed, step, tower, layer, elem0 + (uint64_t)i, thr);
  return MPN_OK;
}

int mpn_debug_criteria(const float *x, const float *d, const int32_t *labels, const float *t, int64_t R, int32_t C, float bbox_w,
                       float *gx, float *gd, float *losses) {
  if (!x || !d || !labels || !t || !gx || !gd || !losses || R <= 0 || C < 2) return MPN_ERR_ARG;
  for (int64_t r = 0; r < R; ++r) if (labels[r] < 1 || labels[r] > C) return MPN_ERR_ARG;
  double ce = 0.0, sl = 0.0;
  for (int64_t r = 0; r < R; ++r) {
    double a, b;
    mpn_criteria_row(x + r * C, d + r * 4 * C, t + r * 4 * C, labels[r], C, 1.0 / (double)R, (double)bbox_w, gx + r * C, gd + r * 4 * C, &a, &b);
    ce += a; sl += b;
  }
  ce *= 1.0 / (double)R; sl *= 1.0 / (double)R;
  losses[0] = (float)(ce + (double)bbox_w * sl); losses[1] = (float)ce; losses[2] = (float)sl;
  return MPN_OK;
}

int mpn_debug_sgd(float *w, const float *g, float *buf, int64_t n, float lr, float momentum, float dampening, float wd, int32_t first) {
  if (!w || !g || !buf || n < 0) return MPN_ERR_ARG;
  for (int64_t i = 0; i < n; ++i) mpn_sgd_elem(w[i], g[i], buf[i], lr, momentum, dampening, wd, first);
  return MPN_OK;
}

int mpn_debug_optim(float *w, const float *g, float *s1, float *s2, const float *a, int64_t n, const mpn_train_optim *o, float lr,
                    float momentum, float dampening, float wd, int64_t t) {
  const mpn_train_optim sgd = {MPN_OPTIM_SGD, 0.0, 0.0, 0.0, 0.0, 0.0};
  if (!o) o = &sgd;
  if (!w || !s1 || n < 0 || t < 0 || mpn_optim_refusal(*o) || (two_states(o->method) && !s2)) return MPN_ERR_ARG;
  const mpn_optim_step h = mpn_optim_scalars(*o, lr, wd, t);
  switch (o->method) {
    case MPN_OPTIM_SGD:
      for (int64_t i = 0; i < n; ++i) {
        const float gi = g ? g[i] : 0.f;
        mpn_sgd_elem(w[i], a ? (a[i] * a[i]) * gi : gi, s1[i], h.lr, momentum, dampening, wd, t == 0 ? 1 : 0);
      }
      break;
    case MPN_OPTIM_ADAM: debug_optim<MPN_OPTIM_ADAM>(w, g, s1, s2, a, n, h); break;
    case MPN_OPTIM_ADAMAX: debug_optim<MPN_OPTIM_ADAMAX>(w, g, s1, s2, a, n, h); break;
    case MPN_OPTIM_ADAGRAD: debug_optim<MPN_OPTIM_ADAGRAD>(w, g, s1, s2, a, n, h); break;
    default: debug_optim<MPN_OPTIM_RMSPROP>(w, g, s1, s2, a, n, h); break;
  }
  return MPN_OK;
}

}  // extern "C"

// post.cu — what follows NMS for one image, on the device (SURVEY 8f-2/3, 8e):
//  (1) pack_detections_kernel: utils.keep_top_k (utils.lua:75-96, Tester_FRCNN.lua:163-168) over the per-class NMS
//      keep lists of ONE image + the fixed-size detection record of the end-of-run all-gather (SURVEY 8e).
//      keep_top_k joins the kept rows of all classes, sorts the scores in descending order, takes
//      thresh = scores[min(n, top_k)] and keeps, per class and in order, every row with score >= thresh
//      (`ge`: ties at the cut all survive, so more than top_k rows can remain).
//      nms.c emits a class's kept rows in non-increasing score order (it selects the maximum of what is
//      left in every round, nms.c:74-81), so the top_k-th largest score of the union lies within the first
//      top_k rows of its own list: only min(count, MAX_DET + 1) candidates per class are looked at
//      (<= 129 x 80 keys in shared memory), a 4-pass radix select finds the threshold, and the surviving
//      prefix of every class is written at its exclusive offset: class-major, emission order inside a
//      class == the order of the reference's per-class tables after keep_top_k.
//  (2) select_boxes_kernel: nn.SelectBoxes:updateOutput (modules/SelectBoxes.lua:26-56): per row the
//      class with the maximum score (first maximum, as torch.max) and that class' 4 box values
//      (optionally * std + mean), the proposals of the next localisation iteration
//      (Tester_FRCNN.lua:82-90) without a host round trip.
#include "common.cuh"

namespace {

constexpr int PACK_THREADS = 1024;

__device__ __forceinline__ uint32_t ordered_key(float s) {     // monotone float -> uint32 (larger score, larger key)
  const uint32_t u = __float_as_uint(s);
  return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}

// one block per image. keys[(C-1) * cand] in dynamic shared memory; cand = max_det + 1.
__device__ __forceinline__ void pack_detections_body(const float *__restrict__ scores, const float *__restrict__ bboxes, int C,
                                                     const int32_t *__restrict__ keep_idx, const int32_t *__restrict__ keep_counts,
                                                     int cap, int top_k, int max_det, float *__restrict__ rec) {
  extern __shared__ uint32_t s_keys[];
  __shared__ int s_hist[256];
  __shared__ int s_cnt[1024];            // per-class surviving rows, then exclusive offsets (C - 1 <= 1024)
  __shared__ uint32_t s_prefix; __shared__ int s_want; __shared__ int s_nall; __shared__ int s_total;
  const int nseg = C - 1, cand = max_det + 1;
  const int tid = threadIdx.x;
  if (tid == 0) { s_nall = 0; s_prefix = 0; }
  for (int j = tid; j < nseg; j += PACK_THREADS) s_cnt[j] = 0;
  __syncthreads();
  // ---- candidates: first min(count, cand) rows of every class; key 0 = no row
  int n_local = 0;
  for (int i = tid; i < nseg * cand; i += PACK_THREADS) {
    const int j = i / cand, k = i - j * cand;
    uint32_t key = 0;
    if (k < keep_counts[j]) {
      const int r = keep_idx[(size_t)j * cap + k];
      key = ordered_key(scores[(size_t)r * C + j + 1]);
      if (key == 0) key = 1;             // (a NaN pattern) keep "no row" distinct
    }
    s_keys[i] = key;
  }
  for (int j = tid; j < nseg; j += PACK_THREADS) n_local += keep_counts[j];
  if (n_local) atomicAdd(&s_nall, n_local);
  __syncthreads();
  const int n_all = s_nall;
  // ---- threshold = the min(n_all, top_k)-th largest key. n_all <= top_k: the smallest score, i.e. every row survives.
  uint32_t thr_key = 1;
  if (n_all > top_k) {
    if (tid == 0) s_want = top_k;
    for (int pass = 0; pass < 4; ++pass) {
      const int shift = 24 - 8 * pass;
      if (tid < 256) s_hist[tid] = 0;
      __syncthreads();
      const uint32_t prefix = s_prefix;
      const uint32_t pmask = pass == 0 ? 0u : (0xffffffffu << (shift + 8));
      for (int i = tid; i < nseg * cand; i += PACK_THREADS) {
        const uint32_t key = s_keys[i];
        if (key != 0 && (key & pmask) == prefix) atomicAdd(&s_hist[(key >> shift) & 255], 1);
      }
      __syncthreads();
      if (tid < 32) {
        // bin holding the `want`-th largest key: suffix sums over the 256 bins, 8 bins per lane (bins 8*lane .. 8*lane+7),
        // one warp scan instead of a serial walk (a single thread walking shared memory cost ~4 us per pass)
        int c[8], own = 0;
#pragma unroll
        for (int e = 0; e < 8; ++e) { c[e] = s_hist[tid * 8 + e]; own += c[e]; }
        int suf = own;                                     // inclusive suffix sum over the lanes: keys in this lane's bins and above
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_down_sync(0xffffffffu, suf, o); if (tid + o < 32) suf += v; }
        const int above = suf - own;
        const int want = s_want;
        __syncwarp();
        if (above < want && want <= suf) {                 // exactly one lane: the wanted key is in one of its 8 bins
          int acc = above, b = tid * 8 + 7;
#pragma unroll
          for (int e = 7; e >= 0; --e) { if (acc + c[e] >= want) { b = tid * 8 + e; break; } acc += c[e]; }
          s_want = want - acc; s_prefix = prefix | ((uint32_t)b << shift);
        }
      }
      __syncthreads();
    }
    thr_key = s_prefix;
  }
  // ---- surviving rows per class (a prefix of the class list), exclusive offsets, total
  for (int i = tid; i < nseg * cand; i += PACK_THREADS) {
    const uint32_t key = s_keys[i];
    if (key != 0 && key >= thr_key) atomicAdd(&s_cnt[i / cand], 1);
  }
  __syncthreads();
  if (tid < 32) {                                          // exclusive offsets over the classes: warp scan, 32 classes per round
    int carry = 0;
    for (int j0 = 0; j0 < nseg; j0 += 32) {
      const int j = j0 + tid;
      const int c = j < nseg ? s_cnt[j] : 0;
      int inc = c;
#pragma unroll
      for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, inc, o); if (tid >= o) inc += v; }
      if (j < nseg) s_cnt[j] = carry + inc - c;
      carry += __shfl_sync(0xffffffffu, inc, 31);
    }
    if (tid == 0) s_total = carry;
  }
  __syncthreads();
  const int total = s_total;
  // count field: the number of rows keep_top_k keeps; > max_det means the record overflowed (rows beyond it are
  // dropped and the host side raises) — a class whose (max_det + 1)-th candidate still survives lands there too.
  if (tid == 0) rec[0] = (float)total;
  for (int i = tid; i < nseg * cand; i += PACK_THREADS) {
    const uint32_t key = s_keys[i];
    if (key == 0 || key < thr_key) continue;
    const int j = i / cand, k = i - j * cand;
    const int dst = s_cnt[j] + k;
    if (dst >= max_det) continue;
    const int r = keep_idx[(size_t)j * cap + k];
    const float4 b = reinterpret_cast<const float4 *>(bboxes)[(size_t)r * C + j + 1];
    float *o = rec + 1 + (size_t)dst * 6;
    o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w; o[4] = scores[(size_t)r * C + j + 1]; o[5] = (float)(j + 1);
  }
  for (int i = min(total, max_det) * 6 + tid; i < max_det * 6; i += PACK_THREADS) rec[1 + i] = 0.f;
}
__global__ void __launch_bounds__(PACK_THREADS)
pack_detections_kernel(const float *__restrict__ scores, const float *__restrict__ bboxes, int C,
                       const int32_t *__restrict__ keep_idx, const int32_t *__restrict__ keep_counts, int cap,
                       int top_k, int max_det, float *__restrict__ rec) {
  MPN_PDL_SYNC();
  pack_detections_body(scores, bboxes, C, keep_idx, keep_counts, cap, top_k, max_det, rec);
}
// the records of a batched detect, block i = image i: its rows [off[i], off[i + 1]) of scores / bboxes, its (C - 1)
// segments of keep lists (capacity cap each, rows within the image) from segment i * (C - 1) on, record i
__global__ void __launch_bounds__(PACK_THREADS)
pack_detections_batch_kernel(const float *__restrict__ scores, const float *__restrict__ bboxes, int C, ImageSegs segs,
                             const int32_t *__restrict__ keep_idx, const int32_t *__restrict__ keep_counts, int cap,
                             int top_k, int max_det, float *__restrict__ rec) {
  MPN_PDL_SYNC();
  const int i = blockIdx.x;
  const int64_t r0 = segs.off[i];
  const size_t s0 = (size_t)i * (C - 1);
  pack_detections_body(scores + r0 * C, bboxes + r0 * 4 * C, C, keep_idx + s0 * cap, keep_counts + s0, cap, top_k, max_det,
                       rec + (size_t)i * MPN_REC_FLOATS);
}

// nn.SelectBoxes: out[r] = ys[r, 4*argmax_c classes[r, c] + (0..3)] (* std + mean)
__global__ void select_boxes_kernel(const float *__restrict__ classes, const float *__restrict__ ys, int64_t R, int C,
                                    int has_norm, float4 mean, float4 stdv, float *__restrict__ out) {
  MPN_PDL_SYNC();
  const int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= R) return;
  const float *row = classes + r * C;
  float best = row[0]; int bi = 0;
  for (int c = 1; c < C; ++c) { const float v = row[c]; if (v > best) { best = v; bi = c; } }   // first maximum (torch.max)
  float4 b = reinterpret_cast<const float4 *>(ys)[r * C + bi];
  if (has_norm) {                                                          // output:cmul(sigma):add(mu)
    b.x = __fadd_rn(__fmul_rn(b.x, stdv.x), mean.x); b.y = __fadd_rn(__fmul_rn(b.y, stdv.y), mean.y);
    b.z = __fadd_rn(__fmul_rn(b.z, stdv.z), mean.z); b.w = __fadd_rn(__fmul_rn(b.w, stdv.w), mean.w);
  }
  reinterpret_cast<float4 *>(out)[r] = b;
}

}  // namespace

int mpn_pack_detections_launch(mpn_ctx *ctx, const float *scores_dev, const float *bboxes_dev, int C, const int32_t *keep_idx_dev,
                               const int32_t *keep_counts_dev, int cap, int top_k, float *rec_dev) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  MPN_CHECK_ARG(ctx, C >= 2 && C - 1 <= 1024, "pack_detections: 1..1024 foreground classes");
  MPN_CHECK_ARG(ctx, top_k >= 1 && top_k <= MPN_MAX_DET, "pack_detections: top_k must be in 1..MPN_MAX_DET");
  const size_t smem = sizeof(uint32_t) * (size_t)(C - 1) * (MPN_MAX_DET + 1);
  MPN_CHECK_ARG(ctx, smem <= 200 * 1024, "pack_detections: too many classes for the candidate table");
  if (smem > 48 * 1024 && !ctx->tc_attr_set[16]) {
    MPN_CUDA(ctx, cudaFuncSetAttribute(pack_detections_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    ctx->tc_attr_set[16] = 1;
  }
  MPN_CUDA(ctx, mpn_launch_pdl(ctx, pack_detections_kernel, dim3(1), dim3(PACK_THREADS), smem, scores_dev, bboxes_dev, C, keep_idx_dev,
                               keep_counts_dev, cap, top_k, (int)MPN_MAX_DET, rec_dev));
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_pack_detections_batch_launch(mpn_ctx *ctx, const float *scores_dev, const float *bboxes_dev, int C, const ImageSegs &segs,
                                     const int32_t *keep_idx_dev, const int32_t *keep_counts_dev, int cap, int top_k, float *rec_dev) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  MPN_CHECK_ARG(ctx, C >= 2 && C - 1 <= 1024, "pack_detections: 1..1024 foreground classes");
  MPN_CHECK_ARG(ctx, top_k >= 1 && top_k <= MPN_MAX_DET, "pack_detections: top_k must be in 1..MPN_MAX_DET");
  if (segs.n <= 0) return MPN_OK;
  const size_t smem = sizeof(uint32_t) * (size_t)(C - 1) * (MPN_MAX_DET + 1);
  MPN_CHECK_ARG(ctx, smem <= 200 * 1024, "pack_detections: too many classes for the candidate table");
  if (smem > 48 * 1024 && !ctx->tc_attr_set[24]) {
    MPN_CUDA(ctx, cudaFuncSetAttribute(pack_detections_batch_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 200 * 1024));
    ctx->tc_attr_set[24] = 1;
  }
  MPN_CUDA(ctx, mpn_launch_pdl(ctx, pack_detections_batch_kernel, dim3(segs.n), dim3(PACK_THREADS), smem, scores_dev, bboxes_dev, C, segs,
                               keep_idx_dev, keep_counts_dev, cap, top_k, (int)MPN_MAX_DET, rec_dev));
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_select_boxes_launch(mpn_ctx *ctx, const float *classes_dev, const float *ys_dev, int64_t R, int C, const float *mean4,
                            const float *std4, float *out_dev) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_ELTWISE);
  if (R <= 0) return MPN_OK;
  const int has = (mean4 && std4) ? 1 : 0;
  const float4 mu = has ? make_float4(mean4[0], mean4[1], mean4[2], mean4[3]) : make_float4(0.f, 0.f, 0.f, 0.f);
  const float4 sd = has ? make_float4(std4[0], std4[1], std4[2], std4[3]) : make_float4(1.f, 1.f, 1.f, 1.f);
  MPN_CUDA(ctx, mpn_launch_pdl(ctx, select_boxes_kernel, dim3((unsigned)((R + 127) / 128)), dim3(128), 0, classes_dev, ys_dev, R, C, has, mu,
                               sd, out_dev));
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

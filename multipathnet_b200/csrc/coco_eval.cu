// coco_eval.cu — COCOeval (iouType 'bbox', default Params) on the device: testCoco.evaluate's score
// (testCoco/coco.lua:24-38, testCoco/init.lua:30-88). The rules restated from pycocotools are listed in DESIGN §4.
//
// Compiled with -fmad=false: the IoU, the thresholds and precision / recall must keep pycocotools' unfused double op order.
//
// Pipeline (all on the ctx stream, deterministic: no floating-point atomics):
//   coco_rows_kernel     validate rows, map ids, keys: score (descending), pair = category * n_images + image rank
//   radix sort 1         stable LSD over (pair, score desc) -> per-pair order; coco_rank_kernel ranks dets within a pair
//   radix sort (GT)      stable over pair -> annotations of a pair contiguous, in input order
//   compaction           stable partition of pair starts (one radix pass on a 0/1 key)
//   coco_match_kernel    one CTA per non-empty pair, one thread per (area range, IoU threshold) greedy walk
//   radix sort 2         of sort 1's order by (category, score desc): ties keep (image rank, rank in pair)
//   coco_accumulate_kernel  one CTA per (category, area range, maxDets, threshold): scans, envelope, recall thresholds
//   coco_stats_kernel    the 12 summary means
#include <cmath>
#include "common.cuh"

namespace {

constexpr int kT = 10, kR = 101, kA = 4, kM = 3, kW = kT * kA;   // thresholds, recall points, area ranges, maxDets, walks
constexpr int kMaxDet = 100;
__device__ __constant__ double kAreaLo[kA] = {0.0, 0.0, 1024.0, 9216.0};
__device__ __constant__ double kAreaHi[kA] = {1e10, 1024.0, 9216.0, 1e10};
__device__ __constant__ int kMaxDets[kM] = {1, 10, 100};

// np.linspace(start, stop, num): i * ((stop - start) / (num - 1)) + start, the last element = stop
__device__ __forceinline__ double iou_thr(int t) { return t == kT - 1 ? 0.95 : (double)t * ((0.95 - 0.5) / (kT - 1)) + 0.5; }
__device__ __forceinline__ double rec_thr(int r) { return r == kR - 1 ? 1.0 : (double)r * (1.0 / (kR - 1)) + 0.0; }

// maskApi.c bbIou, one pair: d = {x, y, w, h, w*h} of the float32 detection promoted to double, g = {x, y, w, h}
__device__ __forceinline__ double bb_iou(const double *d, const double *g, int crowd) {
  const double w = fmin(d[2] + d[0], g[2] + g[0]) - fmax(d[0], g[0]);
  if (w <= 0) return 0.0;
  const double h = fmin(d[3] + d[1], g[3] + g[1]) - fmax(d[1], g[1]);
  if (h <= 0) return 0.0;
  const double i = w * h, ga = g[2] * g[3];
  const double u = crowd ? d[4] : d[4] + ga - i;
  return i / u;
}

// score -> key whose ascending order is descending score; -0 and +0 tie, as numpy's comparisons do
__device__ __forceinline__ uint32_t desc_score_key(float s) {
  if (s == 0.f) s = 0.f;
  const uint32_t u = __float_as_uint(s);
  const uint32_t asc = (u & 0x80000000u) ? ~u : (u | 0x80000000u);
  return ~asc;
}

template <class T>
__device__ __forceinline__ int64_t lower_bound_dev(const T *a, int64_t n, T v) {
  int64_t lo = 0, hi = n;
  while (lo < hi) { const int64_t mid = (lo + hi) >> 1; if (a[mid] < v) lo = mid + 1; else hi = mid; }
  return lo;
}

// ---------------------------------------------------------------------------------------------- stable LSD radix sort
// Sorts a sequence of element indices by key[element], 4 bits per pass. Per pass: per-tile digit histogram,
// one-CTA exclusive scan in digit-major order, stable scatter (items in sequence order within a thread, threads in order).
constexpr int kRT = 256, kRI = 16, kRTile = kRT * kRI;

__global__ void __launch_bounds__(kRT) radix_hist_kernel(const int32_t *seq, const uint32_t *key, int n, int shift, int *hist, int nb) {
  __shared__ int c[16];
  if (threadIdx.x < 16) c[threadIdx.x] = 0;
  __syncthreads();
  const int base = blockIdx.x * kRTile;
  for (int j = threadIdx.x; j < kRTile; j += kRT) {
    const int i = base + j;
    if (i < n) atomicAdd(&c[(key[seq[i]] >> shift) & 15u], 1);
  }
  __syncthreads();
  if (threadIdx.x < 16) hist[threadIdx.x * nb + blockIdx.x] = c[threadIdx.x];
}

// in-place exclusive scan of a[0, m); a[m] = the total
__global__ void __launch_bounds__(1024) scan_exclusive_kernel(int *a, int m) {
  __shared__ int ws[32];
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
  int carry = 0;
  for (int base = 0; base < m; base += 1024) {
    const int i = base + threadIdx.x;
    const int v = i < m ? a[i] : 0;
    int x = v;
    for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(~0u, x, o); if (lane >= o) x += y; }
    if (lane == 31) ws[warp] = x;
    __syncthreads();
    if (warp == 0) {
      int w = ws[lane];
      for (int o = 1; o < 32; o <<= 1) { const int y = __shfl_up_sync(~0u, w, o); if (lane >= o) w += y; }
      ws[lane] = w;
    }
    __syncthreads();
    x += warp ? ws[warp - 1] : 0;
    if (i < m) a[i] = carry + x - v;
    carry += ws[31];
    __syncthreads();
  }
  if (threadIdx.x == 0) a[m] = carry;
}

__global__ void __launch_bounds__(kRT) radix_scatter_kernel(const int32_t *seq, const uint32_t *key, int n, int shift, const int *hist, int nb,
                                                            int32_t *out) {
  __shared__ int s[16 * kRT];
  __shared__ int o[16 * kRT];
  __shared__ int ws[kRT / 32];
  const int t = threadIdx.x, lane = t & 31, warp = t >> 5;
  const int base = blockIdx.x * kRTile + t * kRI;
  int el[kRI], dg[kRI];
  uint64_t c_lo = 0, c_hi = 0;                                // 16 digit counters of 8 bits
#pragma unroll
  for (int j = 0; j < kRI; ++j) {
    const int i = base + j;
    el[j] = 0; dg[j] = 16;
    if (i < n) { el[j] = seq[i]; dg[j] = (key[el[j]] >> shift) & 15u; }
    if (dg[j] < 8) c_lo += 1ull << (8 * dg[j]);
    else if (dg[j] < 16) c_hi += 1ull << (8 * (dg[j] - 8));
  }
#pragma unroll
  for (int d = 0; d < 16; ++d) s[d * kRT + t] = (int)(((d < 8 ? c_lo : c_hi) >> (8 * (d & 7))) & 0xff);
  __syncthreads();
  // exclusive scan of s in digit-major order: thread t owns entries [16 t, 16 t + 16)
  int loc[16], sum = 0;
#pragma unroll
  for (int j = 0; j < 16; ++j) { loc[j] = sum; sum += s[t * 16 + j]; }
  int x = sum;
  for (int of = 1; of < 32; of <<= 1) { const int y = __shfl_up_sync(~0u, x, of); if (lane >= of) x += y; }
  if (lane == 31) ws[warp] = x;
  __syncthreads();
  int pre = x - sum;
  for (int w = 0; w < warp; ++w) pre += ws[w];
  __syncthreads();
#pragma unroll
  for (int j = 0; j < 16; ++j) s[t * 16 + j] = pre + loc[j];
  __syncthreads();
#pragma unroll
  for (int d = 0; d < 16; ++d) o[d * kRT + t] = hist[d * nb + blockIdx.x] + s[d * kRT + t] - s[d * kRT];
#pragma unroll
  for (int j = 0; j < kRI; ++j)
    if (dg[j] < 16) out[o[dg[j] * kRT + t]++] = el[j];
}

__global__ void iota_kernel(int32_t *a, int n) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = i;
}

struct RadixBufs { int32_t *tmp; int *hist; };

// stable sort of seq[0, n) by the low `bits` bits of key[element]; the result is left in seq
int radix_sort(mpn_ctx *ctx, const uint32_t *key, int bits, int32_t *seq, int n, const RadixBufs &rb) {
  if (n <= 0) return MPN_OK;
  const int nb = (n + kRTile - 1) / kRTile;
  int32_t *a = seq, *b = rb.tmp;
  for (int shift = 0; shift < bits; shift += 4) {
    radix_hist_kernel<<<nb, kRT, 0, ctx->stream>>>(a, key, n, shift, rb.hist, nb);
    MPN_LAUNCHED(ctx);
    scan_exclusive_kernel<<<1, 1024, 0, ctx->stream>>>(rb.hist, 16 * nb);
    MPN_LAUNCHED(ctx);
    radix_scatter_kernel<<<nb, kRT, 0, ctx->stream>>>(a, key, n, shift, rb.hist, nb, b);
    MPN_LAUNCHED(ctx);
    std::swap(a, b);
  }
  if (a != seq) MPN_CUDA(ctx, cudaMemcpyAsync(seq, a, sizeof(int32_t) * (size_t)n, cudaMemcpyDeviceToDevice, ctx->stream));
  return MPN_OK;
}

int bits_for(uint64_t max_value) {   // bits to hold 0..max_value, rounded up to a whole number of 4-bit passes
  int b = 0;
  while (b < 32 && (max_value >> b)) ++b;
  return (b + 3) & ~3;
}

// ---------------------------------------------------------------------------------------------- rows and ranks
enum { ERR_NONFINITE = 1, ERR_IMAGE = 2 };

__global__ void coco_rows_kernel(const float *dets, int D, const int64_t *img_tab, int NI, const int64_t *cat_tab, int NC,
                                 uint32_t *skey, uint32_t *pkey, int *present, unsigned *err) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D) return;
  const float *r = dets + 7 * (size_t)i;
  const uint32_t sentinel = (uint32_t)NC * (uint32_t)NI;
  skey[i] = 0; pkey[i] = sentinel;
  bool fin = true;
#pragma unroll
  for (int c = 0; c < 7; ++c) fin = fin && isfinite(r[c]);
  if (!fin) { atomicOr(err, (unsigned)ERR_NONFINITE); return; }
  const int64_t iid = (int64_t)r[0];                         // int() of the float32 value: truncation
  const int64_t ii = lower_bound_dev(img_tab, NI, iid);
  if (ii == NI || img_tab[ii] != iid) { atomicOr(err, (unsigned)ERR_IMAGE); return; }
  present[ii] = 1;
  const int64_t cid = (int64_t)r[6];
  const int64_t ci = lower_bound_dev(cat_tab, NC, cid);
  if (ci < NC && cat_tab[ci] == cid) pkey[i] = (uint32_t)ci * (uint32_t)NI + (uint32_t)ii;
  skey[i] = desc_score_key(r[5]);
}

__global__ void gather_keys_kernel(const int32_t *perm, const uint32_t *key, int n, uint32_t *out) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) out[i] = key[perm[i]];
}

// spk = pair keys in sort-1 order. rank = position within the pair (capped at kMaxDet); start flag 0 at the first detection of a
// scored pair; key2 = category for the detections the evaluation keeps (rank < 100), n_cats for the others
__global__ void coco_rank_kernel(const int32_t *perm1, const uint32_t *spk, int D, int NI, int NC, int *rank_row, uint32_t *start_flag,
                                 uint32_t *key2) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= D) return;
  const uint32_t p = spk[i], sentinel = (uint32_t)NC * (uint32_t)NI;
  int lo = i - kMaxDet > 0 ? i - kMaxDet : 0, hi = i;         // first j in [lo, i] with spk[j] == p
  while (lo < hi) { const int mid = (lo + hi) >> 1; if (spk[mid] < p) lo = mid + 1; else hi = mid; }
  const int rank = i - lo;                                    // == kMaxDet when the pair started earlier still
  const int row = perm1[i];
  const bool valid = p != sentinel;
  rank_row[row] = rank;
  start_flag[i] = (valid && rank == 0) ? 0u : 1u;
  key2[row] = (valid && rank < kMaxDet) ? p / (uint32_t)NI : (uint32_t)NC;
}

__global__ void coco_gt_keys_kernel(const int32_t *gt_img, const int32_t *gt_cat, int G, int NI, uint32_t *gkey) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j < G) gkey[j] = (uint32_t)gt_cat[j] * (uint32_t)NI + (uint32_t)gt_img[j];
}

__global__ void coco_gt_gather_kernel(const int32_t *gperm, const uint32_t *gkey, const double *box, const double *area, const int32_t *crowd,
                                      const int32_t *img, int G, uint32_t *sgk, double *sbox, double *sarea, int32_t *scrowd, int32_t *simg) {
  const int j = blockIdx.x * blockDim.x + threadIdx.x;
  if (j >= G) return;
  const int s = gperm[j];
  sgk[j] = gkey[s];
  for (int c = 0; c < 4; ++c) sbox[4 * (size_t)j + c] = box[4 * (size_t)s + c];
  sarea[j] = area[s]; scrowd[j] = crowd[s]; simg[j] = img[s];
}

// ---------------------------------------------------------------------------------------------- matching
constexpr int kMT = 64;            // two warps: walks 0..31 and 32..39
constexpr int kIouCap = 4096;      // IoU block in shared memory up to nd * ng entries; larger pairs compute IoUs in the walk

// masks[4 * row + {0, 1}]: matched bits of walks 0..31 / 32..39, [4 * row + {2, 3}]: ignored bits; walk w = area * 10 + threshold.
// gtm: one byte per (walk, annotation), owned by the walk's thread while its pair is processed.
__global__ void __launch_bounds__(kMT) coco_match_kernel(const int32_t *starts, const int *n_pairs_p, const int32_t *perm1, const uint32_t *spk,
                                                         int D, const float *dets, const uint32_t *sgk, const double *sbox, const double *sarea,
                                                         const int32_t *scrowd, int G, uint8_t *gtm, uint32_t *masks) {
  __shared__ double s_iou[kIouCap];
  __shared__ double s_d[kMaxDet][5];
  __shared__ float s_fa[kMaxDet];
  __shared__ int s_row[kMaxDet];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int w = tid, a = w / kT, t = w % kT;
  const bool active = w < kW;
  const double thr = active ? fmin(iou_thr(t), 1 - 1e-10) : 0.0;
  const double alo = active ? kAreaLo[a] : 0.0, ahi = active ? kAreaHi[a] : 0.0;
  const int np = *n_pairs_p;
  for (int p = blockIdx.x; p < np; p += gridDim.x) {
    const int s = starts[p];
    const uint32_t key = spk[s];
    int lo = s, hi = s + kMaxDet < D ? s + kMaxDet : D;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (spk[mid] == key) lo = mid + 1; else hi = mid; }
    const int nd = lo - s;
    const int g0 = (int)lower_bound_dev(sgk, G, key);
    const int ng = (int)lower_bound_dev(sgk, G, key + 1) - g0;
    for (int d = tid; d < nd; d += kMT) {
      const int row = perm1[s + d];
      const float *r = dets + 7 * (size_t)row;
      s_row[d] = row;
      s_d[d][0] = r[1]; s_d[d][1] = r[2]; s_d[d][2] = r[3]; s_d[d][3] = r[4];
      s_d[d][4] = (double)r[3] * (double)r[4];
      s_fa[d] = __fmul_rn(r[3], r[4]);                        // loadRes: area = bb[2] * bb[3] of float32 scalars
    }
    __syncthreads();
    const bool blk = nd * ng <= kIouCap;
    if (blk)
      for (int q = tid; q < nd * ng; q += kMT) {
        const int d = q / ng, g = q - d * ng;
        s_iou[q] = bb_iou(s_d[d], sbox + 4 * (size_t)(g0 + g), scrowd[g0 + g]);
      }
    uint8_t *my = gtm + (size_t)(active ? w : 0) * G + g0;
    if (active)
      for (int g = 0; g < ng; ++g) my[g] = 0;
    __syncthreads();
    for (int d = 0; d < nd; ++d) {
      bool matched = false, ign = false;
      if (active) {
        double best = thr;
        int m = -1;
        bool m_ig = false;
        // annotations stably reordered non-ignored first; a match among the non-ignored ends the walk before the ignored ones
        for (int pass = 0; pass < 2 && !(pass == 1 && m >= 0); ++pass) {
          for (int g = 0; g < ng; ++g) {
            const int cr = scrowd[g0 + g];
            const double ga = sarea[g0 + g];
            const bool gi = cr || ga < alo || ga > ahi;
            if ((int)gi != pass) continue;
            if (my[g] && !cr) continue;
            const double v = blk ? s_iou[d * ng + g] : bb_iou(s_d[d], sbox + 4 * (size_t)(g0 + g), cr);
            if (v < best) continue;
            best = v; m = g; m_ig = gi;
          }
        }
        if (m >= 0) { my[m] = 1; matched = true; ign = m_ig; }
        else { const double da = s_fa[d]; ign = da < alo || da > ahi; }
      }
      const unsigned bm = __ballot_sync(~0u, matched), bi = __ballot_sync(~0u, ign);
      if (lane == 0) { masks[4 * (size_t)s_row[d] + warp] = bm; masks[4 * (size_t)s_row[d] + 2 + warp] = bi; }
    }
    __syncthreads();
  }
}

// ---------------------------------------------------------------------------------------------- accumulate
constexpr int kAT = 256;

template <class T, class Op>
__device__ __forceinline__ T block_scan_incl(T v, int idx, T *sh, Op op) {   // inclusive scan in the order of idx (a permutation of 0..255)
  sh[idx] = v;
  __syncthreads();
  for (int off = 1; off < kAT; off <<= 1) {
    const T o = idx >= off ? sh[idx - off] : v;
    __syncthreads();
    if (idx >= off) v = op(o, v);
    sh[idx] = v;
    __syncthreads();
  }
  return v;
}

__global__ void __launch_bounds__(kAT) coco_accumulate_kernel(const int32_t *perm2, const uint32_t *key2, int D, const int *rank_row,
                                                              const uint32_t *masks, const uint32_t *sgk, const double *sarea,
                                                              const int32_t *scrowd, const int32_t *simg, const int *present, int G, int NI,
                                                              int NC, double *precision, double *recall) {
  __shared__ uint32_t sh_u[kAT];
  __shared__ double sh_d[kAT];
  __shared__ int Tr[kR];
  const int k = blockIdx.x, a = blockIdx.y / kM, m = blockIdx.y % kM, t = blockIdx.z, tid = threadIdx.x;
  const int w = a * kT + t, maxdet = kMaxDets[m];
  const double alo = kAreaLo[a], ahi = kAreaHi[a];
  const size_t pidx = (size_t)k * (kA * kM) + a * kM + m;     // [.][.][k][a][m]
  auto sum_u = [](uint32_t x, uint32_t y) { return x + y; };
  // npig: non-ignored annotations of category k on the evaluated images
  const int g0 = (int)lower_bound_dev(sgk, G, (uint32_t)k * (uint32_t)NI), g1 = (int)lower_bound_dev(sgk, G, (uint32_t)(k + 1) * (uint32_t)NI);
  uint32_t cnt = 0;
  for (int j = g0 + tid; j < g1; j += kAT)
    if (present[simg[j]] && !scrowd[j] && !(sarea[j] < alo || sarea[j] > ahi)) ++cnt;
  block_scan_incl(cnt, tid, sh_u, sum_u);
  const uint32_t npig_all = sh_u[kAT - 1];
  __syncthreads();
  if (npig_all == 0) return;                                  // precision / recall stay -1
  const double dn = (double)npig_all;
  if (tid < kR) {                                             // the least tp count whose recall reaches rec_thr(r)
    const double thr = rec_thr(tid);
    int lo = 0, hi = (int)npig_all;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if ((double)mid / dn >= thr) hi = mid; else lo = mid + 1; }
    Tr[tid] = lo;
  }
  // this category's kept detections in sort-2 order
  int c0, c1;
  {
    int lo = 0, hi = D;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (key2[perm2[mid]] < (uint32_t)k) lo = mid + 1; else hi = mid; }
    c0 = lo; hi = D;
    while (lo < hi) { const int mid = (lo + hi) >> 1; if (key2[perm2[mid]] < (uint32_t)k + 1) lo = mid + 1; else hi = mid; }
    c1 = lo;
  }
  const int wq = w >> 5, wb = w & 31;
  auto flags = [&](int i, bool &inc, uint32_t &tpf, uint32_t &fpf) {
    inc = false; tpf = fpf = 0;
    if (i >= c1) return;
    const int row = perm2[i];
    if (rank_row[row] >= maxdet) return;
    inc = true;
    const bool mt = (masks[4 * (size_t)row + wq] >> wb) & 1u, ig = (masks[4 * (size_t)row + 2 + wq] >> wb) & 1u;
    if (!ig) { tpf = mt; fpf = !mt; }
  };
  // totals: tp | fp << 10 | included << 20 per chunk of 256 positions
  uint32_t tp_tot = 0, fp_tot = 0, nd = 0;
  for (int base = c0; base < c1; base += kAT) {
    bool inc; uint32_t tpf, fpf;
    flags(base + tid, inc, tpf, fpf);
    block_scan_incl(tpf | (fpf << 10) | ((uint32_t)inc << 20), tid, sh_u, sum_u);
    const uint32_t tot = sh_u[kAT - 1];
    __syncthreads();
    tp_tot += tot & 0x3ff; fp_tot += (tot >> 10) & 0x3ff; nd += tot >> 20;
  }
  if (tid == 0) recall[(size_t)t * NC * (kA * kM) + pidx] = nd ? (double)tp_tot / dn : 0.0;
  __syncthreads();
  // backwards over the positions: tp / fp counts from the totals, precision, its running maximum from the end (the envelope)
  uint32_t carry_tp = tp_tot, carry_fp = fp_tot;
  double carry_max = -1.0;
  const int rev = kAT - 1 - tid;
  const int nchunks = (c1 - c0 + kAT - 1) / kAT;
  for (int ch = nchunks - 1; ch >= 0; --ch) {
    const int i = c0 + ch * kAT + tid;
    bool inc; uint32_t tpf, fpf;
    flags(i, inc, tpf, fpf);
    const uint32_t suf = block_scan_incl(tpf | (fpf << 16), rev, sh_u, sum_u);   // over positions >= i within the chunk
    const uint32_t chunk = sh_u[kAT - 1];
    __syncthreads();
    const uint32_t tp_i = carry_tp - ((suf & 0xffff) - tpf), fp_i = carry_fp - ((suf >> 16) - fpf);
    const double pr = inc ? (double)tp_i / (((double)fp_i + (double)tp_i) + 2.220446049250313e-16) : -1.0;
    const double env = fmax(block_scan_incl(pr, rev, sh_d, [](double x, double y) { return fmax(x, y); }), carry_max);
    const double chunk_max = sh_d[kAT - 1];
    __syncthreads();
    if (inc && tpf) {                                         // the tp_i-th true positive: q[r] for every r with Tr[r] == tp_i
      int r = 0, hi = kR;
      while (r < hi) { const int mid = (r + hi) >> 1; if (Tr[mid] < (int)tp_i) r = mid + 1; else hi = mid; }
      for (; r < kR && Tr[r] == (int)tp_i; ++r) precision[((size_t)t * kR + r) * NC * (kA * kM) + pidx] = env;
    }
    carry_tp -= chunk & 0xffff; carry_fp -= chunk >> 16;
    carry_max = fmax(carry_max, chunk_max);
  }
  if (tid < kR) {
    double q = -2.0;
    if (Tr[tid] == 0) q = nd ? carry_max : 0.0;               // searchsorted lands on the first position
    else if (Tr[tid] > (int)tp_tot) q = 0.0;                  // recall never reaches the threshold
    if (q > -2.0) precision[((size_t)t * kR + tid) * NC * (kA * kM) + pidx] = q;
  }
}

__global__ void fill_kernel(double *a, size_t n, double v) {
  const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (i < n) a[i] = v;
}

// COCOeval.summarize's 12 entries, one CTA each: mean of the selected entries > -1, or -1. Each thread sums a fixed strided share
// of the (t, r, k) entries, then a fixed-order tree adds the shares: the same bits on every call.
constexpr int kST = 256;
__global__ void __launch_bounds__(kST) coco_stats_kernel(const double *precision, const double *recall, int NC, double *stats) {
  __shared__ double sh_s[kST];
  __shared__ int64_t sh_n[kST];
  const int s = blockIdx.x, tid = threadIdx.x;
  const bool ap = s < 6;
  const double thr_sel = (s == 1) ? 0.5 : (s == 2) ? 0.75 : -1.0;
  const int a = (s == 3 || s == 9) ? 1 : (s == 4 || s == 10) ? 2 : (s == 5 || s == 11) ? 3 : 0;
  const int m = (s == 6) ? 0 : (s == 7) ? 1 : 2;
  const int per_t = (ap ? kR : 1) * NC;                       // entries (r, k) of one threshold
  double sum = 0.0;
  int64_t n = 0;
  for (int64_t e = tid; e < (int64_t)kT * per_t; e += kST) {
    const int t = (int)(e / per_t), rk = (int)(e % per_t);
    if (thr_sel >= 0 && iou_thr(t) != thr_sel) continue;
    const int r = rk / NC, k = rk % NC;
    const size_t pidx = (size_t)k * (kA * kM) + a * kM + m;
    const double v = ap ? precision[((size_t)t * kR + r) * NC * (kA * kM) + pidx] : recall[(size_t)t * NC * (kA * kM) + pidx];
    if (v > -1) { sum += v; ++n; }
  }
  sh_s[tid] = sum; sh_n[tid] = n;
  __syncthreads();
  for (int h = kST / 2; h > 0; h >>= 1) {
    if (tid < h) { sh_s[tid] += sh_s[tid + h]; sh_n[tid] += sh_n[tid + h]; }
    __syncthreads();
  }
  if (tid == 0) stats[s] = sh_n[0] ? sh_s[0] / (double)sh_n[0] : -1.0;
}

inline unsigned grid1(int64_t n, int b = 256) { return (unsigned)((n + b - 1) / b); }

}  // namespace

int mpn_scan_exclusive_launch(mpn_ctx *ctx, int *a, int m) {       // also the training feed's list offsets (roidb.cu)
  scan_exclusive_kernel<<<1, 1024, 0, ctx->stream>>>(a, m);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

extern "C" int mpn_coco_eval(mpn_ctx *ctx, int32_t n_images, const int64_t *image_ids, int32_t n_cats, const int64_t *cat_ids, int64_t G,
                             const int32_t *gt_img, const int32_t *gt_cat, const double *gt_box, const double *gt_area, const int32_t *gt_crowd,
                             int64_t D, const float *dets, double *precision, double *recall, double *stats) {
  if (!ctx) return MPN_ERR_ARG;
  MPN_CUDA(ctx, cudaSetDevice(ctx->device));
  MPN_CHECK_ARG(ctx, n_images >= 1 && n_cats >= 1 && image_ids && cat_ids, "mpn_coco_eval: the image and category id tables must not be empty");
  MPN_CHECK_ARG(ctx, D >= 1 && dets, "mpn_coco_eval: no detection rows (pycocotools' loadRes fails on an empty result)");
  MPN_CHECK_ARG(ctx, precision && recall && stats, "mpn_coco_eval: output buffers missing");
  MPN_CHECK_ARG(ctx, G >= 0 && (G == 0 || (gt_img && gt_cat && gt_box && gt_area && gt_crowd)), "mpn_coco_eval: ground-truth buffers missing");
  MPN_CHECK_ARG(ctx, D < (1 << 30) && G < (1 << 30), "mpn_coco_eval: more than 2^30 detection rows or annotations");
  MPN_CHECK_ARG(ctx, ((uint64_t)n_cats + 1) * (uint64_t)n_images < (1ull << 32), "mpn_coco_eval: (n_cats + 1) * n_images must be < 2^32");
  for (int32_t i = 1; i < n_images; ++i)
    MPN_CHECK_ARG(ctx, image_ids[i] > image_ids[i - 1], "mpn_coco_eval: image ids must be ascending and unique");
  for (int32_t i = 1; i < n_cats; ++i)
    MPN_CHECK_ARG(ctx, cat_ids[i] > cat_ids[i - 1], "mpn_coco_eval: category ids must be ascending and unique");
  for (int64_t j = 0; j < G; ++j) {
    if (gt_img[j] < 0 || gt_img[j] >= n_images || gt_cat[j] < 0 || gt_cat[j] >= n_cats)
      return mpn_fail(ctx, MPN_ERR_ARG, "mpn_coco_eval: annotation " + std::to_string(j) + " has an image or category index out of range");
    if (gt_crowd[j] != 0 && gt_crowd[j] != 1)
      return mpn_fail(ctx, MPN_ERR_ARG, "mpn_coco_eval: annotation " + std::to_string(j) + " has iscrowd not in {0, 1}");
    bool fin = std::isfinite(gt_area[j]);
    for (int c = 0; c < 4; ++c) fin = fin && std::isfinite(gt_box[4 * j + c]);
    if (!fin) return mpn_fail(ctx, MPN_ERR_ARG, "mpn_coco_eval: annotation " + std::to_string(j) + " has a non-finite bbox or area");
  }
  const int NI = n_images, NC = n_cats, nD = (int)D, nG = (int)G;
  const int nmax = nD > nG ? nD : nG;
  const int nb = (nmax + kRTile - 1) / kRTile;
  const size_t n_prec = (size_t)kT * kR * NC * kA * kM, n_rec = (size_t)kT * NC * kA * kM;
  const int G1 = nG > 0 ? nG : 1;

  // one scratch allocation, 256-byte aligned pieces
  size_t off = 0;
  auto take = [&](size_t bytes) { const size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  const size_t o_dets = take(sizeof(float) * 7 * nD), o_img = take(sizeof(int64_t) * NI), o_cat = take(sizeof(int64_t) * NC);
  const size_t o_gimg = take(4 * (size_t)G1), o_gcat = take(4 * (size_t)G1), o_gcr = take(4 * (size_t)G1), o_gbox = take(32 * (size_t)G1),
               o_garea = take(8 * (size_t)G1);
  const size_t o_present = take(4 * (size_t)NI), o_err = take(16);
  const size_t o_skey = take(4 * (size_t)nD), o_pkey = take(4 * (size_t)nD), o_key2 = take(4 * (size_t)nD), o_rank = take(4 * (size_t)nD);
  const size_t o_perm1 = take(4 * (size_t)nD), o_perm2 = take(4 * (size_t)nD), o_starts = take(4 * (size_t)nD), o_spk = take(4 * (size_t)nD),
               o_flag = take(4 * (size_t)nD), o_tmp = take(4 * (size_t)nmax), o_hist = take(4 * ((size_t)16 * nb + 1)), o_npairs = take(4);
  const size_t o_gkey = take(4 * (size_t)G1), o_gperm = take(4 * (size_t)G1), o_sgk = take(4 * (size_t)G1), o_sbox = take(32 * (size_t)G1),
               o_sarea = take(8 * (size_t)G1), o_scr = take(4 * (size_t)G1), o_simg = take(4 * (size_t)G1), o_gtm = take((size_t)kW * G1);
  const size_t o_masks = take(16 * (size_t)nD), o_prec = take(8 * n_prec), o_rec = take(8 * n_rec), o_stats = take(8 * 12);
  void *base_v;
  MPN_TRY(mpn_scratch(ctx, off, &base_v));
  char *base = (char *)base_v;
  auto P = [&](size_t o) { return (void *)(base + o); };
  float *d_dets = (float *)P(o_dets);
  int64_t *d_img = (int64_t *)P(o_img), *d_cat = (int64_t *)P(o_cat);
  int32_t *d_gimg = (int32_t *)P(o_gimg), *d_gcat = (int32_t *)P(o_gcat), *d_gcr = (int32_t *)P(o_gcr);
  double *d_gbox = (double *)P(o_gbox), *d_garea = (double *)P(o_garea);
  int *d_present = (int *)P(o_present);
  unsigned *d_err = (unsigned *)P(o_err);
  uint32_t *d_skey = (uint32_t *)P(o_skey), *d_pkey = (uint32_t *)P(o_pkey), *d_key2 = (uint32_t *)P(o_key2);
  int *d_rank = (int *)P(o_rank);
  int32_t *d_perm1 = (int32_t *)P(o_perm1), *d_perm2 = (int32_t *)P(o_perm2), *d_starts = (int32_t *)P(o_starts);
  uint32_t *d_spk = (uint32_t *)P(o_spk), *d_flag = (uint32_t *)P(o_flag);
  const RadixBufs rb{(int32_t *)P(o_tmp), (int *)P(o_hist)};
  int *d_npairs = (int *)P(o_npairs);
  uint32_t *d_gkey = (uint32_t *)P(o_gkey), *d_sgk = (uint32_t *)P(o_sgk);
  int32_t *d_gperm = (int32_t *)P(o_gperm), *d_scr = (int32_t *)P(o_scr), *d_simg = (int32_t *)P(o_simg);
  double *d_sbox = (double *)P(o_sbox), *d_sarea = (double *)P(o_sarea);
  uint8_t *d_gtm = (uint8_t *)P(o_gtm);
  uint32_t *d_masks = (uint32_t *)P(o_masks);
  double *d_prec = (double *)P(o_prec), *d_rec = (double *)P(o_rec), *d_stats = (double *)P(o_stats);
  cudaStream_t st = ctx->stream;

  MPN_CUDA(ctx, cudaMemcpyAsync(d_dets, dets, sizeof(float) * 7 * (size_t)nD, cudaMemcpyHostToDevice, st));
  MPN_CUDA(ctx, cudaMemcpyAsync(d_img, image_ids, sizeof(int64_t) * NI, cudaMemcpyHostToDevice, st));
  MPN_CUDA(ctx, cudaMemcpyAsync(d_cat, cat_ids, sizeof(int64_t) * NC, cudaMemcpyHostToDevice, st));
  if (nG > 0) {
    MPN_CUDA(ctx, cudaMemcpyAsync(d_gimg, gt_img, 4 * (size_t)nG, cudaMemcpyHostToDevice, st));
    MPN_CUDA(ctx, cudaMemcpyAsync(d_gcat, gt_cat, 4 * (size_t)nG, cudaMemcpyHostToDevice, st));
    MPN_CUDA(ctx, cudaMemcpyAsync(d_gcr, gt_crowd, 4 * (size_t)nG, cudaMemcpyHostToDevice, st));
    MPN_CUDA(ctx, cudaMemcpyAsync(d_gbox, gt_box, 32 * (size_t)nG, cudaMemcpyHostToDevice, st));
    MPN_CUDA(ctx, cudaMemcpyAsync(d_garea, gt_area, 8 * (size_t)nG, cudaMemcpyHostToDevice, st));
  }
  MPN_CUDA(ctx, cudaMemsetAsync(d_present, 0, 4 * (size_t)NI, st));
  MPN_CUDA(ctx, cudaMemsetAsync(d_err, 0, sizeof(unsigned), st));

  // rows: validation and keys; the one host round trip of the call reports bad rows
  coco_rows_kernel<<<grid1(nD), 256, 0, st>>>(d_dets, nD, d_img, NI, d_cat, NC, d_skey, d_pkey, d_present, d_err);
  MPN_LAUNCHED(ctx);
  unsigned err = 0;
  MPN_CUDA(ctx, cudaMemcpyAsync(&err, d_err, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
  MPN_CUDA(ctx, cudaStreamSynchronize(st));
  if (err & ERR_NONFINITE) return mpn_fail(ctx, MPN_ERR_ARG, "mpn_coco_eval: a detection row holds a NaN or infinite value");
  if (err & ERR_IMAGE)
    return mpn_fail(ctx, MPN_ERR_ARG, "mpn_coco_eval: a detection row's image id is not a ground-truth image (pycocotools' loadRes asserts this)");

  const int pbits = bits_for((uint64_t)NC * (uint64_t)NI);
  // sort 1: (pair, score descending, row)
  iota_kernel<<<grid1(nD), 256, 0, st>>>(d_perm1, nD);
  MPN_LAUNCHED(ctx);
  MPN_TRY(radix_sort(ctx, d_skey, 32, d_perm1, nD, rb));
  MPN_TRY(radix_sort(ctx, d_pkey, pbits, d_perm1, nD, rb));
  gather_keys_kernel<<<grid1(nD), 256, 0, st>>>(d_perm1, d_pkey, nD, d_spk);
  MPN_LAUNCHED(ctx);
  coco_rank_kernel<<<grid1(nD), 256, 0, st>>>(d_perm1, d_spk, nD, NI, NC, d_rank, d_flag, d_key2);
  MPN_LAUNCHED(ctx);
  // pair starts, in order: a stable partition on the start flag; their count is the total of digit 0
  iota_kernel<<<grid1(nD), 256, 0, st>>>(d_starts, nD);
  MPN_LAUNCHED(ctx);
  MPN_TRY(radix_sort(ctx, d_flag, 4, d_starts, nD, rb));
  MPN_CUDA(ctx, cudaMemcpyAsync(d_npairs, rb.hist + (nD + kRTile - 1) / kRTile, sizeof(int), cudaMemcpyDeviceToDevice, st));
  // annotations grouped by pair, input order kept
  if (nG > 0) {
    coco_gt_keys_kernel<<<grid1(nG), 256, 0, st>>>(d_gimg, d_gcat, nG, NI, d_gkey);
    MPN_LAUNCHED(ctx);
    iota_kernel<<<grid1(nG), 256, 0, st>>>(d_gperm, nG);
    MPN_LAUNCHED(ctx);
    MPN_TRY(radix_sort(ctx, d_gkey, pbits, d_gperm, nG, rb));
    coco_gt_gather_kernel<<<grid1(nG), 256, 0, st>>>(d_gperm, d_gkey, d_gbox, d_garea, d_gcr, d_gimg, nG, d_sgk, d_sbox, d_sarea, d_scr, d_simg);
    MPN_LAUNCHED(ctx);
  }
  coco_match_kernel<<<ctx->sm_count * 8, kMT, 0, st>>>(d_starts, d_npairs, d_perm1, d_spk, nD, d_dets, d_sgk, d_sbox, d_sarea, d_scr, nG, d_gtm,
                                                      d_masks);
  MPN_LAUNCHED(ctx);
  // sort 2: sort 1's order by (category, score descending); unscored detections last
  MPN_CUDA(ctx, cudaMemcpyAsync(d_perm2, d_perm1, 4 * (size_t)nD, cudaMemcpyDeviceToDevice, st));
  MPN_TRY(radix_sort(ctx, d_skey, 32, d_perm2, nD, rb));
  MPN_TRY(radix_sort(ctx, d_key2, bits_for((uint64_t)NC), d_perm2, nD, rb));
  fill_kernel<<<grid1((int64_t)n_prec), 256, 0, st>>>(d_prec, n_prec, -1.0);
  MPN_LAUNCHED(ctx);
  fill_kernel<<<grid1((int64_t)n_rec), 256, 0, st>>>(d_rec, n_rec, -1.0);
  MPN_LAUNCHED(ctx);
  coco_accumulate_kernel<<<dim3(NC, kA * kM, kT), kAT, 0, st>>>(d_perm2, d_key2, nD, d_rank, d_masks, d_sgk, d_sarea, d_scr, d_simg, d_present,
                                                               nG, NI, NC, d_prec, d_rec);
  MPN_LAUNCHED(ctx);
  coco_stats_kernel<<<12, kST, 0, st>>>(d_prec, d_rec, NC, d_stats);
  MPN_LAUNCHED(ctx);
  MPN_CUDA(ctx, cudaMemcpyAsync(precision, d_prec, 8 * n_prec, cudaMemcpyDeviceToHost, st));
  MPN_CUDA(ctx, cudaMemcpyAsync(recall, d_rec, 8 * n_rec, cudaMemcpyDeviceToHost, st));
  MPN_CUDA(ctx, cudaMemcpyAsync(stats, d_stats, 8 * 12, cudaMemcpyDeviceToHost, st));
  MPN_CUDA(ctx, cudaStreamSynchronize(st));
  return MPN_OK;
}

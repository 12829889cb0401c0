// nms.cu — batched greedy NMS on sm_90a, bit-exact against the reference nms.c.
//
// Replaces utils.nms -> nms.c:NMS (reference nms.c:59-108, utils.lua:29-33), which the
// reference calls once per class per image on the CPU (Tester_FRCNN.lua:106-117).
// Here all classes (segments) of an image go through one launch set:
//   1. nms_rank_kernel   : stable descending rank of every row by counting (exact,
//                          ties broken by ascending row => detects ties as a by-product)
//   2. nms_mask_kernel   : 64x64 tiles of the upper-triangular IoU>thr bitmask, IoU in
//                          the exact fp32 op order of nms.c:14-41 (no FMA: __f*_rn)
//   3. nms_scan_kernel   : per segment, 64-row chunks: serial resolve of the diagonal
//                          word + parallel OR of the kept rows into the removed-bitset
//   4. nms_exact_kernel  : ONLY for segments that contain tied scores: block-parallel
//                          emulation of nms.c's pointer-permutation walk (first strict max
//                          in the current order, swap-to-front, order-preserving survivor
//                          compaction), because nms.c's tie order is an artefact of that
//                          permutation and not of any sort order.
// With distinct scores nms.c keeps rows in descending-score order, which is what 1-3 emit.
// Layout: segments have uniform capacity `cap`; segment s owns rows [s*cap, s*cap+count[s]).
#include "common.cuh"

namespace {

// nms.c:14-41 op for op. a = the selected ("best") box, b = the other (argument order of nms.c:92).
__device__ __forceinline__ float iou_ref(float ax1, float ay1, float ax2, float ay2,
                                         float bx1, float by1, float bx2, float by2) {
  float x1 = (ax1 > bx1) ? ax1 : bx1;   // MAX macro: (a>b)?a:b
  float y1 = (ay1 > by1) ? ay1 : by1;
  float x2 = (ax2 < bx2) ? ax2 : bx2;   // MIN macro: (a<b)?a:b
  float y2 = (ay2 < by2) ? ay2 : by2;
  float w = __fadd_rn(__fsub_rn(x2, x1), 1.0f);
  float h = __fadd_rn(__fsub_rn(y2, y1), 1.0f);
  float inter = __fmul_rn(w, h);
  float aarea = __fmul_rn(__fadd_rn(__fsub_rn(ax2, ax1), 1.0f), __fadd_rn(__fsub_rn(ay2, ay1), 1.0f));
  float barea = __fmul_rn(__fadd_rn(__fsub_rn(bx2, bx1), 1.0f), __fadd_rn(__fsub_rn(by2, by1), 1.0f));
  float iou = __fdiv_rn(inter, __fsub_rn(__fadd_rn(aarea, barea), inter));
  return (w <= 0.0f || h <= 0.0f) ? 0.0f : iou;
}

constexpr int RANK_THREADS = 256;
constexpr int RANK_ELEMS = 64;            // rows ranked per block; 4 threads per row, each scanning a quarter of every tile

// grid (ceil(cap/64), nseg). rank[i] = #{j: s_j > s_i or (s_j == s_i and j < i)}.
__global__ void __launch_bounds__(RANK_THREADS)
nms_rank_kernel(const float *__restrict__ sb, int cap, const int32_t *__restrict__ counts,
                int32_t *__restrict__ order, float4 *__restrict__ sorted_boxes,
                int32_t *__restrict__ tie_flag, float *__restrict__ sorted_score) {
  MPN_PDL_SYNC();
  const int seg = blockIdx.y;
  const int n = counts ? counts[seg] : cap;
  if ((int)blockIdx.x * RANK_ELEMS >= n) return;
  const float *seg_sb = sb + (size_t)seg * cap * 5;
  constexpr int TILE = 1024;
  __shared__ float s_tile[TILE];
  __shared__ int s_rank[RANK_ELEMS], s_tied[RANK_ELEMS];
  const int el = threadIdx.x & (RANK_ELEMS - 1), part = threadIdx.x / RANK_ELEMS;
  const int i = blockIdx.x * RANK_ELEMS + el;
  const bool valid = i < n;
  const float si = valid ? seg_sb[(size_t)i * 5 + 4] : 0.0f;
  if (threadIdx.x < RANK_ELEMS) { s_rank[threadIdx.x] = 0; s_tied[threadIdx.x] = 0; }
  int rank = 0; int tied = 0;
  for (int base = 0; base < n; base += TILE) {
    for (int t = threadIdx.x; t < TILE; t += RANK_THREADS) {
      const int j = base + t;
      s_tile[t] = (j < n) ? seg_sb[(size_t)j * 5 + 4] : 0.0f;
    }
    __syncthreads();
    const int t0 = part * (TILE / 4), lim = min(TILE / 4, n - base - t0);
    if (valid) {
#pragma unroll 8
      for (int t = 0; t < lim; ++t) {
        const float sj = s_tile[t0 + t];
        const int jj = base + t0 + t;
        const bool eq = (sj == si);
        rank += (sj > si) || (eq && jj < i);
        tied |= (eq && jj != i);
      }
    }
    __syncthreads();
  }
  if (valid) { atomicAdd(&s_rank[el], rank); if (tied) atomicOr(&s_tied[el], 1); }
  __syncthreads();
  if (valid && part == 0) {
    const int r = s_rank[el];
    order[(size_t)seg * cap + r] = i;
    const float *b = seg_sb + (size_t)i * 5;
    sorted_boxes[(size_t)seg * cap + r] = make_float4(b[0], b[1], b[2], b[3]);
    if (sorted_score) sorted_score[(size_t)seg * cap + r] = si;
    if (s_tied[el]) atomicOr(&tie_flag[seg], 1);
  }
}

// grid (nwords, nwords, nseg), 64 threads. Block (cb, rb): rows rb*64.., cols cb*64..; only cb >= rb.
// mask[seg][row][cb] bit c set iff col j=cb*64+c > row i and !(iou(i,j) <= thr)  (nms.c:93 keeps <=).
__global__ void __launch_bounds__(64)
nms_mask_kernel(const float4 *__restrict__ sorted_boxes, int cap, int nwords_cap,
                const int32_t *__restrict__ counts, const int32_t *__restrict__ tie_flag, int skip_tied,
                float thr, unsigned long long *__restrict__ mask) {
  MPN_PDL_SYNC();
  // grid.x enumerates the nb*(nb+1)/2 tiles of the upper triangle: tile t -> (rb, cb >= rb)
  const int seg = blockIdx.z;
  int rb = 0, cb = (int)blockIdx.x;
  for (int rowlen = nwords_cap; cb >= rowlen; cb -= rowlen, --rowlen) ++rb;
  cb += rb;
  if (skip_tied && tie_flag[seg]) return;       // large-N path: nms_exact_kernel handles tied segments
  const int n = counts ? counts[seg] : cap;
  if (rb * 64 >= n || cb * 64 >= n) return;
  const float4 *boxes = sorted_boxes + (size_t)seg * cap;
  __shared__ float4 s_col[64];
  const int t = threadIdx.x;
  const int cj = cb * 64 + t;
  s_col[t] = (cj < n) ? boxes[cj] : make_float4(0, 0, 0, 0);
  __syncthreads();
  const int i = rb * 64 + t;
  if (i >= n) return;
  const float4 a = boxes[i];
  unsigned long long bits = 0ull;
  const int ncols = min(64, n - cb * 64);
  const int start = (rb == cb) ? t + 1 : 0;
  for (int c = start; c < ncols; ++c) {
    float4 b = s_col[c];
    float v = iou_ref(a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w);
    if (!(v <= thr)) bits |= (1ull << c);
  }
  if (rb == cb) bits |= 1ull << t;              // a selected box also removes itself (saves the special case in the walk)
  mask[((size_t)seg * cap + i) * nwords_cap + cb] = bits;
}

constexpr int SCAN_THREADS = 256;

// one block per segment. keep_idx[seg*cap + k] = original row (via order, then src_idx if given).
__global__ void __launch_bounds__(SCAN_THREADS)
nms_scan_kernel(const unsigned long long *__restrict__ mask, const int32_t *__restrict__ order,
                int cap, int nwords_cap, const int32_t *__restrict__ counts,
                const int32_t *__restrict__ tie_flag, const int32_t *__restrict__ src_idx,
                int32_t *__restrict__ keep_idx, int32_t *__restrict__ keep_counts) {
  const int seg = blockIdx.x;
  if (tie_flag[seg]) return;
  const int n = counts ? counts[seg] : cap;
  extern __shared__ unsigned long long s_removed[];   // nwords_cap words
  __shared__ unsigned long long s_diag[64];
  __shared__ unsigned long long s_keepbits;
  const int nwords = (n + 63) / 64;
  const unsigned long long *m = mask + (size_t)seg * cap * nwords_cap;
  const int32_t *ord = order + (size_t)seg * cap;
  for (int w = threadIdx.x; w < nwords; w += SCAN_THREADS) s_removed[w] = 0ull;
  int nkeep = 0;
  __syncthreads();
  for (int c = 0; c < nwords; ++c) {
    const int row0 = c * 64;
    if (threadIdx.x < 64) {
      int r = row0 + threadIdx.x;
      s_diag[threadIdx.x] = (r < n) ? m[(size_t)r * nwords_cap + c] : 0ull;
    }
    __syncthreads();
    if (threadIdx.x == 0) {
      unsigned long long cur = s_removed[c], kb = 0ull;
      const int lim = min(64, n - row0);
      for (int b = 0; b < lim; ++b) {
        if (!((cur >> b) & 1ull)) { kb |= (1ull << b); cur |= s_diag[b]; }
      }
      s_keepbits = kb;
    }
    __syncthreads();
    const unsigned long long kb = s_keepbits;
    if (threadIdx.x < 64 && ((kb >> threadIdx.x) & 1ull)) {
      int pos = nkeep + __popcll(kb & ((1ull << threadIdx.x) - 1ull));
      int o = ord[row0 + threadIdx.x];
      keep_idx[(size_t)seg * cap + pos] = src_idx ? src_idx[(size_t)seg * cap + o] : o;
    }
    nkeep += __popcll(kb);
    // OR the rows of the kept boxes of this chunk into the words after c
    for (int w = c + 1 + threadIdx.x; w < nwords; w += SCAN_THREADS) {
      unsigned long long acc = s_removed[w], bits = kb;
      while (bits) {
        int b = __ffsll((long long)bits) - 1;
        bits &= bits - 1ull;
        acc |= m[(size_t)(row0 + b) * nwords_cap + w];
      }
      s_removed[w] = acc;
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) keep_counts[seg] = nkeep;
}

// ---- segments up to 4096 boxes: ONE warp walks the greedy selection round by round, the removed-bitset lives in
// registers (2 x 64 bits per lane), the suppression mask in shared memory when it fits (n <= 1024) else in L2.
// No block barrier sits on the serial chain (~100-150 cycles per kept box with the smem mask).
//
// Tied scores are resolved exactly like nms.c WITHOUT re-running its O(N) pointer walk per round:
//   nms.c's array order only ever changes by "the element in the first live slot moves into the slot of the
//   selected box" (the swap at nms.c:83-86; the survivor compaction at :90-99 is order preserving). So each element
//   carries a slot label (initially its row index), the head is the live occupant of the smallest live slot (a
//   monotone pointer finds it), and "first strict maximum in current order" (nms.c:74-81) = among the live boxes
//   sharing the top score, the one with the smallest label.
//   The label bookkeeping is LAZY: the walk records every selection and each box's death round; only when a round
//   actually has two live boxes with the top score is the slot history replayed up to that round (by one lane,
//   no warp collectives), and the tie broken by label. Segments whose ties never meet pay (almost) nothing.
__device__ int g_nms_trace = 0;      // MPN_NMS_TRACE=1: block 0 of the warp kernel prints its phase times (tools/nms_diag.py)
constexpr int WARP_CAP = 4096;
constexpr int WARP_SMEM_MASK_CAP = 1024;
constexpr int WARPK_THREADS = 256;

struct WalkCtx {
  const unsigned long long *s_mask, *m, *s_tn; unsigned long long *s_diag; const float *s_score; int *s_label, *s_owner; unsigned long long *s_rrem;
  unsigned short *s_keep, *s_death, *s_qalt;
  int n, nwords, nwords_cap, use_smem_mask;
};

// The serial walk, one warp. TIE: the segment has equal scores. TWO: more than 32 mask words (n > 2048) -> two
// removed-words per lane. A single warp cannot hide instruction latency, so every instruction on this chain costs
// ~5 cycles: the common path is kept to a few dozen instructions per kept box, and the slot-label bookkeeping that
// nms.c's tie order needs is LAZY: only when a round really has two live boxes with the top score does `replay`
// re-walk the recorded selections [replayed, nkeep) (liveness re-derived from the same mask rows) while tracking the
// head moves, after which the tie is broken by slot label. Segments whose ties never meet pay one shuffle per round.
template <bool TIE, bool TWO, bool SMEM>
__device__ __forceinline__ int nms_walk(const WalkCtx &c, const int lane) {
  const int n = c.n, nwords = c.nwords;
  auto init_word = [&](int w) -> unsigned long long {
    if (w >= nwords) return ~0ull;
    return (w == nwords - 1 && (n & 63)) ? (~0ull << (n & 63)) : 0ull;
  };
  auto mask_word = [&](int row, int w) -> unsigned long long {
    return SMEM ? c.s_mask[row * nwords + w] : __ldg(c.m + (size_t)row * c.nwords_cap + w);
  };
  unsigned long long rem0 = init_word(lane), rem1 = TWO ? init_word(lane + 32) : ~0ull;
  // tienext bit p: score[p] == score[p+1] in sorted order (ballots of the whole block, see the kernel prologue)
  const unsigned long long tn0 = TIE ? c.s_tn[lane] : 0ull, tn1 = (TIE && TWO) ? c.s_tn[lane + 32] : 0ull;
  unsigned long long rr0 = rem0, rr1 = rem1;       // replay state: removed-set at round `replayed`
  int nkeep = 0, hp = 0, replayed = 0;
  while (true) {
    // ---- first 64-row chunk (mask word cw) that still has a live box in (score desc, row asc) order
    unsigned ball = __ballot_sync(0xffffffffu, rem0 != ~0ull);
    int half = 0;
    if (!ball) {
      if (!TWO) break;
      ball = __ballot_sync(0xffffffffu, rem1 != ~0ull); half = 1;
      if (!ball) break;
    }
    const int wl = __ffs(ball) - 1;
    const int cw = wl + (TWO ? 32 * half : 0);
    const int row0 = cw * 64;
    unsigned long long cur = __shfl_sync(0xffffffffu, (TWO && half) ? rem1 : rem0, wl);
    const unsigned long long tw = TIE ? __shfl_sync(0xffffffffu, (TWO && half) ? tn1 : tn0, wl) : 0ull;
    // ---- resolve the chunk: every lane runs the same scalar loop over the LIVE rows only (typically 5-15 of 64): next
    //      live bit, its diagonal word (one broadcast load) clears what it suppresses inside the chunk; in the same
    //      iteration, off the serial chain, each lane ORs its own later word of that row into its removed-set and lane 0
    //      records the row. A single warp pays ~5-10 cycles per dependent instruction, so the chain is ffs -> address ->
    //      load -> and. A live box whose score continues into the next row (tie) stops the loop: general round below.
    int tie_b = -1;
    {
      // lanes that own no later word read the diagonal word instead and discard it: no divergent branch in the loop
      const bool on0 = (lane > cw) && (lane < nwords);
      const bool on1 = TWO && (lane + 32 > cw) && (lane + 32 < nwords);
      const int w0 = on0 ? lane : cw, w1 = on1 ? lane + 32 : cw;
      const unsigned long long k0 = on0 ? ~0ull : 0ull, k1 = on1 ? ~0ull : 0ull;
      unsigned long long acc0 = 0ull, acc1 = 0ull;
      unsigned lo = ~(unsigned)cur, hi = ~(unsigned)(cur >> 32);       // live rows of the chunk, as two 32-bit halves
      const unsigned tlo = (unsigned)tw, thi = (unsigned)(tw >> 32);
      // one iteration = one kept row `b` (bit index inside the chunk)
      // mask in L2 (n > 1024): the chunk's 64 diagonal words are prefetched into shared memory with one round trip, the
      // kept rows are only recorded in the loop, and their later words are OR-ed in afterwards with eight loads in flight
      unsigned kb_lo = 0u, kb_hi = 0u;
      if (!SMEM) {
        c.s_diag[lane] = __ldg(c.m + (size_t)min(row0 + lane, n - 1) * c.nwords_cap + cw);
        c.s_diag[lane + 32] = __ldg(c.m + (size_t)min(row0 + 32 + lane, n - 1) * c.nwords_cap + cw);
        __syncwarp();
      }
#define MPN_NMS_KEEP_ROW(b)                                                         \
      {                                                                            \
        const int row = row0 + (b);                                                \
        const unsigned long long d = SMEM ? mask_word(row, cw) : c.s_diag[(b)];    \
        if (SMEM) {                                                                \
          acc0 |= mask_word(row, w0) & k0;                                         \
          if (TWO) acc1 |= mask_word(row, w1) & k1;                                \
        } else {                                                                   \
          if ((b) < 32) kb_lo |= 1u << ((b) & 31); else kb_hi |= 1u << ((b) & 31); \
        }                                                                          \
        c.s_keep[nkeep] = (unsigned short)row;   /* every lane, same value */      \
        ++nkeep;                                                                   \
        lo &= ~(unsigned)d; hi &= ~(unsigned)(d >> 32);                            \
      }
      while (lo) {
        const int b = __ffs(lo) - 1;
        if (TIE && ((tlo >> b) & 1u)) {
          // tied with the next row; skipped when that row is already dead and the tie group ends there (the common pair case)
          const unsigned nl = (b < 31) ? (lo >> (b + 1)) & 1u : (hi & 1u), nt = (b < 31) ? (tlo >> (b + 1)) & 1u : (thi & 1u);
          if (nl | nt) { tie_b = b; break; }
        }
        MPN_NMS_KEEP_ROW(b)
      }
      while (tie_b < 0 && hi) {
        const int b = __ffs(hi) - 1;
        if (TIE && ((thi >> b) & 1u)) {
          const bool pair_done = (b < 31) && !((hi >> (b + 1)) & 1u) && !((thi >> (b + 1)) & 1u);
          if (!pair_done) { tie_b = 32 + b; break; }
        }
        MPN_NMS_KEEP_ROW(32 + b)
      }
#undef MPN_NMS_KEEP_ROW
      if (!SMEM) {
        unsigned long long bits = ((unsigned long long)kb_hi << 32) | kb_lo;
        while (bits) {
          int rb[8];
#pragma unroll
          for (int t = 0; t < 8; ++t) { rb[t] = bits ? __ffsll((long long)bits) - 1 : rb[0]; bits &= bits - 1ull; }
          unsigned long long m0[8], m1[8];
#pragma unroll
          for (int t = 0; t < 8; ++t) {
            m0[t] = mask_word(row0 + rb[t], w0);
            if (TWO) m1[t] = mask_word(row0 + rb[t], w1);
          }
#pragma unroll
          for (int t = 0; t < 8; ++t) { acc0 |= m0[t] & k0; if (TWO) acc1 |= m1[t] & k1; }
        }
      }
      cur = ~(((unsigned long long)hi << 32) | lo);
      rem0 |= acc0; if (TWO) rem1 |= acc1;
      if (lane == wl) { if (TWO && half) rem1 = cur; else rem0 = cur; }
    }
    if (!TIE || tie_b < 0) continue;
    // ---- general round for a candidate with a tied successor (rare)
    const int qb = tie_b;
    const int q = row0 + qb;
    int pb = q;
    if (TIE) {
      {                                  // q's score continues into q+1: is a tied box still alive?
        // publish the current removed-set so any lane can test liveness
        c.s_rrem[lane] = rem0; if (TWO) c.s_rrem[lane + 32] = rem1;
        __syncwarp();
        const float sq = c.s_score[q];
        int need = 0;
        if (lane == 0)
          for (int r = q + 1; r < n && c.s_score[r] == sq; ++r)
            if (!((c.s_rrem[r >> 6] >> (r & 63)) & 1ull)) { need = 1; break; }
        need = __shfl_sync(0xffffffffu, need, 0);
        if (need) {
          // ---- replay rounds [replayed, nkeep). (a) death round of every box removed in those rounds: the same mask rows
          //      as the forward pass, word-parallel over lanes, recording the round that first sets each bit
          for (int tt = replayed; tt < nkeep; ++tt) {
            const int kt = c.s_keep[tt];
            const int pbt = kt & 0x7fff;
            const int wbt = pbt >> 6;
            if (lane >= wbt && lane < nwords) {
              const unsigned long long mw = mask_word(pbt, lane);
              unsigned long long nb = mw & ~rr0; rr0 |= mw;
              while (nb) { const int bb = __ffsll((long long)nb) - 1; nb &= nb - 1ull; c.s_death[lane * 64 + bb] = (unsigned short)tt; }
            }
            if (TWO && lane + 32 >= wbt && lane + 32 < nwords) {
              const unsigned long long mw = mask_word(pbt, lane + 32);
              unsigned long long nb = mw & ~rr1; rr1 |= mw;
              while (nb) { const int bb = __ffsll((long long)nb) - 1; nb &= nb - 1ull; c.s_death[(lane + 32) * 64 + bb] = (unsigned short)tt; }
            }
            if (kt & 0x8000) {                   // a tie round that did not pick the first live box: symmetric suppression of [q, pb)
              const int qt = c.s_qalt[tt];
              for (int e = qt; e < pbt; ++e)
                if ((mask_word(e, wbt) >> (pbt & 63)) & 1ull) {
                  if (lane == (e >> 6) && !((rr0 >> (e & 63)) & 1ull)) { rr0 |= 1ull << (e & 63); c.s_death[e] = (unsigned short)tt; }
                  if (TWO && lane + 32 == (e >> 6) && !((rr1 >> (e & 63)) & 1ull)) { rr1 |= 1ull << (e & 63); c.s_death[e] = (unsigned short)tt; }
                }
            }
          }
          __syncwarp();
          // (b) nms.c:83-86, every round: the head (live occupant of the first live slot) moves into the selected box's
          //     slot. The head slot only moves forward. Every lane runs the same scalar walk and stores the same values
          //     (later rounds never write what an earlier round reads), so no warp collective sits on this chain.
          for (int tt = replayed; tt < nkeep; ++tt) {
            const int pbt = c.s_keep[tt] & 0x7fff;
            int head = -1;
            while (hp < n) {
              const int e = c.s_owner[hp];
              if (e >= 0 && (int)c.s_death[e] >= tt) { head = e; break; }      // alive at the start of round tt
              ++hp;
            }
            if (head < 0) break;
            const int lb = c.s_label[pbt];
            if (head != pbt) { c.s_owner[lb] = head; c.s_label[head] = lb; }
            c.s_owner[hp] = -1;
          }
          replayed = nkeep;
          __syncwarp();
          // ---- nms.c:74-81: first strict maximum in current order = smallest slot label among the live tied boxes
          c.s_rrem[lane] = rem0; if (TWO) c.s_rrem[lane + 32] = rem1;
          __syncwarp();
          if (lane == 0) {
            int bl = c.s_label[q];
            for (int r = q + 1; r < n && c.s_score[r] == sq; ++r)
              if (!((c.s_rrem[r >> 6] >> (r & 63)) & 1ull) && c.s_label[r] < bl) { pb = r; bl = c.s_label[r]; }
          }
          pb = __shfl_sync(0xffffffffu, pb, 0);
        }
      }
    }
    if (lane == 0) {                                            // no global access on the serial chain
      c.s_keep[nkeep] = (unsigned short)(pb | ((TIE && pb != q) ? 0x8000 : 0));
      if (TIE && pb != q) c.s_qalt[nkeep] = (unsigned short)q;
    }
    // ---- suppress: removed |= mask row of pb (upper triangle incl. the diagonal bit = pb itself)
    const int wb = pb >> 6;
    if (lane >= wb && lane < nwords) rem0 |= mask_word(pb, lane);
    if (TWO && lane + 32 >= wb && lane + 32 < nwords) rem1 |= mask_word(pb, lane + 32);
    if (TIE && pb != q) {
      // live boxes of the same score that precede pb in sorted order: suppression is symmetric (IoU is): bit [e][pb]
      for (int e = q; e < pb; ++e)
        if ((mask_word(e, wb) >> (pb & 63)) & 1ull) {
          if (lane == (e >> 6)) rem0 |= 1ull << (e & 63);
          if (TWO && lane + 32 == (e >> 6)) rem1 |= 1ull << (e & 63);
        }
    }
    ++nkeep;
  }
  return nkeep;
}

__global__ void __launch_bounds__(WARPK_THREADS)
nms_scan_warp_kernel(const unsigned long long *__restrict__ mask, const int32_t *__restrict__ order,
                     const float *__restrict__ sorted_score, int cap, int nwords_cap, int use_smem_mask,
                     const int32_t *__restrict__ counts, int32_t *__restrict__ tie_flag,
                     const int32_t *__restrict__ src_idx, int32_t *__restrict__ keep_idx,
                     int32_t *__restrict__ keep_counts) {
  MPN_PDL_SYNC();
  extern __shared__ unsigned long long s_dyn[];
  const int seg = blockIdx.x;
  const bool trace = (g_nms_trace != 0) && seg == 0;
  const long long t0 = clock64();
  const int n = counts ? counts[seg] : cap;
  if (n <= 0) { if (threadIdx.x == 0) { keep_counts[seg] = 0; tie_flag[seg] = 0; } return; }
  const int nwords = (n + 63) >> 6;
  const bool tie = tie_flag[seg] != 0;
  // dynamic smem carve-up: [mask n*nwords u64 (optional)] [rrem 64 u64] [tn 64 u64] [diag 64 u64] [score f32 cap] [label i32 cap] [owner i32 cap]
  //                        [keep u16 cap] [death u16 cap] [qalt u16 cap] [ord u16 cap]
  unsigned long long *s_mask = s_dyn;
  unsigned long long *s_rrem = s_dyn + (use_smem_mask ? (size_t)cap * nwords_cap : 0);
  unsigned long long *s_tn = s_rrem + 64;
  unsigned long long *s_diag = s_tn + 64;
  float *s_score = reinterpret_cast<float *>(s_diag + 64);
  int *s_label = reinterpret_cast<int *>(s_score + cap);
  int *s_owner = s_label + cap;
  unsigned short *s_keep = reinterpret_cast<unsigned short *>(s_owner + cap);
  unsigned short *s_death = s_keep + cap;      // round in which a box was removed (0xffff = alive); filled lazily by the tie replay
  unsigned short *s_qalt = s_death + cap;
  unsigned short *s_ord = s_qalt + cap;        // sorted position -> original row (n <= 4096)
  const unsigned long long *m = mask + (size_t)seg * cap * nwords_cap;
  const int32_t *ord = order + (size_t)seg * cap;
  // ---- prologue, whole block: everything the serial warp will need goes to shared memory with coalesced loads
  if (use_smem_mask) {
    if (nwords == nwords_cap && !(nwords & 1)) {
      // same row pitch: straight 16-byte copy (the never-written lower triangle is never read either)
      const uint4 *src = reinterpret_cast<const uint4 *>(m);
      uint4 *dst = reinterpret_cast<uint4 *>(s_mask);
      const int n4 = (n * nwords) >> 1;
#pragma unroll 8
      for (int i = threadIdx.x; i < n4; i += WARPK_THREADS) dst[i] = __ldg(src + i);
    } else {
#pragma unroll 8
      for (int i = threadIdx.x; i < n * nwords; i += WARPK_THREADS) {
        const int r = i / nwords, w = i - r * nwords;
        s_mask[i] = (w >= (r >> 6)) ? __ldg(m + (size_t)r * nwords_cap + w) : 0ull;   // only the upper triangle was computed
      }
    }
  }
  for (int p = threadIdx.x; p < n; p += WARPK_THREADS) {
    const int o = ord[p];
    s_ord[p] = (unsigned short)o;
    if (tie) {
      s_label[p] = o;            // slot label = position in the reference's pointer array
      s_score[p] = sorted_score[(size_t)seg * cap + p];
      s_owner[o] = p;            // slot -> sorted position of its occupant
      s_death[p] = 0xffffu;
    }
  }
  __syncthreads();
  if (tie) {
    // tienext bit p = (score[p] == score[p+1]): one ballot per 32 positions
    unsigned *tn32 = reinterpret_cast<unsigned *>(s_tn);
    for (int base = 0; base < nwords * 64; base += WARPK_THREADS) {
      const int p = base + threadIdx.x;
      const bool eq = (p + 1 < n) && (s_score[p] == s_score[p + 1]);
      const unsigned b = __ballot_sync(0xffffffffu, eq);
      if ((threadIdx.x & 31) == 0 && p < nwords * 64) tn32[p >> 5] = b;
    }
    __syncthreads();
  }
  if (threadIdx.x >= 32) return;
  const int lane = threadIdx.x;
  const long long t1 = clock64();
  int nkeep;
  const WalkCtx wc{s_mask, m, s_tn, s_diag, s_score, s_label, s_owner, s_rrem, s_keep, s_death, s_qalt, n, nwords, nwords_cap, use_smem_mask};
  if (use_smem_mask) {          // n <= 1024, hence one removed-word per lane
    nkeep = tie ? nms_walk<true, false, true>(wc, lane) : nms_walk<false, false, true>(wc, lane);
  } else {
    if (tie) nkeep = (nwords > 32) ? nms_walk<true, true, false>(wc, lane) : nms_walk<true, false, false>(wc, lane);
    else nkeep = (nwords > 32) ? nms_walk<false, true, false>(wc, lane) : nms_walk<false, false, false>(wc, lane);
  }
  __syncwarp();
  const long long t2 = clock64();
  for (int k = lane; k < nkeep; k += 32) {
    const int o = s_ord[s_keep[k] & 0x7fff];
    keep_idx[(size_t)seg * cap + k] = src_idx ? src_idx[(size_t)seg * cap + o] : o;
  }
  if (lane == 0) { keep_counts[seg] = nkeep; tie_flag[seg] = 0; }     // last reader of the flag: leave it zero for the next call
  if (trace && lane == 0)
    printf("[nms trace] seg 0: n %d tie %d kept %d | prologue %lld cyc, walk %lld cyc, output %lld cyc\n", n, (int)tie, nkeep,
           t1 - t0, t2 - t1, clock64() - t2);
}

constexpr int EXACT_THREADS = 512;

// Exact emulation of nms.c:66-100 for segments with tied scores. One block per segment.
// cur[] (scratch, cap ints per segment) is the reference's pointer array as row indices.
__global__ void __launch_bounds__(EXACT_THREADS)
nms_exact_kernel(const float *__restrict__ sb, int cap, const int32_t *__restrict__ counts,
                 const int32_t *__restrict__ tie_flag, float thr, int32_t *__restrict__ cur_all,
                 const int32_t *__restrict__ src_idx, int32_t *__restrict__ keep_idx,
                 int32_t *__restrict__ keep_counts) {
  const int seg = blockIdx.x;
  if (!tie_flag[seg]) return;
  const int n = counts ? counts[seg] : cap;
  const float *seg_sb = sb + (size_t)seg * cap * 5;
  int32_t *cur = cur_all + (size_t)seg * cap;
  __shared__ float s_best_s[EXACT_THREADS / 32];
  __shared__ int s_best_p[EXACT_THREADS / 32];
  __shared__ int s_warp_tot[EXACT_THREADS / 32];
  __shared__ int s_sel, s_tile_total;
  const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
  for (int i = tid; i < n; i += EXACT_THREADS) cur[i] = i;
  __syncthreads();
  int base = 0, num = n, nkeep = 0;
  while (num > 0) {
    // ---- first strict maximum in current order (nms.c:74-81): max score, lowest position
    float bs = -10000000.0f; int bp = -1;
    for (int p = tid; p < num; p += EXACT_THREADS) {   // ascending p per thread => strict > keeps first
      float s = seg_sb[(size_t)cur[base + p] * 5 + 4];
      if (s > bs) { bs = s; bp = p; }
    }
#pragma unroll
    for (int off = 16; off > 0; off >>= 1) {
      float os = __shfl_xor_sync(0xffffffffu, bs, off);
      int op = __shfl_xor_sync(0xffffffffu, bp, off);
      bool take = (op >= 0) && (bp < 0 || os > bs || (os == bs && op < bp));
      if (take) { bs = os; bp = op; }
    }
    if (lane == 0) { s_best_s[wid] = bs; s_best_p[wid] = bp; }
    __syncthreads();
    if (tid == 0) {
      float fs = s_best_s[0]; int fp = s_best_p[0];
      for (int w = 1; w < EXACT_THREADS / 32; ++w) {
        float os = s_best_s[w]; int op = s_best_p[w];
        if ((op >= 0) && (fp < 0 || os > fs || (os == fs && op < fp))) { fs = os; fp = op; }
      }
      if (fp >= 0) {                                   // swap to front (nms.c:83-86)
        int32_t b = cur[base + fp]; cur[base + fp] = cur[base]; cur[base] = b;
        keep_idx[(size_t)seg * cap + nkeep] = src_idx ? src_idx[(size_t)seg * cap + b] : b;
      }
      s_sel = fp;
    }
    __syncthreads();
    if (s_sel < 0) break;      // every remaining score <= -1e7 (or NaN): the reference reads boxes[-1] here (UB)
    const int32_t bidx = cur[base];
    const float *bb = seg_sb + (size_t)bidx * 5;
    const float bx1 = bb[0], by1 = bb[1], bx2 = bb[2], by2 = bb[3];
    nkeep++; base++;
    const int m = num - 1;
    // ---- order-preserving survivor compaction (nms.c:90-99)
    int good = 0;
    for (int t0 = 0; t0 < m; t0 += EXACT_THREADS) {
      int p = t0 + tid; int32_t v = -1; int flag = 0;
      if (p < m) {
        v = cur[base + p];
        const float *o = seg_sb + (size_t)v * 5;
        float ov = iou_ref(bx1, by1, bx2, by2, o[0], o[1], o[2], o[3]);
        flag = (ov <= thr) ? 1 : 0;
      }
      unsigned ball = __ballot_sync(0xffffffffu, flag);
      int pre = __popc(ball & ((1u << lane) - 1u));
      if (lane == 0) s_warp_tot[wid] = __popc(ball);
      __syncthreads();                                  // all reads of this tile done
      if (tid == 0) {
        int acc = 0;
        for (int w = 0; w < EXACT_THREADS / 32; ++w) { int t = s_warp_tot[w]; s_warp_tot[w] = acc; acc += t; }
        s_tile_total = acc;
      }
      __syncthreads();
      if (flag) cur[base + good + s_warp_tot[wid] + pre] = v;
      good += s_tile_total;
      __syncthreads();
    }
    num = good;
  }
  if (tid == 0) keep_counts[seg] = nkeep;
}

}  // namespace

// ---- internal launcher (device buffers, uniform capacity) --------------------------
// Workspace layout inside ctx scratch slot 2.
int mpn_nms_launch(mpn_ctx *ctx, const float *sb_dev, int cap, int nseg, const int32_t *counts_dev,
                   const int32_t *src_idx_dev, float thr, int32_t *keep_idx_dev,
                   int32_t *keep_counts_dev) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_NMS);
  if (nseg <= 0 || cap <= 0) return MPN_OK;
  const int nwords = (cap + 63) / 64;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  size_t o_order = take(sizeof(int32_t) * (size_t)nseg * cap);
  size_t o_cur = take(sizeof(int32_t) * (size_t)nseg * cap);
  size_t o_sorted = take(sizeof(float4) * (size_t)nseg * cap);
  size_t o_tie = take(sizeof(int32_t) * (size_t)nseg);
  size_t o_sscore = take(sizeof(float) * (size_t)nseg * cap);
  size_t o_mask = take(sizeof(unsigned long long) * (size_t)nseg * cap * nwords);
  char *ws = nullptr;
  MPN_TRY(mpn_scratch2(ctx, off, (void **)&ws));
  int32_t *order = (int32_t *)(ws + o_order);
  int32_t *cur = (int32_t *)(ws + o_cur);
  float4 *sorted = (float4 *)(ws + o_sorted);
  int32_t *tie = (int32_t *)(ws + o_tie);
  float *sscore = (float *)(ws + o_sscore);
  unsigned long long *mask = (unsigned long long *)(ws + o_mask);
  const bool small = cap <= WARP_CAP;
  // the warp kernel (last reader) leaves the flags zero, so steady-state calls with the same layout need no memset
  if (!small || ctx->nms_tie_ptr != (void *)tie || ctx->nms_tie_n < nseg) {
    MPN_CUDA(ctx, cudaMemsetAsync(tie, 0, sizeof(int32_t) * nseg, ctx->stream));
    ctx->nms_tie_ptr = small ? (void *)tie : nullptr; ctx->nms_tie_n = small ? nseg : 0;
  }
  if (!small) MPN_CUDA(ctx, cudaMemsetAsync(keep_counts_dev, 0, sizeof(int32_t) * nseg, ctx->stream));   // the warp kernel writes every count
  dim3 g1((cap + RANK_ELEMS - 1) / RANK_ELEMS, nseg);
  MPN_CUDA(ctx, mpn_launch_pdl(ctx, nms_rank_kernel, g1, dim3(RANK_THREADS), 0, sb_dev, cap, counts_dev, order, sorted, tie, sscore));
  MPN_LAUNCHED(ctx);
  dim3 g2((unsigned)(nwords * (nwords + 1) / 2), 1, nseg);   // upper-triangle tiles only
  MPN_CUDA(ctx, mpn_launch_pdl(ctx, nms_mask_kernel, g2, dim3(64), 0, (const float4 *)sorted, cap, nwords, counts_dev, (const int32_t *)tie, small ? 0 : 1, thr, mask));
  MPN_LAUNCHED(ctx);
  if (small) {
    const int use_smem_mask = cap <= WARP_SMEM_MASK_CAP ? 1 : 0;
    const size_t smem = (use_smem_mask ? sizeof(unsigned long long) * (size_t)cap * nwords : 0) + (size_t)cap * 20 + 192 * 8 + 64;
    if (smem > 48 * 1024)
      MPN_CUDA(ctx, cudaFuncSetAttribute(nms_scan_warp_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    {
      static int trace_set = -1;
      if (trace_set < 0) {
        const char *e = getenv("MPN_NMS_TRACE");
        trace_set = (e && e[0] == '1') ? 1 : 0;
        if (trace_set) MPN_CUDA(ctx, cudaMemcpyToSymbol(g_nms_trace, &trace_set, sizeof(int)));
      }
    }
    MPN_CUDA(ctx, mpn_launch_pdl(ctx, nms_scan_warp_kernel, dim3(nseg), dim3(WARPK_THREADS), smem, (const unsigned long long *)mask,
                                 (const int32_t *)order, (const float *)sscore, cap, nwords, use_smem_mask, counts_dev, tie,
                                 src_idx_dev, keep_idx_dev, keep_counts_dev));
    MPN_LAUNCHED(ctx);
    return MPN_OK;
  }
  nms_scan_kernel<<<nseg, SCAN_THREADS, sizeof(unsigned long long) * nwords, ctx->stream>>>(
      mask, order, cap, nwords, counts_dev, tie, src_idx_dev, keep_idx_dev, keep_counts_dev);
  MPN_LAUNCHED(ctx);
  nms_exact_kernel<<<nseg, EXACT_THREADS, 0, ctx->stream>>>(sb_dev, cap, counts_dev, tie, thr, cur,
                                                            src_idx_dev, keep_idx_dev, keep_counts_dev);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// ---- the keep lists of a batched detect's (image, class) segments (capacity cap each) into image-major blocks: image i's
// (C - 1) x R_i block starts at (C - 1) * off[i], class j's list at row j - 1 of it; entries past a list's count are -1
namespace {
__global__ void nms_keep_image_major_kernel(const int32_t *__restrict__ keep_seg, const int32_t *__restrict__ counts, ImageSegs segs,
                                            int nfg, int cap, int32_t *__restrict__ keep_out) {
  MPN_PDL_SYNC();
  const int i = blockIdx.y, j = blockIdx.x;
  const int64_t r0 = segs.off[i], Ri = segs.off[i + 1] - r0;
  const size_t s = (size_t)i * nfg + j;
  const int n = counts[s];
  int32_t *o = keep_out + nfg * r0 + j * Ri;
  for (int64_t k = threadIdx.x; k < Ri; k += blockDim.x) o[k] = k < n ? keep_seg[s * cap + k] : -1;
}
}  // namespace

int mpn_nms_keep_image_major_launch(mpn_ctx *ctx, const int32_t *keep_seg_dev, const int32_t *counts_dev, const ImageSegs &segs, int nfg,
                                    int cap, int32_t *keep_out_dev) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_NMS);
  if (nfg <= 0 || segs.n <= 0 || cap <= 0) return MPN_OK;
  MPN_CUDA(ctx, mpn_launch_pdl(ctx, nms_keep_image_major_kernel, dim3(nfg, segs.n), dim3(128), 0, keep_seg_dev, counts_dev, segs, nfg, cap,
                               keep_out_dev));
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// ---- nms_dense (utils.lua:402-462): different IoU rounding order, index output -------
namespace {
__device__ __forceinline__ float iou_dense(float4 c, float areac, float4 j, float areaj) {
  float xx1 = (j.x < c.x) ? c.x : j.x;                       // clamp(x1[c], inf)
  float yy1 = (j.y < c.y) ? c.y : j.y;
  float xx2 = (j.z < 0.f) ? 0.f : ((j.z > c.z) ? c.z : j.z); // clamp(0, x2[c])
  float yy2 = (j.w < 0.f) ? 0.f : ((j.w > c.w) ? c.w : j.w);
  float w = __fadd_rn(__fsub_rn(xx2, xx1), 1.0f); if (w < 0.f) w = 0.f;
  float h = __fadd_rn(__fsub_rn(yy2, yy1), 1.0f); if (h < 0.f) h = 0.f;
  float inter = __fmul_rn(w, h);
  float uni = __fadd_rn(__fsub_rn(areaj, inter), areac);
  return __fdiv_rn(inter, uni);
}
// same tiling as nms_mask_kernel, but nms_dense marks EVERY j (also j<i; those are
// already decided when i is reached, so only j>i matters) => identical structure.
__global__ void __launch_bounds__(64)
nms_dense_mask_kernel(const float4 *__restrict__ boxes, int n, int nwords, float thr,
                      unsigned long long *__restrict__ mask) {
  const int rb = blockIdx.y, cb = blockIdx.x;
  if (cb < rb) return;
  __shared__ float4 s_col[64];
  const int t = threadIdx.x, cj = cb * 64 + t;
  s_col[t] = (cj < n) ? boxes[cj] : make_float4(0, 0, 0, 0);
  __syncthreads();
  const int i = rb * 64 + t;
  if (i >= n) return;
  const float4 a = boxes[i];
  const float areaa = __fmul_rn(__fadd_rn(__fsub_rn(a.z, a.x), 1.0f), __fadd_rn(__fsub_rn(a.w, a.y), 1.0f));
  unsigned long long bits = 0ull;
  const int ncols = min(64, n - cb * 64);
  const int start = (rb == cb) ? t + 1 : 0;
  for (int c = start; c < ncols; ++c) {
    float4 b = s_col[c];
    float areab = __fmul_rn(__fadd_rn(__fsub_rn(b.z, b.x), 1.0f), __fadd_rn(__fsub_rn(b.w, b.y), 1.0f));
    float v = iou_dense(a, areaa, b, areab);
    if (v > thr) bits |= (1ull << c);
  }
  if (rb == cb) bits |= 1ull << t;
  mask[(size_t)i * nwords + cb] = bits;
}
}  // namespace

int mpn_nms_dense_launch(mpn_ctx *ctx, const float *sb_dev, int n, float thr, int32_t *pick_dev,
                         int32_t *count_dev) {
  if (n <= 0) return MPN_OK;
  const int nwords = (n + 63) / 64;
  size_t off = 0;
  auto take = [&](size_t bytes) { size_t o = off; off += (bytes + 255) & ~(size_t)255; return o; };
  size_t o_order = take(sizeof(int32_t) * n), o_sorted = take(sizeof(float4) * n),
         o_tie = take(sizeof(int32_t) * 2), o_mask = take(sizeof(unsigned long long) * (size_t)n * nwords);
  char *ws = nullptr;
  MPN_TRY(mpn_scratch2(ctx, off, (void **)&ws));
  int32_t *order = (int32_t *)(ws + o_order);
  float4 *sorted = (float4 *)(ws + o_sorted);
  int32_t *tie = (int32_t *)(ws + o_tie);            // tie[0]: real flag (ignored), tie[1]: always 0
  ctx->nms_tie_ptr = nullptr; ctx->nms_tie_n = 0;    // scratch2 is re-laid out: the batched path must zero its flags again
  unsigned long long *mask = (unsigned long long *)(ws + o_mask);
  MPN_CUDA(ctx, cudaMemsetAsync(tie, 0, sizeof(int32_t) * 2, ctx->stream));
  MPN_CUDA(ctx, cudaMemsetAsync(count_dev, 0, sizeof(int32_t), ctx->stream));
  dim3 g1((n + RANK_ELEMS - 1) / RANK_ELEMS, 1);
  nms_rank_kernel<<<g1, RANK_THREADS, 0, ctx->stream>>>(sb_dev, n, nullptr, order, sorted, tie, nullptr);
  MPN_LAUNCHED(ctx);
  dim3 g2(nwords, nwords, 1);
  nms_dense_mask_kernel<<<g2, 64, 0, ctx->stream>>>(sorted, n, nwords, thr, mask);
  MPN_LAUNCHED(ctx);
  nms_scan_kernel<<<1, SCAN_THREADS, sizeof(unsigned long long) * nwords, ctx->stream>>>(
      mask, order, n, nwords, nullptr, tie + 1, nullptr, pick_dev, count_dev);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// ---- bbox_vote (nms.c:110-142): one block per NMS box, fixed-order accumulation -------
namespace {
// The reference accumulates over j = 0..N-1 sequentially in fp32. A parallel tree would
// change the rounding, so each block walks j in order in chunks: lanes evaluate the
// overlaps in parallel, then ONE thread adds the selected terms in ascending j.
__global__ void __launch_bounds__(256)
bbox_vote_kernel(const float *__restrict__ nms_boxes, int K, const float *__restrict__ sb, int N,
                 float thr, float *__restrict__ res) {
  const int i = blockIdx.x;
  if (i >= K) return;
  __shared__ unsigned char s_sel[256];
  const float *nb = nms_boxes + (size_t)i * 5;
  const float nx1 = nb[0], ny1 = nb[1], nx2 = nb[2], ny2 = nb[3];
  float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f, acc4 = 0.f;
  for (int base = 0; base < N; base += 256) {
    int j = base + threadIdx.x;
    unsigned char sel = 0;
    if (j < N) {
      const float *o = sb + (size_t)j * 5;
      float ov = iou_ref(o[0], o[1], o[2], o[3], nx1, ny1, nx2, ny2);   // overlap(scored_j, nms_i), nms.c:129
      sel = (ov > thr) ? 1 : 0;
    }
    s_sel[threadIdx.x] = sel;
    __syncthreads();
    if (threadIdx.x == 0) {
      int lim = min(256, N - base);
      for (int t = 0; t < lim; ++t) {
        if (s_sel[t]) {
          const float *o = sb + (size_t)(base + t) * 5;
          float s = o[4];
          acc0 = __fadd_rn(acc0, __fmul_rn(o[0], s));
          acc1 = __fadd_rn(acc1, __fmul_rn(o[1], s));
          acc2 = __fadd_rn(acc2, __fmul_rn(o[2], s));
          acc3 = __fadd_rn(acc3, __fmul_rn(o[3], s));
          acc4 = __fadd_rn(acc4, s);
        }
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float *r = res + (size_t)i * 5;
    r[0] = __fdiv_rn(acc0, acc4); r[1] = __fdiv_rn(acc1, acc4);
    r[2] = __fdiv_rn(acc2, acc4); r[3] = __fdiv_rn(acc3, acc4);
    r[4] = nb[4];
  }
}
}  // namespace

// Batched form for Tester_FRCNN:testOne on the device (Tester_FRCNN.lua:118-124): block (i, seg) votes the i-th NMS box of
// class seg + 1 — row keep_idx[seg][i] of the detect outputs — over the class's gathered rows sb[seg][0 .. counts[seg])
// with their scores raised to score_pow (opt.test_bbox_voting_score_pow; 1 = untouched, the only bit-exact setting:
// powf is not libm's). Same sequential accumulation as bbox_vote_kernel. res: nseg x cap x 5.
namespace {
__global__ void __launch_bounds__(256)
bbox_vote_batched_kernel(const float *__restrict__ sb, const int32_t *__restrict__ counts, const int32_t *__restrict__ keep_idx,
                         const int32_t *__restrict__ keep_counts, const float *__restrict__ scores, const float *__restrict__ bboxes,
                         int C, int cap, float thr, float score_pow, float *__restrict__ res) {
  const int seg = blockIdx.y, i = blockIdx.x;
  if (i >= keep_counts[seg]) return;
  __shared__ unsigned char s_sel[256];
  const int row = keep_idx[(size_t)seg * cap + i], N = counts[seg];
  const float4 nbx = reinterpret_cast<const float4 *>(bboxes)[(size_t)row * C + seg + 1];
  const float nscore = scores[(size_t)row * C + seg + 1];
  const float *seg_sb = sb + (size_t)seg * cap * 5;
  float acc0 = 0.f, acc1 = 0.f, acc2 = 0.f, acc3 = 0.f, acc4 = 0.f;
  for (int base = 0; base < N; base += 256) {
    const int j = base + threadIdx.x;
    unsigned char sel = 0;
    if (j < N) {
      const float *o = seg_sb + (size_t)j * 5;
      sel = (iou_ref(o[0], o[1], o[2], o[3], nbx.x, nbx.y, nbx.z, nbx.w) > thr) ? 1 : 0;
    }
    s_sel[threadIdx.x] = sel;
    __syncthreads();
    if (threadIdx.x == 0) {
      const int lim = min(256, N - base);
      for (int t = 0; t < lim; ++t) {
        if (s_sel[t]) {
          const float *o = seg_sb + (size_t)(base + t) * 5;
          const float s = score_pow == 1.f ? o[4] : powf(o[4], score_pow);
          acc0 = __fadd_rn(acc0, __fmul_rn(o[0], s));
          acc1 = __fadd_rn(acc1, __fmul_rn(o[1], s));
          acc2 = __fadd_rn(acc2, __fmul_rn(o[2], s));
          acc3 = __fadd_rn(acc3, __fmul_rn(o[3], s));
          acc4 = __fadd_rn(acc4, s);
        }
      }
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float *r = res + ((size_t)seg * cap + i) * 5;
    r[0] = __fdiv_rn(acc0, acc4); r[1] = __fdiv_rn(acc1, acc4);
    r[2] = __fdiv_rn(acc2, acc4); r[3] = __fdiv_rn(acc3, acc4);
    r[4] = nscore;
  }
}
}  // namespace

int mpn_bbox_vote_batched_launch(mpn_ctx *ctx, const float *sb_dev, const int32_t *counts_dev, const int32_t *keep_idx_dev,
                                 const int32_t *keep_counts_dev, const float *scores_dev, const float *bboxes_dev, int C, int cap,
                                 float thr, float score_pow, float *res_dev) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_NMS);
  if (C <= 1 || cap <= 0) return MPN_OK;
  bbox_vote_batched_kernel<<<dim3((unsigned)cap, (unsigned)(C - 1)), 256, 0, ctx->stream>>>(sb_dev, counts_dev, keep_idx_dev, keep_counts_dev,
                                                                                         scores_dev, bboxes_dev, C, cap, thr, score_pow, res_dev);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

int mpn_bbox_vote_launch(mpn_ctx *ctx, const float *nms_dev, int K, const float *sb_dev, int N,
                         float thr, float *res_dev) {
  if (K <= 0) return MPN_OK;
  bbox_vote_kernel<<<K, 256, 0, ctx->stream>>>(nms_dev, K, sb_dev, N, thr, res_dev);
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// gemm_tc.cu — the tensor-core engine: implicit-GEMM convolution / Linear on Hopper warpgroup MMA (wgmma) with
// register accumulators, operands staged by TMA. sm_90a.
//
// Replaces cudnn.SpatialConvolution and nn.Linear (cuBLAS SGEMM) on the reference hot path
// (SURVEY 2.2: trunks of models/{vgg,multipathnet,resnet}.lua, fc6/fc7/cls/bbox of
// model_utils.lua:105-119, 1x1 conv_mix of model_utils.lua:242).
//
// Numerics: fp32-faithful "bf16x3" — every operand is held as two bf16 planes
// (hi = rn(x), lo = rn(x-hi)); each k16 step issues A_lo*B_hi + A_hi*B_lo + A_hi*B_hi into one fp32
// accumulator (the dropped lo*lo term is ~2^-18 relative). Result error ~1e-5 relative,
// well inside the 1e-3 parity bar that single-pass TF32 (10-bit mantissa) misses over
// 13 convs + 2 fcs, at 3 bf16 MMAs per step = 1.5x the cost of one TF32 pass.
//
// Kernel shape (one output tile of 128 pixels x BN channels per CTA, warp-specialised, 3 warpgroups):
//   warpgroup 0    : TMA producer (one thread) — per K block: A tile (128 pixels x 64 ch, hi+lo) by a 4-D tiled
//                    tensor map over the NHWC activation whose box is a tn x th x tw pixel patch shifted by the filter
//                    tap (zero OOB fill = conv padding, elementStrides = conv stride), B tile (BN x 64, hi+lo) from the
//                    [Cout][kh*kw*Cin] weights, into a ring of S stages (full / empty mbarriers).
//   warpgroups 1-2 : consumers — each owns 64 rows of the tile: wgmma m64nBNk16 straight from the 128B-swizzled smem
//                    tiles into registers; then the epilogue: the fp32 tile is staged in shared memory and every thread
//                    finishes one pixel row: + bias (+ residual) (ReLU), re-split to hi/lo (NHWC, next layer's A
//                    operand) and/or fp32, optional fused 2x2/2 max pool.
#include "conv_gemm.cuh"
#include "wgmma.cuh"
#include <algorithm>
#include <stdlib.h>
#include <string.h>

namespace {

constexpr int BM = 128;          // pixels per tile (two m64 warpgroup MMAs)
constexpr int BK = 64;           // bf16 elements per K block = one 128B swizzle row
constexpr int TC_THREADS = 384;  // producer warpgroup + two consumer warpgroups
constexpr int CONS_THREADS = 256;
constexpr int A_TILE_BYTES = BM * BK * 2;   // 16 KB per plane
constexpr int SMEM_BUDGET = 196608;         // pipeline ring; the epilogue staging tile reuses it

// W16: the B operand is one fp16 plane instead of the bf16 hi/lo pair
__host__ __device__ constexpr int stage_bytes(int BN, bool W16 = false) { return 2 * A_TILE_BYTES + (W16 ? 1 : 2) * BN * BK * 2; }
__host__ __device__ constexpr int num_stages(int BN, bool W16 = false) {
  return (SMEM_BUDGET / stage_bytes(BN, W16)) > 4 ? 4 : (SMEM_BUDGET / stage_bytes(BN, W16));
}
__host__ __device__ constexpr int stg_ld(int BN) { return BN + 4; }     // fp32 staging row stride: conflict-free float4 row reads
static_assert(BM * (256 + 4) * 4 <= 2 * stage_bytes(256), "staging tile must fit in the ring");

struct TcParams {
  int N, Ho, Wo, Cout;           // output geometry (flat mode: N=1, Ho=1, Wo=pixels)
  int kh, kw, stride, pad;
  int cblocks;                   // Cin / 64
  int tn, th, tw;                // tile decomposition (powers of two)
  int tiles_img, tiles_h, tiles_w, tiles_n;
  const float *bias;
  const __nv_bfloat16 *res_hi, *res_lo; long long res_ld;
  __nv_bfloat16 *out_hi, *out_lo; long long out_ld;
  float *out_f32; long long out_f32_ld;
  __nv_bfloat16 *pool_hi, *pool_lo; long long pool_ld; int Hp, Wp;   // fused 2x2/2 max pool of the output (16 x 8 patches only)
  int relu;
  int splitk, kb_per_split;      // split-K: unit = (tile, split); each split owns kb_per_split K blocks and writes raw fp32 partials
  long long split_stride;        // elements between the partial planes of consecutive splits (out_f32 is the workspace then)
  unsigned long long *tl_min, *tl_max;   // diagnostics: %globaltimer stamps of this launch (4 + 4 u64) or null
  float acc_scale;               // W16 kernels: accumulator * acc_scale (= 1 / the weight plane's power-of-two scale) before the bias; 1 otherwise
  int out_fmt;                   // plane format of out_hi / out_lo (and the pooled output): 0 = bf16 split, 1 = fp16 split
  unsigned *ovf;                 // fp16-overflow flag of the ctx (out_fmt == 1)
};

// ---------------------------------------------------------------- timeline stamps (diagnostics)
__device__ __forceinline__ unsigned long long gtimer() {
  unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t;
}
__device__ __forceinline__ void tl_min_stamp(const unsigned long long *base_, int i) {
  if (base_) atomicMin(const_cast<unsigned long long *>(base_) + i, gtimer());
}
__device__ __forceinline__ void tl_max_stamp(const unsigned long long *base_, int i) {
  if (base_) atomicMax(const_cast<unsigned long long *>(base_) + i, gtimer());
}
// ---------------------------------------------------------------- PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
  asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
// Bounded spin: a protocol bug must surface as a trap (a launch error), never as a silent
// GPU hang. ~2^26 polls is seconds of wall time. No printf here: a function call inside the
// consumer K loop, where a wgmma group is in flight, makes ptxas serialise every wgmma (C7510).
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
  uint32_t done;
  uint32_t spins = 0;
  do {
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(done) : "r"(bar), "r"(parity) : "memory");
    if (!done && ++spins == (1u << 26)) __trap();
  } while (!done);
}
__device__ __forceinline__ void tma_load_4d(uint32_t dst, const CUtensorMap *tm, uint32_t bar, int c0, int c1,
                                            int c2, int c3) {
  asm volatile(
      "cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_2d(uint32_t dst, const CUtensorMap *tm, uint32_t bar, int c0, int c1) {
  asm volatile(
      "cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
      ::"r"(dst), "l"(reinterpret_cast<uint64_t>(tm)), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void prefetch_tmap(const CUtensorMap *tm) {
  asm volatile("prefetch.tensormap [%0];" ::"l"(reinterpret_cast<uint64_t>(tm)) : "memory");
}
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// K-major, 128B-swizzled smem tile descriptor (GMMA descriptor): start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled
// K-major; 1) | SBO>>4 [32,46) = 1024B/16 (stride between 8-row groups) | layout SWIZZLE_128B=1 [62,64)
__device__ __forceinline__ uint64_t make_smem_desc(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(1024 >> 4) << 32;
  d |= (uint64_t)1 << 62;
  return d;
}

// one K block (64 = 4 x k16) of a 64-row warpgroup slice: three bf16 products per k16 (A_lo x B_hi, A_hi x B_lo,
// A_hi x B_hi), or two fp16 products (A_lo x W16, A_hi x W16; b_hi holds the single fp16 weight plane). first: zero-init.
template <int BN, bool W16>
__device__ __forceinline__ void mma_kblock(float (&acc)[BN / 2], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, bool first) {
#pragma unroll
  for (int k = 0; k < BK / 16; ++k) {
    const uint64_t adv = (uint64_t)((k * 16 * 2) >> 4);     // +32B per k16 inside the swizzle atom
    const uint32_t later = (first && k == 0) ? 0u : 1u;
    wgmma_nk16<BN, W16>(acc, a_lo + adv, b_hi + adv, later);
    if (!W16) wgmma_nk16<BN, W16>(acc, a_hi + adv, b_lo + adv, 1u);
    wgmma_nk16<BN, W16>(acc, a_hi + adv, b_hi + adv, 1u);
  }
}

// the warpgroup's accumulator fragment -> rows [64 g, 64 g + 64) of the fp32 staging tile (row stride stg_ld(BN))
template <int BN>
__device__ __forceinline__ void stage_acc(float *stg, const float (&acc)[BN / 2], int g, int t) {
  const int r0 = g * 64 + (t >> 5) * 16 + ((t & 31) >> 2), c0 = 2 * (t & 3);
#pragma unroll
  for (int j = 0; j < BN / 8; ++j) {
    *reinterpret_cast<float2 *>(stg + r0 * stg_ld(BN) + 8 * j + c0) = make_float2(acc[4 * j], acc[4 * j + 1]);
    *reinterpret_cast<float2 *>(stg + (r0 + 8) * stg_ld(BN) + 8 * j + c0) = make_float2(acc[4 * j + 2], acc[4 * j + 3]);
  }
}

// ---------------------------------------------------------------- epilogue of one pixel row (shared by both kernels)
// srow = the row's BN fp32 accumulators in shared memory; this thread takes the 32-channel chunks ch_first, ch_first + 2, ...
// + bias (+ residual) (ReLU); re-split to hi/lo and/or fp32. Rows of a warp are 32 consecutive tile rows.
template <int BN, bool W16>
__device__ __forceinline__ void epilogue_row(const TcParams &p, const float *srow, int nt, bool row_ok, long long pix,
                                             float *out_f32, int ch_first, long long ppix) {
  // fused 2x2/2 max pool (16 x 8 patches: lane = (h & 3) * 8 + w, so a window is lanes {l, l^1, l^8, l^9});
  // ppix = pooled pixel this lane writes (its window's top-left lane), -1 otherwise. pool is warp-uniform.
  const bool pool = (p.pool_hi != nullptr);
  const int tile_end = min(p.Cout, nt * BN + BN);
#pragma unroll 1
  for (int ch = ch_first; ch < BN / 32; ch += 2) {
    const int col0 = nt * BN + ch * 32;
    if (col0 >= tile_end) break;
    float v[32];
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float4 x = *reinterpret_cast<const float4 *>(srow + ch * 32 + 4 * j);
      v[4 * j] = x.x; v[4 * j + 1] = x.y; v[4 * j + 2] = x.z; v[4 * j + 3] = x.w;
    }
    if (W16) {                             // undo the weight plane's power-of-two scale (exact)
#pragma unroll
      for (int e = 0; e < 32; ++e) v[e] *= p.acc_scale;
    }
    if (!(row_ok || pool)) continue;
#pragma unroll
    for (int g = 0; g < 4; ++g) {             // 8 output channels per group
      const int c = col0 + g * 8;
      if (c >= tile_end) break;
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = v[g * 8 + e];
      const bool full8 = (c + 8 <= tile_end);
      if (p.bias) {
        if (full8) {
          const float4 b0 = __ldg(reinterpret_cast<const float4 *>(p.bias + c));
          const float4 b1 = __ldg(reinterpret_cast<const float4 *>(p.bias + c + 4));
          f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
          f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
        } else {
          for (int e = 0; e < 8 && c + e < p.Cout; ++e) f[e] += __ldg(p.bias + c + e);
        }
      }
      if (p.res_hi && full8 && row_ok) {
        const uint4 rh = *reinterpret_cast<const uint4 *>(p.res_hi + pix * p.res_ld + c);
        const uint4 rl = *reinterpret_cast<const uint4 *>(p.res_lo + pix * p.res_ld + c);
        const uint32_t hh[4] = {rh.x, rh.y, rh.z, rh.w}, ll[4] = {rl.x, rl.y, rl.z, rl.w};
#pragma unroll
        for (int t = 0; t < 4; ++t) {
          float2 x = bf16x2_to_float2(hh[t]), y = bf16x2_to_float2(ll[t]);
          f[2 * t] += x.x + y.x; f[2 * t + 1] += x.y + y.y;
        }
      }
      if (p.relu) {
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = fmaxf(f[e], 0.f);
      }
      if (p.out_hi && full8 && row_ok) {
        uint32_t oh[4], ol[4];
#pragma unroll
        for (int t = 0; t < 4; ++t) split_x2(p.out_fmt, f[2 * t], f[2 * t + 1], oh[t], ol[t], p.ovf);      // packed cvt.rn.{bf16x2,f16x2}.f32
        *reinterpret_cast<uint4 *>(p.out_hi + pix * p.out_ld + c) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
        *reinterpret_cast<uint4 *>(p.out_lo + pix * p.out_ld + c) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
      }
      if (pool) {
        // rows outside the image hold bias-only garbage: exclude them (ceil-mode windows at odd borders)
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          float x = row_ok ? f[e] : -INFINITY;
          x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 1));
          x = fmaxf(x, __shfl_xor_sync(0xffffffffu, x, 8));
          f[e] = x;
        }
        if (ppix >= 0 && full8) {
          uint32_t oh[4], ol[4];
#pragma unroll
          for (int t = 0; t < 4; ++t) split_x2(p.out_fmt, f[2 * t], f[2 * t + 1], oh[t], ol[t], p.ovf);
          *reinterpret_cast<uint4 *>(p.pool_hi + ppix * p.pool_ld + c) = make_uint4(oh[0], oh[1], oh[2], oh[3]);
          *reinterpret_cast<uint4 *>(p.pool_lo + ppix * p.pool_ld + c) = make_uint4(ol[0], ol[1], ol[2], ol[3]);
        }
      }
      if (out_f32 && row_ok) {
        float *o = out_f32 + pix * p.out_f32_ld + c;
        if (full8 && ((reinterpret_cast<uintptr_t>(o) & 15) == 0)) {
          reinterpret_cast<float4 *>(o)[0] = make_float4(f[0], f[1], f[2], f[3]);
          reinterpret_cast<float4 *>(o)[1] = make_float4(f[4], f[5], f[6], f[7]);
        } else {
          for (int e = 0; e < 8 && c + e < p.Cout; ++e) o[e] = f[e];
        }
      }
    }
  }
}

// ---------------------------------------------------------------- the kernel
// one CTA = one (tile, split) unit; grid = tiles x splits. The kernel is not persistent: with 1 CTA per SM the next
// CTA's pipeline fill overlaps nothing, but programmatic dependent launch lets its prologue overlap the previous grid.
template <int BN, bool W16 = false>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                    const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
                    const TcParams p) {
  constexpr int S = num_stages(BN, W16);
  constexpr int STAGE = stage_bytes(BN, W16);
  constexpr int B_TILE_BYTES = BN * BK * 2;
  static_assert(BM * stg_ld(BN) * 4 <= S * STAGE, "staging tile must fit in the ring");
  extern __shared__ uint8_t smem_raw[];
  // 1024B alignment for SWIZZLE_128B tiles
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem + (size_t)S * STAGE);
  // bars[0..S) full, [S..2S) empty
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_base = smem_u32(bars);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };

  const int tid = threadIdx.x, lane = tid & 31;
  const int unit = (int)blockIdx.x;
  const int tile = unit / p.splitk, split = unit - tile * p.splitk;
  const int nt = tile % p.tiles_n, mt = tile / p.tiles_n;
  const int twi = mt % p.tiles_w, thi = (mt / p.tiles_w) % p.tiles_h, tni = mt / (p.tiles_w * p.tiles_h);
  const int num_kb = p.kh * p.kw * p.cblocks;
  const int kb0 = split * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);

  if (tid == 0) {
    tl_min_stamp(p.tl_min, 0);
    prefetch_tmap(&tmA_hi); prefetch_tmap(&tmA_lo); prefetch_tmap(&tmB_hi); prefetch_tmap(&tmB_lo);
    // full: one arrival (the producer's expect_tx) + the TMA bytes; empty: one arrival per consumer warp
    for (int s = 0; s < S; ++s) { mbar_init(full_bar(s), 1); mbar_init(empty_bar(s), CONS_THREADS / 32); }
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  // Programmatic dependent launch: everything above may overlap the tail of the previous kernel in the stream; no global
  // memory is touched before the previous grid has completed.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  if (tid == 0) tl_min_stamp(p.tl_min, 1);

  if (tid < 128) {
    // ===================== TMA producer (one thread) =====================
    if (tid == 0) {
      const int w_in0 = twi * p.tw * p.stride - p.pad, h_in0 = thi * p.th * p.stride - p.pad, n0 = tni * p.tn;
      const int b_row0 = nt * BN;
      for (int kb = kb0, it = 0; kb < kb1; ++kb, ++it) {
        const int s = it % S; const uint32_t ph = (uint32_t)(it / S) & 1u;
        mbar_wait(empty_bar(s), ph ^ 1u);
        const int tap = kb / p.cblocks, cb = kb - tap * p.cblocks;
        const int khi = tap / p.kw, kwi = tap - khi * p.kw;
        const uint32_t sa = smem_base + (uint32_t)s * STAGE;
        mbar_expect_tx(full_bar(s), (uint32_t)STAGE);
        tma_load_4d(sa, &tmA_hi, full_bar(s), cb * BK, w_in0 + kwi, h_in0 + khi, n0);
        tma_load_4d(sa + A_TILE_BYTES, &tmA_lo, full_bar(s), cb * BK, w_in0 + kwi, h_in0 + khi, n0);
        tma_load_2d(sa + 2 * A_TILE_BYTES, &tmB_hi, full_bar(s), kb * BK, b_row0);
        if (!W16) tma_load_2d(sa + 2 * A_TILE_BYTES + B_TILE_BYTES, &tmB_lo, full_bar(s), kb * BK, b_row0);
      }
    }
    return;
  }

  // ===================== consumers: MMA over the K range, then the epilogue =====================
  const int e = tid - 128;                     // 0..255
  const int g = e >> 7, t = e & 127;           // warpgroup, thread within it
  float acc[BN / 2];
#pragma unroll
  for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
  for (int kb = kb0, it = 0; kb < kb1; ++kb, ++it) {
    const int s = it % S; const uint32_t ph = (uint32_t)(it / S) & 1u;
    mbar_wait(full_bar(s), ph);                // TMA bytes landed
    if (it == 0 && e == 0) tl_min_stamp(p.tl_min, 2);
    const uint32_t sa = smem_base + (uint32_t)s * STAGE;
    const uint64_t a_hi = make_smem_desc(sa + (uint32_t)g * (A_TILE_BYTES / 2));
    const uint64_t a_lo = make_smem_desc(sa + A_TILE_BYTES + (uint32_t)g * (A_TILE_BYTES / 2));
    const uint64_t b_hi = make_smem_desc(sa + 2 * A_TILE_BYTES);
    const uint64_t b_lo = make_smem_desc(sa + 2 * A_TILE_BYTES + B_TILE_BYTES);
    wgmma_fence_acc(acc);
    wgmma_fence();
    mma_kblock<BN, W16>(acc, a_hi, a_lo, b_hi, b_lo, it == 0);
    wgmma_commit();
    wgmma_wait<1>();                           // the previous K block's MMAs have retired: its stage is free
    wgmma_fence_acc(acc);
    if (it > 0 && lane == 0) mbar_arrive(empty_bar((it - 1) % S));
  }
  wgmma_wait<0>();
  wgmma_fence_acc(acc);
  if (e == 0) tl_max_stamp(p.tl_max, 0);
  // every stage has been consumed by both warpgroups before the ring is overwritten by the staging tile
  consumers_sync();
  float *stg = reinterpret_cast<float *>(smem);
  stage_acc<BN>(stg, acc, g, t);
  consumers_sync();

  const int row = e & 127;                     // tile row = pixel; warp = 32 consecutive rows
  const int wl = row & (p.tw - 1), hl = (row / p.tw) & (p.th - 1), nl = row / (p.tw * p.th);
  const int wo = twi * p.tw + wl, ho = thi * p.th + hl, n = tni * p.tn + nl;
  const bool row_ok = (wo < p.Wo) && (ho < p.Ho) && (n < p.N);
  const long long pix = ((long long)n * p.Ho + ho) * p.Wo + wo;
  const long long ppix = (p.pool_hi && row_ok && !(lane & 9)) ? ((long long)n * p.Hp + (ho >> 1)) * p.Wp + (wo >> 1) : -1;
  float *const out_f32 = p.out_f32 ? p.out_f32 + (long long)split * p.split_stride : nullptr;
  epilogue_row<BN, W16>(p, stg + row * stg_ld(BN), nt, row_ok, pix, out_f32, e >> 7, ppix);
  if (e == 0) tl_max_stamp(p.tl_max, 1);
}

// ---------------------------------------------------------------- first layer: 3x3 / pad 1 / Cin = 3 / Cout = 64 on wgmma
// K = 27 cannot come through TMA (NCHW fp32 image, 3 channels), so the threads do the im2col themselves: each builds half
// of one pixel row of the 128-pixel A tile (16 of the 32 k columns), split to bf16 hi/lo and written straight into the
// K-major SWIZZLE_128B layout (row = 128 B, only k < 32 populated; the MMAs read two k16 steps), then
// fence.proxy.async. The 64 x 27 filter bank is split once per CTA into a resident B tile. Each warpgroup multiplies its
// 64 rows (N = 64, three products per k16), stages them, and the generic row epilogue (bias, ReLU, split) writes them.
constexpr int C1_THREADS = 256;
constexpr int C1_B_BYTES = 2 * 64 * 128;
constexpr int C1_SMEM = 2 * A_TILE_BYTES + C1_B_BYTES + BM * stg_ld(64) * 4 + 1024;

__global__ void __launch_bounds__(C1_THREADS, 2)
conv1_tc_kernel(const float *__restrict__ x, int N, int H, int W, const float *__restrict__ w, const TcParams p) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *sB = smem + 2 * A_TILE_BYTES;
  float *stg = reinterpret_cast<float *>(sB + C1_B_BYTES);
  const uint32_t a_base = smem_u32(smem), b_base = smem_u32(sB);
  const int tid = threadIdx.x, lane = tid & 31;
  const int g = tid >> 7, t = tid & 127;
  const int pixels = N * H * W;                        // < 2^31 (checked by the launcher): 32-bit index math throughout
  const int total_tiles = (pixels + BM - 1) / BM;
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // resident B tile: row = output channel, 128 B per row (k < 32 used), 16-byte chunk j stored at j ^ (row & 7)
  for (int i = tid; i < 64 * 4; i += C1_THREADS) {
    const int row = i >> 2, j = i & 3;
    uint32_t hh[4], ll[4];
#pragma unroll
    for (int q = 0; q < 4; ++q) {
      const int k0 = j * 8 + 2 * q;
      const float v0 = (k0 < 27) ? __ldg(w + row * 27 + k0) : 0.f, v1 = (k0 + 1 < 27) ? __ldg(w + row * 27 + k0 + 1) : 0.f;
      split_bf16x2(v0, v1, hh[q], ll[q]);
    }
    const uint32_t off = (uint32_t)row * 128u + (uint32_t)((j ^ (row & 7)) * 16);
    *reinterpret_cast<uint4 *>(sB + off) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
    *reinterpret_cast<uint4 *>(sB + 64 * 128 + off) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
  }
  const int HW = H * W;
  const int brow = tid & 127, bhalf = tid >> 7;          // builder: A row, k columns [16 bhalf, 16 bhalf + 16)
  for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
    // ---- im2col: one pixel row per thread pair, 32-bit index math
    const int pix = tile * BM + brow;
    float in[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) in[k] = 0.f;
    if (pix < pixels) {
      const int n = pix / HW, rem = pix - n * HW;
      const int ho = rem / W, wo = rem - ho * W;
      const float *x0 = x + ((size_t)n * 3 * HW + (size_t)(ho - 1) * W + (wo - 1));      // tap (kh = 0, kw = 0) of channel 0
      const bool rok[3] = {ho >= 1, true, ho + 1 < H}, cok[3] = {wo >= 1, true, wo + 1 < W};
#pragma unroll
      for (int k = 0; k < 16; ++k) {
        const int kk = 16 * bhalf + k;                   // k = (ci * 3 + r) * 3 + q
        if (kk < 27) {
          const int ci = kk / 9, r = (kk / 3) % 3, q = kk % 3;
          in[k] = (rok[r] && cok[q]) ? __ldg(x0 + ci * HW + r * W + q) : 0.f;
        }
      }
    }
    uint8_t *pa = smem + (size_t)brow * 128;
#pragma unroll
    for (int jj = 0; jj < 2; ++jj) {
      const int j = 2 * bhalf + jj;
      uint32_t hh[4], ll[4];
#pragma unroll
      for (int q = 0; q < 4; ++q) split_bf16x2(in[jj * 8 + 2 * q], in[jj * 8 + 2 * q + 1], hh[q], ll[q]);
      const int pj = (j ^ (brow & 7)) * 16;
      *reinterpret_cast<uint4 *>(pa + pj) = make_uint4(hh[0], hh[1], hh[2], hh[3]);
      *reinterpret_cast<uint4 *>(pa + A_TILE_BYTES + pj) = make_uint4(ll[0], ll[1], ll[2], ll[3]);
    }
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");      // generic-proxy stores -> visible to the tensor core
    __syncthreads();
    // ---- MMA: this warpgroup's 64 rows x 64 channels, two k16 steps
    float acc[32];
#pragma unroll
    for (int i = 0; i < 32; ++i) acc[i] = 0.f;
    const uint64_t a_hi = make_smem_desc(a_base + (uint32_t)g * (A_TILE_BYTES / 2));
    const uint64_t a_lo = make_smem_desc(a_base + A_TILE_BYTES + (uint32_t)g * (A_TILE_BYTES / 2));
    const uint64_t b_hi = make_smem_desc(b_base), b_lo = make_smem_desc(b_base + 64 * 128);
    wgmma_fence_acc(acc);
    wgmma_fence();
#pragma unroll
    for (int k = 0; k < 2; ++k) {
      const uint64_t adv = (uint64_t)((k * 16 * 2) >> 4);
      wgmma_nk16<64, false>(acc, a_lo + adv, b_hi + adv, k ? 1u : 0u);
      wgmma_nk16<64, false>(acc, a_hi + adv, b_lo + adv, 1u);
      wgmma_nk16<64, false>(acc, a_hi + adv, b_hi + adv, 1u);
    }
    wgmma_commit();
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    stage_acc<64>(stg, acc, g, t);
    __syncthreads();                                  // staging complete; both warpgroups are done reading the A tile
    // ---- epilogue: thread = (row, 32-channel half)
    const int row = tid & 127;
    const int opix = tile * BM + row;
    epilogue_row<64, false>(p, stg + row * stg_ld(64), 0, opix < pixels, (long long)opix, nullptr, tid >> 7, -1);
    __syncthreads();                                  // staging / A tile reused by the next tile
  }
  (void)lane;
}

// split-K second pass: out = epilogue(sum over splits in FIXED order) — deterministic (no atomics), so the
// row-chunk invariance the reference asserts (modules/test.lua:85-98) still holds bit for bit.
struct ReduceParams {
  const float *ws; long long split_stride; int splitk; long long pixels; int Cout;
  const float *bias; const __nv_bfloat16 *res_hi, *res_lo; long long res_ld; int relu;
  __nv_bfloat16 *out_hi, *out_lo; long long out_ld; float *out_f32; long long out_f32_ld;
  OutScatter scatter;
};
__global__ void __launch_bounds__(256) splitk_reduce_kernel(const ReduceParams r) {
  MPN_PDL_SYNC();
  const long long idx = (long long)blockIdx.x * blockDim.x + threadIdx.x;
  if (idx >= r.pixels * r.Cout) return;
  const long long pix = idx / r.Cout; const int c = (int)(idx - pix * r.Cout);
  float acc = 0.f;
  for (int s = 0; s < r.splitk; ++s) acc += r.ws[(long long)s * r.split_stride + idx];
  if (r.bias) acc += __ldg(r.bias + c);
  if (r.res_hi) acc += join_bf16(r.res_hi[pix * r.res_ld + c], r.res_lo[pix * r.res_ld + c]);
  if (r.relu) acc = fmaxf(acc, 0.f);
  if (r.out_hi) { __nv_bfloat16 h, l; split_bf16(acc, h, l); r.out_hi[pix * r.out_ld + c] = h; r.out_lo[pix * r.out_ld + c] = l; }
  if (r.scatter.n > 0) {                      // several heads in one GEMM: each column range has its own dense destination
#pragma unroll 1
    for (int g = 0; g < r.scatter.n; ++g)
      if (c >= r.scatter.seg[g].c0 && c < r.scatter.seg[g].c1) { r.scatter.seg[g].ptr[pix * r.scatter.seg[g].ld + (c - r.scatter.seg[g].c0)] = acc; break; }
  } else if (r.out_f32) r.out_f32[pix * r.out_f32_ld + c] = acc;
}

// ---------------------------------------------------------------- host: TMA descriptors
typedef CUresult (*PFN_encodeTiled)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                    const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                    CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);
PFN_encodeTiled get_encode_fn() {
  static PFN_encodeTiled fn = nullptr;
  if (!fn) {
    void *p = nullptr; cudaDriverEntryPointQueryResult q;
    if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
        q == cudaDriverEntryPointSuccess)
      fn = reinterpret_cast<PFN_encodeTiled>(p);
  }
  return fn;
}

int encode_map(mpn_ctx *ctx, CUtensorMap *tm, const void *base, int rank, const cuuint64_t *dims,
               const cuuint64_t *strides_bytes /* rank-1 */, const cuuint32_t *box, const cuuint32_t *estr) {
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return mpn_fail(ctx, MPN_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  CUresult r = fn(tm, CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void *>(base), dims,
                  strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char b[256];
    snprintf(b, sizeof b, "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu box %u %u", (int)r, rank,
             (unsigned long long)dims[0], (unsigned long long)dims[1], box[0], box[1]);
    return mpn_fail(ctx, MPN_ERR_CUDA, b);
  }
  return MPN_OK;
}

// MPN_TC_PDL=0 disables programmatic dependent launch (debug knob)
inline bool tc_use_pdl() {
  static const int on = [] { const char *e = getenv("MPN_TC_PDL"); return (e && e[0] == '0') ? 0 : 1; }();
  return on != 0;
}

template <int BN, bool W16 = false>
int launch_bn(mpn_ctx *ctx, const ConvPlan &pl, const TcParams &tp) {
  const int smem = num_stages(BN, W16) * stage_bytes(BN, W16) + 1024 /*align*/ + 256 /*barriers*/;
  constexpr int slot = W16 ? 3 : (BN == 256 ? 2 : (BN == 128 ? 1 : 0));
  if (!ctx->tc_attr_set[slot]) {     // per ctx (= per device): the attribute is per device function
    MPN_CUDA(ctx, cudaFuncSetAttribute(conv_gemm_tc_kernel<BN, W16>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    ctx->tc_attr_set[slot] = 1;
  }
  const long long units = (long long)pl.tiles_img * pl.tiles_h * pl.tiles_w * pl.tiles_n * pl.splitk;
  MPN_CHECK_ARG(ctx, units > 0 && units < (1ll << 31), "conv_tc: grid size out of range");
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)units); cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (tc_use_pdl()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr; cfg.numAttrs = na;
  MPN_CUDA(ctx, cudaLaunchKernelEx(&cfg, conv_gemm_tc_kernel<BN, W16>, pl.tmA_hi, pl.tmA_lo, pl.tmB_hi, pl.tmB_lo, tp));
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

}  // namespace

// first layer on the tensor cores (see conv1_tc_kernel); y: NHWC split planes with 64 channels
int conv1_tc_launch(mpn_ctx *ctx, const float *x_nchw, int N, int H, int W, const float *w_dev, const float *bias_dev, int relu,
                    DTensor &y) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_CONV_DIRECT);
  MPN_CHECK_ARG(ctx, y.hi && y.lo && y.C == 64 && y.ld % 8 == 0, "conv1_tc: output must be 64-channel split planes");
  TcParams tp;
  memset(&tp, 0, sizeof(tp));
  tp.N = N; tp.Ho = H; tp.Wo = W; tp.Cout = 64; tp.bias = bias_dev; tp.relu = relu;
  tp.out_hi = y.hi; tp.out_lo = y.lo; tp.out_ld = y.ld; tp.acc_scale = 1.f;
  MPN_CHECK_ARG(ctx, y.ld == 64 && (long long)N * H * W < (1ll << 31) - 256, "conv1_tc: dense 64-channel output and < 2^31 pixels");
  if (!ctx->tc_attr_set[4]) {       // per ctx (= per device): the attribute is per device function
    MPN_CUDA(ctx, cudaFuncSetAttribute(conv1_tc_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, C1_SMEM));
    ctx->tc_attr_set[4] = 1;
  }
  const long long tiles = ((long long)N * H * W + BM - 1) / BM;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)std::min<long long>(tiles, 2ll * ctx->sm_count)); cfg.blockDim = dim3(C1_THREADS);
  cfg.dynamicSmemBytes = (size_t)C1_SMEM; cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (tc_use_pdl()) { attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization; attr[na].val.programmaticStreamSerializationAllowed = 1; ++na; }
  cfg.attrs = attr; cfg.numAttrs = na;
  MPN_CUDA(ctx, cudaLaunchKernelEx(&cfg, conv1_tc_kernel, x_nchw, N, H, W, w_dev, tp));
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

double conv_flops(const ConvProblem &p) {
  const double Ho = (double)p.y.H, Wo = (double)p.y.W;
  return 2.0 * (double)p.x.C * p.Cout * p.kh * p.kw * Ho * Wo * (double)p.y.N;
}

// choose_only: stop after the (kernel, BN, split-K, patch) choice — no pointers, no TMA descriptors, no GPU
// (mpn_debug_plan: CPU tests pin the planner's choices for the BASELINE layers).
static int conv_tc_plan_impl(mpn_ctx *ctx, int sm_count, const ConvProblem &p, ConvPlan &pl, bool choose_only) {
  pl.valid = 0;
  MPN_CHECK_ARG(ctx, choose_only || (p.x.hi && p.x.lo && ((p.w_hi && p.w_lo) || p.w16)), "conv_tc: operands must be split-bf16 (or an fp16 weight plane)");
  pl.w16 = p.w16 ? 1 : 0;
  MPN_CHECK_ARG(ctx, choose_only || (p.x.fmt == 1) == (pl.w16 == 1), "conv_tc: fp16 activation planes go with the fp16 weight plane (and only with it)");
  MPN_CHECK_ARG(ctx, p.x.C % BK == 0, "conv_tc: Cin must be a multiple of 64");
  MPN_CHECK_ARG(ctx, p.x.ld % 8 == 0, "conv_tc: input pixel stride must be a multiple of 8 elements");
  MPN_CHECK_ARG(ctx, p.stride >= 1 && p.stride <= 2, "conv_tc: stride must be 1 or 2");
  const int Ho = (int)p.y.H, Wo = (int)p.y.W, N = (int)p.y.N;
  pl.flat = (p.kh == 1 && p.kw == 1 && p.stride == 1 && p.pad == 0) ? 1 : 0;
  pl.mode = 0; pl.splitk = 1;
  cuuint64_t dims[4], strides[3]; cuuint32_t box[4], estr[4];
  int gtn = 1, gth = 1, gtw = BM;                       // generic-mode patch
  if (!pl.flat) {
    // choose the power-of-two patch tn x th x tw (=128) that wastes the fewest MMA rows
    double best = -1.0;
    for (int tw = 1; tw <= 128; tw <<= 1)
      for (int th = 1; th * tw <= 128; th <<= 1) {
        const int tn = 128 / (tw * th);
        if (tw * p.stride > 256 || th * p.stride > 256) continue;
        const long long tiles = (long long)((Wo + tw - 1) / tw) * ((Ho + th - 1) / th) * ((N + tn - 1) / tn);
        const double util = (double)N * Ho * Wo / (double)(tiles * 128) + 1e-6 * tw;   // tie-break: wider rows
        if (util > best) { best = util; gtn = tn; gth = th; gtw = tw; }
      }
  }
  const long long P = (long long)p.x.N * p.x.H * p.x.W;
  // 3x3 / stride 1 / pad 1 convolutions take 16 x 8 patches (mode 1): patches start at even coordinates, so the
  // epilogue can fuse a following 2x2/2 max pool (no window straddles two tiles)
  {
    const bool r3_ok = (p.kh == 3 && p.kw == 3 && p.stride == 1 && p.pad == 1);
    const char *env3 = getenv("MPN_TC_R3");
    // experiment knob: maps with fewer output pixels than MPN_TC_R3_MINPIX keep the waste-minimising generic patch
    // (16 x 8 patches pad a 38 x 50 map by 29 %); unset = 0 = no effect
    const char *env3m = getenv("MPN_TC_R3_MINPIX");
    const long long r3_minpix = env3m ? atoll(env3m) : 0;
    pl.mode = (r3_ok && !(env3 && env3[0] == '0') && P >= r3_minpix) ? 1 : 0;
  }
  const long long tiles_m = pl.flat ? (P + BM - 1) / BM
                                    : (pl.mode ? (long long)((Wo + 7) / 8) * ((Ho + 15) / 16) * N
                                               : (long long)((Wo + gtw - 1) / gtw) * ((Ho + gth - 1) / gth) * ((N + gtn - 1) / gtn));
  // N tile: estimated cycles = rounds x (K blocks x max(MMA, operand ingest) + fixed per-tile cost), rounds =
  // ceil(units / SMs) (one CTA per SM). Per K block: the tensor pipe does 3 x 128 x BN x 64 MACs (2 for w16) at ~1024
  // bf16 MACs per cycle per SM; the operands are (128 + BN) rows x 128 B per plane.
  {
    const int taps = p.kh * p.kw;
    const double kblocks = (double)taps * (double)(p.x.C / BK);
    double best = 1e300; int best_bn = 64;
    for (int bi = 0; bi < 3; ++bi) {
      const int bn = bi == 0 ? 256 : (bi == 1 ? 128 : 64);
      if (pl.w16 && bn != 256) continue;                          // the fp16-weight kernel exists for the wide tile only
      if (!p.m_invariant && bn > 64 && bn > ((p.Cout + 63) / 64) * 64) continue;   // do not pad N by more than one 64-block
      // per-ROI layers: the N tile is a function of Cout alone, so the plan of a row never depends on the row count
      if (p.m_invariant && bn != (p.Cout > 128 ? 256 : (p.Cout > 64 ? 128 : 64))) continue;
      const long long units = tiles_m * ((p.Cout + bn - 1) / bn);
      const long long rounds = (units + sm_count - 1) / sm_count;
      const double mma = (pl.w16 ? 2.0 : 3.0) * 128.0 * bn * 64.0 / 1024.0;
      const double ingest = (pl.w16 ? 2.0 * 128 + bn : 2.0 * (128 + bn)) * 128.0 / 48.0;
      const double cost = (double)rounds * (kblocks * std::max(mma, ingest) + 1500.0 + 8.0 * bn);
      if (cost < best * 0.999) { best = cost; best_bn = bn; }
    }
    pl.BN = best_bn;
    pl.tiles_n = (p.Cout + pl.BN - 1) / pl.BN;
  }
  if (pl.flat) {
    pl.tn = 1; pl.th = 1; pl.tw = BM;
    pl.tiles_img = 1; pl.tiles_h = 1; pl.tiles_w = (int)((P + BM - 1) / BM);
    dims[0] = (cuuint64_t)p.x.C; dims[1] = (cuuint64_t)P; dims[2] = 1; dims[3] = 1;
    strides[0] = (cuuint64_t)p.x.ld * 2; strides[1] = (cuuint64_t)P * p.x.ld * 2; strides[2] = strides[1];
    box[0] = BK; box[1] = BM; box[2] = 1; box[3] = 1;
    estr[0] = estr[1] = estr[2] = estr[3] = 1;
  } else {
    if (pl.mode == 1) { pl.tn = 1; pl.th = 16; pl.tw = 8; }
    else { pl.tn = gtn; pl.th = gth; pl.tw = gtw; }
    pl.tiles_w = (Wo + pl.tw - 1) / pl.tw; pl.tiles_h = (Ho + pl.th - 1) / pl.th; pl.tiles_img = (N + pl.tn - 1) / pl.tn;
    dims[0] = (cuuint64_t)p.x.C; dims[1] = (cuuint64_t)p.x.W; dims[2] = (cuuint64_t)p.x.H; dims[3] = (cuuint64_t)p.x.N;
    strides[0] = (cuuint64_t)p.x.ld * 2; strides[1] = (cuuint64_t)p.x.W * p.x.ld * 2;
    strides[2] = (cuuint64_t)p.x.H * p.x.W * p.x.ld * 2;
    box[0] = BK; box[1] = (cuuint32_t)(pl.tw * p.stride); box[2] = (cuuint32_t)(pl.th * p.stride); box[3] = (cuuint32_t)pl.tn;
    estr[0] = 1; estr[1] = (cuuint32_t)p.stride; estr[2] = (cuuint32_t)p.stride; estr[3] = 1;
  }
  {
    // split-K for GEMMs too small to fill the machine (cls/bbox heads: a handful of tiles, 64 K blocks each,
    // latency-bound): the split count depends on K only (so results do not change with the number of rows, as long as
    // the GEMM stays small); it is either that value or 1
    const long long units = tiles_m * pl.tiles_n;
    const long long num_kb = (long long)p.kh * p.kw * (p.x.C / BK);
    long long sk = std::min<long long>(num_kb / 8, 8);
    if (p.m_invariant) { if (!(pl.flat && p.Cout <= 128) || sk < 2) sk = 1; }      // a function of (Cout, K) only
    else if (pl.mode == 1 || sk < 2 || units * sk > sm_count) sk = 1;
    const char *env2 = getenv("MPN_TC_SPLITK");
    if (env2 && env2[0] == '0') sk = 1;
    pl.splitk = (int)std::max<long long>(sk, 1);
    pl.kb_per_split = (int)((num_kb + pl.splitk - 1) / pl.splitk);
    pl.splitk = (int)((num_kb + pl.kb_per_split - 1) / pl.kb_per_split);     // no empty splits
  }
  if (choose_only) return MPN_OK;
  MPN_TRY(encode_map(ctx, &pl.tmA_hi, p.x.hi, 4, dims, strides, box, estr));
  MPN_TRY(encode_map(ctx, &pl.tmA_lo, p.x.lo, 4, dims, strides, box, estr));
  const long long Ktot = (long long)p.kh * p.kw * p.x.C;
  cuuint64_t bd[2] = {(cuuint64_t)Ktot, (cuuint64_t)p.Cout}, bs[1] = {(cuuint64_t)Ktot * 2};
  cuuint32_t bb[2] = {BK, (cuuint32_t)pl.BN}, be[2] = {1, 1};
  if (pl.w16) {
    MPN_CHECK_ARG(ctx, pl.mode == 0 && pl.flat && pl.splitk == 1 && pl.BN == 256, "conv_tc: the fp16-weight path is for wide flat GEMMs without split-K");
    MPN_TRY(encode_map(ctx, &pl.tmB_hi, p.w16, 2, bd, bs, bb, be));      // 16-bit elements: the TMA only moves bytes
    pl.tmB_lo = pl.tmB_hi;
  } else {
    MPN_TRY(encode_map(ctx, &pl.tmB_hi, p.w_hi, 2, bd, bs, bb, be));
    MPN_TRY(encode_map(ctx, &pl.tmB_lo, p.w_lo, 2, bd, bs, bb, be));
  }
  pl.valid = 1;
  return MPN_OK;
}

int conv_tc_plan(mpn_ctx *ctx, const ConvProblem &p, ConvPlan &pl) { return conv_tc_plan_impl(ctx, ctx->sm_count, p, pl, false); }

int conv_tc_launch(mpn_ctx *ctx, const ConvProblem &p, const ConvPlan &pl) {
  MpnProfScope prof_scope__(ctx, MPN_CAT_CONV_TC);
  MPN_CHECK_ARG(ctx, pl.valid, "conv_tc_launch: invalid plan");
  TcParams tp;
  memset(&tp, 0, sizeof(tp));
  if (pl.flat) { tp.N = 1; tp.Ho = 1; tp.Wo = (int)(p.y.N * p.y.H * p.y.W); }
  else { tp.N = (int)p.y.N; tp.Ho = (int)p.y.H; tp.Wo = (int)p.y.W; }
  tp.Cout = p.Cout; tp.kh = p.kh; tp.kw = p.kw; tp.stride = p.stride; tp.pad = p.pad;
  tp.cblocks = (int)(p.x.C / BK);
  tp.tn = pl.tn; tp.th = pl.th; tp.tw = pl.tw;
  tp.tiles_img = pl.tiles_img; tp.tiles_h = pl.tiles_h; tp.tiles_w = pl.tiles_w; tp.tiles_n = pl.tiles_n;
  tp.bias = p.bias;
  tp.res_hi = p.res.hi; tp.res_lo = p.res.lo; tp.res_ld = p.res.ld;
  tp.out_hi = p.y.hi; tp.out_lo = p.y.lo; tp.out_ld = p.y.ld;
  tp.out_f32 = p.y.f32; tp.out_f32_ld = p.y_f32_ld;
  tp.relu = p.relu;
  tp.splitk = pl.splitk; tp.kb_per_split = pl.kb_per_split; tp.split_stride = 0;
  tp.acc_scale = pl.w16 ? p.w16_inv_scale : 1.f;
  tp.out_fmt = p.y.fmt; tp.ovf = nullptr;
  if (p.y.fmt) MPN_TRY(mpn_ovf_flag(ctx, &tp.ovf));
  MPN_CHECK_ARG(ctx, !p.pool.hi || p.pool.fmt == p.y.fmt, "conv_tc: pooled output must share the output's plane format");
  MPN_CHECK_ARG(ctx, !(p.y.fmt && pl.splitk > 1), "conv_tc: fp16 output planes are not written by the split-K reduce");
  MPN_CHECK_ARG(ctx, !p.res.hi || p.res.fmt == 0, "conv_tc: residual inputs are bf16 split planes");
  if (ctx->tl_on && ctx->tl_n < ctx->tl_cap) { tp.tl_min = ctx->tl_min + 4 * ctx->tl_n; tp.tl_max = ctx->tl_max + 4 * ctx->tl_n; ++ctx->tl_n; }
  if (p.pool.hi) {
    // fused 2x2/2 (ceil) max pool: the 16 x 8 patches start at even coordinates, so no window straddles tiles
    MPN_CHECK_ARG(ctx, pl.mode == 1 && pl.splitk == 1 && !p.res.hi && p.Cout % 8 == 0 && p.pool.ld % 8 == 0,
                  "conv_tc: fused pooling needs the 3x3 kernel, no residual, Cout multiple of 8");
    MPN_CHECK_ARG(ctx, p.pool.H == (p.y.H + 1) / 2 && p.pool.W == (p.y.W + 1) / 2 && p.pool.N == p.y.N, "conv_tc: pooled geometry mismatch");
    tp.pool_hi = p.pool.hi; tp.pool_lo = p.pool.lo; tp.pool_ld = p.pool.ld; tp.Hp = (int)p.pool.H; tp.Wp = (int)p.pool.W;
    if (p.pool_only) { tp.out_hi = tp.out_lo = nullptr; tp.out_f32 = nullptr; }
  }
  if (p.y.hi) MPN_CHECK_ARG(ctx, p.Cout % 8 == 0 && p.y.ld % 8 == 0, "conv_tc: split output needs Cout, ld multiples of 8");
  MPN_CHECK_ARG(ctx, p.scatter.n == 0 || pl.splitk > 1, "conv_tc: scattered outputs need a split-K plan");
  if (pl.splitk > 1) {
    // partial accumulators go to a dense fp32 workspace [split][pixel][Cout]; bias/residual/ReLU/output split move to the reduce
    const long long pixels = (long long)p.y.N * p.y.H * p.y.W;
    float *ws = nullptr;
    MPN_TRY(mpn_scratch3(ctx, sizeof(float) * (size_t)pl.splitk * pixels * p.Cout, (void **)&ws));
    tp.bias = nullptr; tp.res_hi = tp.res_lo = nullptr; tp.relu = 0; tp.out_hi = tp.out_lo = nullptr;
    tp.out_f32 = ws; tp.out_f32_ld = p.Cout; tp.split_stride = pixels * p.Cout;
    const int rc = pl.BN == 256 ? launch_bn<256>(ctx, pl, tp) : (pl.BN == 128 ? launch_bn<128>(ctx, pl, tp) : launch_bn<64>(ctx, pl, tp));
    MPN_TRY(rc);
    ReduceParams r;
    r.ws = ws; r.split_stride = tp.split_stride; r.splitk = pl.splitk; r.pixels = pixels; r.Cout = p.Cout;
    r.bias = p.bias; r.res_hi = p.res.hi; r.res_lo = p.res.lo; r.res_ld = p.res.ld; r.relu = p.relu;
    r.out_hi = p.y.hi; r.out_lo = p.y.lo; r.out_ld = p.y.ld; r.out_f32 = p.y.f32; r.out_f32_ld = p.y_f32_ld;
    r.scatter = p.scatter;
    const long long total = pixels * p.Cout;
    MPN_CUDA(ctx, mpn_launch_pdl(ctx, splitk_reduce_kernel, dim3((unsigned)((total + 255) / 256)), dim3(256), 0, r));
    MPN_LAUNCHED(ctx);
    return MPN_OK;
  }
  if (pl.w16) return launch_bn<256, true>(ctx, pl, tp);
  switch (pl.BN) {
    case 256: return launch_bn<256>(ctx, pl, tp);
    case 128: return launch_bn<128>(ctx, pl, tp);
    default: return launch_bn<64>(ctx, pl, tp);
  }
}

// Host-only view of the planner (no GPU): which engine configuration conv_tc_plan would pick for a layer on a device
// with `sm_count` SMs. out[8] = {mode (bit 0: 16 x 8 patches of the 3x3 / stride 1 convolutions), CTA group (always 1),
// BN, split-K, stream-K (always 0), tn, th, tw}.
extern "C" int mpn_debug_plan(int64_t N, int64_t Cin, int64_t H, int64_t W, int64_t Cout, int32_t k, int32_t stride, int32_t pad,
                              int32_t per_roi, int32_t sm_count, int32_t *out) {
  if (!out || N <= 0 || Cin <= 0 || Cin % 64 || H <= 0 || W <= 0 || Cout <= 0 || k <= 0 || stride < 1 || stride > 2 || pad < 0 || sm_count < 2)
    return MPN_ERR_ARG;
  ConvProblem p;
  p.x.N = N; p.x.H = H; p.x.W = W; p.x.C = Cin; p.x.ld = Cin;
  p.Cout = (int)Cout; p.kh = p.kw = k; p.stride = stride; p.pad = pad; p.m_invariant = per_roi ? 1 : 0;
  p.y.N = N; p.y.H = (H + 2 * pad - k) / stride + 1; p.y.W = (W + 2 * pad - k) / stride + 1; p.y.C = Cout; p.y.ld = Cout;
  if (p.y.H <= 0 || p.y.W <= 0) return MPN_ERR_ARG;
  ConvPlan pl;
  const int rc = conv_tc_plan_impl(nullptr, sm_count, p, pl, true);
  if (rc != MPN_OK) return rc;
  out[0] = pl.mode; out[1] = 1; out[2] = pl.BN; out[3] = pl.splitk; out[4] = 0; out[5] = pl.tn; out[6] = pl.th; out[7] = pl.tw;
  return MPN_OK;
}

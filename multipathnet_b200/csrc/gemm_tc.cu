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
// 13 convs + 2 fcs, at 3 bf16 MMAs per step = 1.5x the cost of one TF32 pass. The kernel is templated on the operand
// scheme (conv_gemm.cuh: OperandScheme): BF16X3 above; FP16X2, the two fp16 products of fc6 / fc7 ("w16"); BF16X1, the
// opt-in bf16 inference numerics (option "bf16"): only the hi planes are staged (half the bytes per K block) and each
// k16 step issues ONE product A_hi*B_hi. FP8X1, the opt-in fp8 inference numerics (option "fp8"): A and B are ONE e4m3
// plane each (fp8_e4m3.cuh), staged as 64-byte rows (a K block is still 64 elements, so Cin = 64 layers need no special
// case) in 64B-swizzled tiles; each k32 step issues one e4m3 product. The tensor pipe's fp8 accumulation keeps fewer
// bits than fp32 (measured on an H100: 1.5e-4 normwise when two k32 steps share a fragment, 3-7e-5 with one), so every
// k32 product goes to a zeroed fragment that is then added to the fp32 accumulator (promotion interval 32 MACs); that
// second fragment is why FP8X1 tiles are at most 128 channels wide. The
// epilogue multiplies by 2^-(e_a[sample] + e_w[channel]), exact. The epilogue and the output formats are the same in
// every scheme.
//
// Kernel shape (output tiles of 128 pixels x BN channels, persistent CTAs, warp-specialised, 3 warpgroups):
//   warpgroup 0    : TMA producer (one thread) — per K block of each of the CTA's tiles: A tile (128 pixels x 64 ch, hi+lo) by a 4-D tiled
//                    tensor map over the NHWC activation whose box is a tn x th x tw pixel patch shifted by the filter
//                    tap (zero OOB fill = conv padding, and the channels of a tap's last K block beyond Cin; elementStrides = conv
//                    stride), B tile (BN x 64, hi+lo) from the [Cout][kh*kw*conv_k_pad(Cin)] weights, into a ring of S
//                    stages (full / empty mbarriers).
//                    A stage holds a whole K block (128-byte rows) or half of one (64-byte rows; see row_bytes).
//   warpgroups 1-2 : consumers — each owns 64 rows of the tile: wgmma m64nBNk16 straight from the swizzled smem
//                    tiles into registers; then the epilogue on the fragments (tile_epilogue): + bias (+ residual)
//                    (ReLU), re-split to hi/lo (NHWC, next layer's A operand; through a per-warp shared buffer) and/or
//                    fp32, optional fused 2x2/2 max pool, while the producer already loads the next tile.
#include "conv_gemm.cuh"
#include "wgmma.cuh"
#include "fp8_e4m3.cuh"
#include <algorithm>
#include <stdlib.h>
#include <string.h>

namespace {

constexpr int BM = 128;          // pixels per tile (two m64 warpgroup MMAs)
constexpr int BK = 64;           // elements per K block (a tap's last block is zero beyond Cin: see conv_k_pad)
constexpr int TC_THREADS = 384;  // producer warpgroup + two consumer warpgroups
constexpr int CONS_THREADS = 256;
constexpr int A_TILE_BYTES = BM * BK * 2;   // first-layer kernel: 16 KB per plane (128-byte rows)
constexpr int SMEM_BUDGET = 196608;         // pipeline ring; the epilogue staging tile reuses it

// operand planes staged per ring stage: FP16X2 has one (fp16) B plane, BF16X1 one A and one B plane (the hi planes), FP8X1
// one A and one B plane of 1-byte elements
__host__ __device__ constexpr int a_planes(OperandScheme ops) { return (ops == OperandScheme::BF16X1 || ops == OperandScheme::FP8X1) ? 1 : 2; }
__host__ __device__ constexpr int b_planes(OperandScheme ops) { return ops == OperandScheme::BF16X3 ? 2 : 1; }
__host__ __device__ constexpr int elem_bytes(OperandScheme ops) { return ops == OperandScheme::FP8X1 ? 1 : 2; }
// Bytes per row of a staged operand tile: 64 (one 64B swizzle row) or 128 (one 128B swizzle row). FP8X1 rows are a whole
// K block of e4m3. The 256-wide 16-bit tiles stage half a K block (32 elements) per ring stage: that doubles their ring
// depth at the same bytes in flight, so the TMA of a stage starts while the MMAs of the stages before it still run (with
// whole-K-block stages the BN = 256 bf16x3 ring had room for two 96 KB stages); on an H100 this makes conv3 / conv4 of
// VGG-16 1.2-1.5x faster. The narrower 16-bit tiles keep whole-K-block (128-byte) rows: they are bound by operand
// ingest, not by ring depth, and half stages (which halve the bytes per TMA row) made them 5-20 % slower.
__host__ __device__ constexpr int row_bytes(int BN, OperandScheme ops) { return (ops == OperandScheme::FP8X1 || BN == 256) ? 64 : 128; }
__host__ __device__ constexpr int stage_k(int BN, OperandScheme ops) { return row_bytes(BN, ops) / elem_bytes(ops); }
__host__ __device__ constexpr int kb_steps(int BN, OperandScheme ops) { return BK / stage_k(BN, ops); }   // ring stages per K block
__host__ __device__ constexpr int a_tile_bytes(int BN, OperandScheme ops) { return BM * row_bytes(BN, ops); }
__host__ __device__ constexpr int stage_bytes(int BN, OperandScheme ops = OperandScheme::BF16X3) {
  return (a_planes(ops) * BM + b_planes(ops) * BN) * row_bytes(BN, ops);
}
// up to 4 stages of 128-byte rows, 8 of 64-byte rows
__host__ __device__ constexpr int max_stages(int BN, OperandScheme ops) { return row_bytes(BN, ops) == 64 ? 8 : 4; }
__host__ __device__ constexpr int num_stages(int BN, OperandScheme ops = OperandScheme::BF16X3) {
  return (SMEM_BUDGET / stage_bytes(BN, ops)) > max_stages(BN, ops) ? max_stages(BN, ops) : (SMEM_BUDGET / stage_bytes(BN, ops));
}
// the epilogue's own shared memory, beside the ring: per consumer warp one 16-row x 64-channel plane chunk (2 KB)
constexpr int EPI_WARP_BYTES = 16 * 128;
constexpr int EPI_BYTES = (CONS_THREADS / 32) * EPI_WARP_BYTES;
__host__ __device__ constexpr int tc_smem_bytes(int BN, OperandScheme ops) {
  return num_stages(BN, ops) * stage_bytes(BN, ops) + EPI_BYTES + 1024 /*align*/ + 256 /*barriers*/;
}

struct TcParams {
  int N, Ho, Wo, Cout;           // output geometry (flat mode: N=1, Ho=1, Wo=pixels)
  int kh, kw, stride, pad_h, pad_w;
  int cblocks;                   // K blocks per tap: ceil(Cin / 64)
  int tn, th, tw;                // tile decomposition (powers of two)
  int tiles_img, tiles_h, tiles_w, tiles_n;
  int units;                     // tiles x splits; CTA b runs units b, b + gridDim.x, ...
  const float *bias;
  const __nv_bfloat16 *res_hi, *res_lo; long long res_ld;
  __nv_bfloat16 *out_hi, *out_lo; long long out_ld;
  float *out_f32; long long out_f32_ld;
  __nv_bfloat16 *pool_hi, *pool_lo; long long pool_ld; int Hp, Wp;   // fused 2x2/2 max pool of the output (16 x 8 patches only)
  int relu;
  int splitk, kb_per_split;      // split-K: unit = (tile, split); each split owns kb_per_split K blocks and writes raw fp32 partials
  long long split_stride;        // elements between the partial planes of consecutive splits (out_f32 is the workspace then)
  unsigned long long *tl_min, *tl_max;   // diagnostics: %globaltimer stamps of this launch (4 + 4 u64) or null
  float acc_scale;               // FP16X2 kernels: accumulator * acc_scale (= 1 / the weight plane's power-of-two scale) before the bias; 1 otherwise
  int out_fmt;                   // plane format of out_hi / out_lo (and the pooled output): 0 = bf16 split, 1 = fp16 split
  unsigned *ovf;                 // fp16-overflow flag of the ctx (out_fmt == 1)
  // FP8X1 kernels: accumulator * 2^-(a_exp[pixel / sample_pix] + b_exp[channel]) before the bias
  const int *a_exp, *b_exp; long long sample_pix;
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

// K-major, 64B-swizzled tile of 64-byte rows (64 e4m3 or 32 bf16 / fp16 per row): SBO = 8 rows x 64 B, layout SWIZZLE_64B = 2
__device__ __forceinline__ uint64_t make_smem_desc_64b(uint32_t saddr) {
  uint64_t d = 0;
  d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
  d |= (uint64_t)1 << 16;
  d |= (uint64_t)(512 >> 4) << 32;
  d |= (uint64_t)2 << 62;
  return d;
}

// one ring stage (a K block or half of one: 4 or 2 x k16) of a 64-row warpgroup slice: three bf16 products per k16 (A_lo x B_hi,
// A_hi x B_lo, A_hi x B_hi; BF16X3), two fp16 products (A_lo x W16, A_hi x W16; b_hi holds the single fp16 weight plane;
// FP16X2), or one bf16 product (A_hi x B_hi; BF16X1, a_lo / b_lo unused). first: zero-init.
template <int BN, OperandScheme OPS>
__device__ __forceinline__ void mma_kstep(float (&acc)[BN / 2], uint64_t a_hi, uint64_t a_lo, uint64_t b_hi, uint64_t b_lo, bool first) {
  constexpr bool F16 = (OPS == OperandScheme::FP16X2);
#pragma unroll
  for (int k = 0; k < stage_k(BN, OPS) / 16; ++k) {
    const uint64_t adv = (uint64_t)((k * 16 * 2) >> 4);     // +32B per k16 inside the swizzle atom
    const uint32_t later = (first && k == 0) ? 0u : 1u;
    if constexpr (OPS == OperandScheme::BF16X1) {
      wgmma_nk16<BN, false>(acc, a_hi + adv, b_hi + adv, later);
    } else {
      wgmma_nk16<BN, F16>(acc, a_lo + adv, b_hi + adv, later);
      if (!F16) wgmma_nk16<BN, F16>(acc, a_hi + adv, b_lo + adv, 1u);
      wgmma_nk16<BN, F16>(acc, a_hi + adv, b_hi + adv, 1u);
    }
  }
}

// ---------------------------------------------------------------- epilogue on the accumulator fragments
// a (tile, split) unit: N tile, patch coordinates, split
struct UnitPos { int nt, twi, thi, tni, split; };
__device__ __forceinline__ UnitPos unit_pos(const TcParams &p, int unit) {
  UnitPos u;
  const int tile = unit / p.splitk;
  u.split = unit - tile * p.splitk;
  u.nt = tile % p.tiles_n;
  const int mt = tile / p.tiles_n;
  u.twi = mt % p.tiles_w; u.thi = (mt / p.tiles_w) % p.tiles_h; u.tni = mt / (p.tiles_w * p.tiles_h);
  return u;
}
// pixel of tile row `row` (tile rows = the tn x th x tw patch, w fastest); ok = inside the output; whn = (wo, ho, n)
__device__ __forceinline__ long long row_pixel(const TcParams &p, const UnitPos &u, int row, bool &ok, int *whn = nullptr) {
  const int lw = __ffs(p.tw) - 1, lh = __ffs(p.th) - 1;      // tw, th are powers of two
  const int wl = row & (p.tw - 1), hl = (row >> lw) & (p.th - 1), nl = row >> (lw + lh);
  const int wo = u.twi * p.tw + wl, ho = u.thi * p.th + hl, n = u.tni * p.tn + nl;
  ok = (wo < p.Wo) && (ho < p.Ho) && (n < p.N);
  if (whn) { whn[0] = wo; whn[1] = ho; whn[2] = n; }
  return ((long long)n * p.Ho + ho) * p.Wo + wo;
}

// One 64-channel plane chunk of a warp's 16 tile rows: the fragment's packed channel pairs v[j] (row lane / 4, channels
// 8 j + 2 (lane % 4) + {0, 1}) and v[8 + j] (row lane / 4 + 8) -> the warp's XOR-swizzled 2 KB shared buffer -> 16-byte
// chunks in address order, so every warp store covers four whole 128-byte rows. Store row 4 q + lane / 8 (tile row
// rbase + 4 q + lane / 8) goes to out + pixel * ld + col0 (nothing outside the output or where the 8 channels lie past
// Cout; Cout is a multiple of 8).
__device__ __forceinline__ void store_plane_chunk(uint32_t so, const uint32_t (&v)[16], __nv_bfloat16 *out, long long ld,
                                                  const TcParams &p, const UnitPos &u, int rbase, int col0, int lane) {
  const int r = lane >> 2;
  const uint32_t wr = so + (uint32_t)(r * 128 + 4 * (lane & 3));
  __syncwarp();                                        // the warp's reads of the previous chunk are done
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t a = wr + (uint32_t)((j ^ r) * 16);
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v[j]) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + 8 * 128), "r"(v[8 + j]) : "memory");
  }
  __syncwarp();
  const int row0 = lane >> 3, ch = lane & 7;           // rows row0 + 4 q: 8 lanes per 128-byte row
  const uint32_t rd0 = so + (uint32_t)(row0 * 128 + ((ch ^ row0) * 16)), rd1 = so + (uint32_t)(row0 * 128 + ((ch ^ row0 ^ 4) * 16));
  const bool col_ok = col0 + 8 * ch < p.Cout;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 d;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(d.x), "=r"(d.y), "=r"(d.z), "=r"(d.w)
                 : "r"(((q & 1) ? rd1 : rd0) + (uint32_t)(q * 4 * 128)) : "memory");
    bool ok;
    const long long pix = row_pixel(p, u, rbase + 4 * q + row0, ok);
    if (ok && col_ok) *reinterpret_cast<uint4 *>(out + pix * ld + col0 + 8 * ch) = d;
  }
}

// The epilogue of one tile, run by each consumer warp on its 16 rows straight from the accumulator fragment, 64 channels
// at a time: x acc_scale (FP16X2) or x 2^-(e_a + e_w) (FP8X1), + bias, + residual (hi + lo), ReLU, then the split planes
// (through the warp's shared buffer), the fused 2x2/2 max pool and / or fp32 (split-K partials, heads; stored directly).
// Fragment rows: this thread holds tile rows 64 g + 16 wq + lane / 4 + 8 i (i = 0, 1), channels 8 j + 2 (lane % 4) + {0, 1}.
template <int BN, OperandScheme OPS>
__device__ __forceinline__ void tile_epilogue(const TcParams &p, const UnitPos &u, float (&acc)[BN / 2], int g, int wq,
                                              int lane, uint32_t so) {
  const int rbase = 64 * g + 16 * wq;                // the warp's first tile row
  const int c0 = 2 * (lane & 3);
  bool fok[2]; long long fpix[2];                    // the fragment rows
#pragma unroll
  for (int i = 0; i < 2; ++i) fpix[i] = row_pixel(p, u, rbase + (lane >> 2) + 8 * i, fok[i]);
  int ea[2] = {0, 0};
  if constexpr (OPS == OperandScheme::FP8X1) {
#pragma unroll
    for (int i = 0; i < 2; ++i) ea[i] = fok[i] ? __ldg(p.a_exp + fpix[i] / p.sample_pix) : 0;
  }
  // fused 2x2/2 max pool (mode 1, 16 x 8 patches): fragment rows i = 0, 1 are image rows h (even) and h + 1 at w = lane / 4,
  // so a window is the thread's two rows and those of lane ^ 4; lanes with even w hold the result. Pooled row pr = lane / 8
  // of the warp is the window whose top-left pixel is tile row rbase + 2 pr.
  const bool pool = (p.pool_hi != nullptr);
  bool pok = false; long long ppix = 0;
  if (pool) {
    int whn[3];
    row_pixel(p, u, rbase + 2 * (lane >> 3), pok, whn);
    ppix = ((long long)whn[2] * p.Hp + (whn[1] >> 1)) * p.Wp + (whn[0] >> 1);
  }
  float *const out_f32 = p.out_f32 ? p.out_f32 + (long long)u.split * p.split_stride : nullptr;
  // The chunk body is emitted once (not unrolled over the chunks): unrolled, the 256-wide kernels were 160 KB of code
  // (three times the 64-wide ones) and their epilogue took 30-34 us per tile on an H100 against 11-16 us with one body,
  // most likely instruction-cache misses. The chunk being finished is always acc[0, 32): after each chunk the
  // accumulators move down by 32 registers.
#pragma unroll 1
  for (int m = 0; m < BN / 64; ++m) {
    const int col0 = u.nt * BN + 64 * m;
    if (col0 >= p.Cout) break;
    float *f = acc;                                  // f[4 j + 2 i + {0, 1}] = row i, channels 8 j + c0 + {0, 1}
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const int c = col0 + 8 * j + c0;
      const bool full8 = col0 + 8 * j + 8 <= p.Cout;
      float b[2] = {0.f, 0.f};
      int eb[2] = {0, 0};
#pragma unroll
      for (int k = 0; k < 2; ++k) {
        if (p.bias && c + k < p.Cout) b[k] = __ldg(p.bias + c + k);
        if constexpr (OPS == OperandScheme::FP8X1) eb[k] = __ldg(p.b_exp + c + k);
      }
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        float &f0 = f[4 * j + 2 * i], &f1 = f[4 * j + 2 * i + 1];
        if constexpr (OPS == OperandScheme::FP16X2) { f0 *= p.acc_scale; f1 *= p.acc_scale; }   // the weight plane's power-of-two scale (exact)
        if constexpr (OPS == OperandScheme::FP8X1) {   // both operands' power-of-two scales (exact): sample's and channel's
          f0 *= mpn_fp8::pow2(-(ea[i] + eb[0])); f1 *= mpn_fp8::pow2(-(ea[i] + eb[1]));
        }
        if (p.bias) {
          if (c < p.Cout) f0 += b[0];
          if (c + 1 < p.Cout) f1 += b[1];
        }
        if (p.res_hi && full8 && fok[i]) {
          const float2 x = bf16x2_to_float2(*reinterpret_cast<const uint32_t *>(p.res_hi + fpix[i] * p.res_ld + c));
          const float2 y = bf16x2_to_float2(*reinterpret_cast<const uint32_t *>(p.res_lo + fpix[i] * p.res_ld + c));
          f0 += x.x + y.x; f1 += x.y + y.y;
        }
        if (p.relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
        if (out_f32 && fok[i]) {
          float *o = out_f32 + fpix[i] * p.out_f32_ld + c;
          if (c < p.Cout) o[0] = f0;
          if (c + 1 < p.Cout) o[1] = f1;
        }
      }
    }
    // pooled chunk: mx[2 j + k] = channel 8 j + c0 + k of pooled row lane / 8 (valid on lanes with even w), in the order
    // max(max(top-left, top-right), max(bottom-left, bottom-right)); rows outside the image are -inf (ceil-mode borders)
    float mx[16];
    if (pool) {
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int k = 0; k < 2; ++k) {
          float top = fok[0] ? f[4 * j + k] : -INFINITY, bot = fok[1] ? f[4 * j + 2 + k] : -INFINITY;
          top = fmaxf(top, __shfl_xor_sync(0xffffffffu, top, 4));
          bot = fmaxf(bot, __shfl_xor_sync(0xffffffffu, bot, 4));
          mx[2 * j + k] = fmaxf(top, bot);
        }
    }
#pragma unroll 1
    for (int plane = 0; plane < 2; ++plane) {        // the split is recomputed per plane: 16 fewer live registers
      if (p.out_hi) {
        uint32_t v[16];
#pragma unroll
        for (int j = 0; j < 8; ++j)
#pragma unroll
          for (int i = 0; i < 2; ++i) {
            uint32_t hi2 = 0, lo2 = 0;
            if (fok[i]) split_x2(p.out_fmt, f[4 * j + 2 * i], f[4 * j + 2 * i + 1], hi2, lo2, p.ovf);   // packed cvt.rn.{bf16x2,f16x2}.f32
            v[8 * i + j] = plane ? lo2 : hi2;
          }
        store_plane_chunk(so, v, plane ? p.out_lo : p.out_hi, p.out_ld, p, u, rbase, col0, lane);
      }
      if (pool) {
        // pooled rows 0..3 of the buffer (lanes with even w write), then one 16-byte chunk per lane
        const int pr = lane >> 3;
        __syncwarp();
        if (!(lane & 4) && fok[0]) {
#pragma unroll
          for (int j = 0; j < 8; ++j) {
            uint32_t hi2, lo2;
            split_x2(p.out_fmt, mx[2 * j], mx[2 * j + 1], hi2, lo2, p.ovf);
            const uint32_t a = so + (uint32_t)(pr * 128 + ((j ^ pr) * 16) + 4 * (lane & 3));
            asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(plane ? lo2 : hi2) : "memory");
          }
        }
        __syncwarp();
        const int ch = lane & 7;
        uint4 d;
        asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(d.x), "=r"(d.y), "=r"(d.z), "=r"(d.w)
                     : "r"(so + (uint32_t)(pr * 128 + ((ch ^ pr) * 16))) : "memory");
        if (pok && col0 + 8 * ch < p.Cout)
          *reinterpret_cast<uint4 *>((plane ? p.pool_lo : p.pool_hi) + ppix * p.pool_ld + col0 + 8 * ch) = d;
      }
    }
#pragma unroll
    for (int k = 0; k + 32 < BN / 2; ++k) acc[k] = acc[k + 32];   // the next chunk to acc[0, 32)
  }
}

// ---------------------------------------------------------------- the kernel
// Persistent: CTA b runs the (tile, split) units b, b + gridDim.x, ... in order (grid = min(units, SMs)). The producer
// walks the K blocks of its units without stopping; the ring counter and the barrier phases carry across tiles, so
// while the consumers finish tile i from their registers, the first stages of tile i + 1 are already landing.
// Programmatic dependent launch lets the prologue overlap the previous grid.
template <int BN, OperandScheme OPS = OperandScheme::BF16X3>
__global__ void __launch_bounds__(TC_THREADS, 1)
conv_gemm_tc_kernel(const __grid_constant__ CUtensorMap tmA_hi, const __grid_constant__ CUtensorMap tmA_lo,
                    const __grid_constant__ CUtensorMap tmB_hi, const __grid_constant__ CUtensorMap tmB_lo,
                    const TcParams p) {
  constexpr int S = num_stages(BN, OPS);
  constexpr int STAGE = stage_bytes(BN, OPS);
  constexpr int A_TILE = a_tile_bytes(BN, OPS);
  constexpr int B_TILE_BYTES = BN * row_bytes(BN, OPS);
  constexpr int B_OFF = a_planes(OPS) * A_TILE;            // stage layout: A_hi [A_lo] B_hi [B_lo]
  constexpr int KSTEPS = kb_steps(BN, OPS);
  static_assert(S >= 2 && 2 * S * 8 <= 256, "ring depth: at least two stages, barriers in their 256 bytes");
  extern __shared__ uint8_t smem_raw[];
  // 1024B alignment for SWIZZLE_128B tiles; layout: ring | epilogue buffers | barriers
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint64_t *bars = reinterpret_cast<uint64_t *>(smem + (size_t)S * STAGE + EPI_BYTES);
  // bars[0..S) full, [S..2S) empty
  const uint32_t smem_base = smem_u32(smem);
  const uint32_t bar_base = smem_u32(bars);
  auto full_bar = [&](int s) { return bar_base + 8u * s; };
  auto empty_bar = [&](int s) { return bar_base + 8u * (S + s); };

  const int tid = threadIdx.x, lane = tid & 31;
  const int num_kb = p.kh * p.kw * p.cblocks;

  if (tid == 0) {
    tl_min_stamp(p.tl_min, 0);
    if (a_planes(OPS) == 1) { prefetch_tmap(&tmA_hi); prefetch_tmap(&tmB_hi); }     // the lo maps are never read
    else { prefetch_tmap(&tmA_hi); prefetch_tmap(&tmA_lo); prefetch_tmap(&tmB_hi); prefetch_tmap(&tmB_lo); }
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

  // Registers move from the producer warpgroup to the consumers, which hold up to 128 accumulators per thread across
  // the epilogue (128 x 24 + 256 x 240 <= 64K).
  if (tid < 128) {
    // ===================== TMA producer (one thread) =====================
    asm volatile("setmaxnreg.dec.sync.aligned.u32 24;" ::: "memory");
    if (tid == 0) {
      int it = 0;                                    // ring counter, carried across the CTA's units
      for (int unit = (int)blockIdx.x; unit < p.units; unit += (int)gridDim.x) {
        const UnitPos u = unit_pos(p, unit);
        const int kb0 = u.split * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);
        const int w_in0 = u.twi * p.tw * p.stride - p.pad_w, h_in0 = u.thi * p.th * p.stride - p.pad_h, n0 = u.tni * p.tn;
        const int b_row0 = u.nt * BN;
        for (int kb = kb0; kb < kb1; ++kb) {
          const int tap = kb / p.cblocks, cb = kb - tap * p.cblocks;
          const int khi = tap / p.kw, kwi = tap - khi * p.kw;
#pragma unroll
          for (int h = 0; h < KSTEPS; ++h, ++it) {    // stage = elements [h * stage_k, (h + 1) * stage_k) of the K block
            const int s = it % S; const uint32_t ph = (uint32_t)(it / S) & 1u;
            const int ka = cb * BK + h * stage_k(BN, OPS), kk = kb * BK + h * stage_k(BN, OPS);
            mbar_wait(empty_bar(s), ph ^ 1u);
            const uint32_t sa = smem_base + (uint32_t)s * STAGE;
            mbar_expect_tx(full_bar(s), (uint32_t)STAGE);
            tma_load_4d(sa, &tmA_hi, full_bar(s), ka, w_in0 + kwi, h_in0 + khi, n0);
            if (a_planes(OPS) == 2) tma_load_4d(sa + A_TILE, &tmA_lo, full_bar(s), ka, w_in0 + kwi, h_in0 + khi, n0);
            tma_load_2d(sa + B_OFF, &tmB_hi, full_bar(s), kk, b_row0);
            if (b_planes(OPS) == 2) tma_load_2d(sa + B_OFF + B_TILE_BYTES, &tmB_lo, full_bar(s), kk, b_row0);
          }
        }
      }
    }
    return;
  }

  // ===================== consumers: per unit, MMA over its K range, then the epilogue =====================
  asm volatile("setmaxnreg.inc.sync.aligned.u32 240;" ::: "memory");
  const int e = tid - 128;                     // 0..255
  const int g = e >> 7, wq = (e >> 5) & 3;     // warpgroup, warp within it
  const uint32_t so = smem_base + (uint32_t)(S * STAGE + (e >> 5) * EPI_WARP_BYTES);   // this warp's epilogue buffer
  int it = 0;                                  // ring counter, carried across the CTA's units
  for (int unit = (int)blockIdx.x; unit < p.units; unit += (int)gridDim.x) {
    const UnitPos u = unit_pos(p, unit);
    const int kb0 = u.split * p.kb_per_split, kb1 = min(num_kb, kb0 + p.kb_per_split);
    float acc[BN / 2];
#pragma unroll
    for (int i = 0; i < BN / 2; ++i) acc[i] = 0.f;
    if constexpr (OPS == OperandScheme::FP8X1) {
      // promotion: every k32 product goes to a zeroed fragment, which is added to the fp32 accumulator once it has retired
      float part[BN / 2];
#pragma unroll
      for (int i = 0; i < BN / 2; ++i) part[i] = 0.f;
      for (int kb = kb0; kb < kb1; ++kb, ++it) {
        const int s = it % S; const uint32_t ph = (uint32_t)(it / S) & 1u;
        mbar_wait(full_bar(s), ph);
        if (it == 0 && e == 0) tl_min_stamp(p.tl_min, 2);
        const uint32_t sa = smem_base + (uint32_t)s * STAGE;
        const uint64_t a8 = make_smem_desc_64b(sa + (uint32_t)g * (A_TILE / 2));
        const uint64_t b8 = make_smem_desc_64b(sa + B_OFF);
#pragma unroll
        for (int k = 0; k < BK / 32; ++k) {                 // +32B per k32 inside the 64B swizzle atom
          wgmma_fence_acc(part);
          wgmma_fence();
          wgmma_e4m3_nk32<BN>(part, a8 + (uint64_t)(2 * k), b8 + (uint64_t)(2 * k), 0u);
          wgmma_commit();
          wgmma_wait<0>();
          wgmma_fence_acc(part);
#pragma unroll
          for (int i = 0; i < BN / 2; ++i) acc[i] += part[i];
        }
        if (lane == 0) mbar_arrive(empty_bar(s));
      }
    } else {
      const int steps = (kb1 - kb0) * KSTEPS;
      for (int i = 0; i < steps; ++i, ++it) {
        const int s = it % S; const uint32_t ph = (uint32_t)(it / S) & 1u;
        mbar_wait(full_bar(s), ph);              // TMA bytes landed
        if (it == 0 && e == 0) tl_min_stamp(p.tl_min, 2);
        const uint32_t sa = smem_base + (uint32_t)s * STAGE;
        auto desc = [](uint32_t a) { return row_bytes(BN, OPS) == 64 ? make_smem_desc_64b(a) : make_smem_desc(a); };
        const uint64_t a_hi = desc(sa + (uint32_t)g * (A_TILE / 2));
        const uint64_t a_lo = desc(sa + A_TILE + (uint32_t)g * (A_TILE / 2));
        const uint64_t b_hi = desc(sa + B_OFF);
        const uint64_t b_lo = desc(sa + B_OFF + B_TILE_BYTES);
        wgmma_fence_acc(acc);
        wgmma_fence();
        mma_kstep<BN, OPS>(acc, a_hi, a_lo, b_hi, b_lo, i == 0);
        wgmma_commit();
        wgmma_wait<1>();                         // the previous stage's MMAs have retired: it is free
        wgmma_fence_acc(acc);
        if (i > 0 && lane == 0) mbar_arrive(empty_bar((it - 1) % S));
      }
      wgmma_wait<0>();
      wgmma_fence_acc(acc);
      if (lane == 0) mbar_arrive(empty_bar((it - 1) % S));   // the unit's last stage
    }
    if (e == 0) tl_max_stamp(p.tl_max, 0);
    const uint32_t t_epi = (p.tl_max && e == 0) ? (uint32_t)gtimer() : 0u;     // a tile's epilogue is far below 2^32 ns
    tile_epilogue<BN, OPS>(p, u, acc, g, wq, lane, so);
    if (e == 0) {
      tl_max_stamp(p.tl_max, 1);
      if (p.tl_max) atomicAdd(p.tl_max + 3, (unsigned long long)((uint32_t)gtimer() - t_epi));
    }
  }
}


// ---------------------------------------------------------------- first layer: 3x3 / pad 1 / Cin = 3 / Cout = 64 on wgmma
// K = 27 cannot come through TMA (NCHW fp32 image, 3 channels), so the threads do the im2col themselves: each builds half
// of one pixel row of the 128-pixel A tile (16 of the 32 k columns), split to bf16 hi/lo and written straight into the
// K-major SWIZZLE_128B layout (row = 128 B, only k < 32 populated; the MMAs read two k16 steps), then
// fence.proxy.async. The 64 x 27 filter bank is split once per CTA into a resident B tile. Each warpgroup multiplies its
// 64 rows (N = 64, three products per k16).
//
// The layer is bound by its output (64 channels x hi + lo bf16 = 256 B per pixel against 12 B of input), so the kernel is
// built around the stores. CTAs are persistent over flat 128-pixel tiles and overlap the tile stages:
//   - the A tile is double-buffered, so one barrier per tile suffices and a warpgroup may build tile i + 1 while the
//     other still multiplies tile i;
//   - the image taps of tile i + 1 are loaded into registers right after tile i's A tile is built, and are in flight
//     while tile i multiplies and stores;
//   - the epilogue runs on the accumulator fragments (+ bias, ReLU, split: the arithmetic of tile_epilogue) and is
//     warp-private: a warp owns 16 whole pixel rows of the wgmma fragment, passes each plane through a 2 KB
//     XOR-swizzled shared buffer, and writes it back as 16-byte chunks in address order, so every warp store covers
//     four whole 128-byte lines.
constexpr int C1_THREADS = 256;
constexpr int C1_A_BYTES = 2 * A_TILE_BYTES;                 // one A tile, hi + lo planes
constexpr int C1_B_BYTES = 2 * 64 * 128;
constexpr int C1_OUT_WARP = 16 * 128;                        // a warp's 16 pixel rows of one output plane
constexpr int C1_SMEM = 2 * C1_A_BYTES + C1_B_BYTES + (C1_THREADS / 32) * C1_OUT_WARP + 1024;

// the 16 image taps k = 16 bhalf + [0, 16) of pixel pix (k = (ci * 3 + r) * 3 + q; zero padding and k >= 27 are 0)
__device__ __forceinline__ void conv1_gather(const float *__restrict__ x, int pix, int pixels, int H, int W, int bhalf,
                                             float (&in)[16]) {
#pragma unroll
  for (int k = 0; k < 16; ++k) in[k] = 0.f;
  if (pix < pixels) {
    const int HW = H * W;
    const int n = pix / HW, rem = pix - n * HW;
    const int ho = rem / W, wo = rem - ho * W;
    const float *x0 = x + ((size_t)n * 3 * HW + (size_t)(ho - 1) * W + (wo - 1));      // tap (kh = 0, kw = 0) of channel 0
    const bool rok[3] = {ho >= 1, true, ho + 1 < H}, cok[3] = {wo >= 1, true, wo + 1 < W};
#pragma unroll
    for (int k = 0; k < 16; ++k) {
      const int kk = 16 * bhalf + k;
      if (kk < 27) {
        const int ci = kk / 9, r = (kk / 3) % 3, q = kk % 3;
        in[k] = (rok[r] && cok[q]) ? __ldg(x0 + ci * HW + r * W + q) : 0.f;
      }
    }
  }
}

// one output plane of a warp's 16 pixel rows: the fragment's packed channel pairs v[j] (row lane / 4, chunk j) and
// v[8 + j] (row lane / 4 + 8) -> swizzled shared rows -> 16-byte chunks in address order (4 whole lines per store)
// (so: 32-bit shared address of the warp's buffer)
__device__ __forceinline__ void conv1_store_plane(uint32_t so, const uint32_t (&v)[16], __nv_bfloat16 *out, int pix0,
                                                  int pixels, int lane) {
  const int r = lane >> 2;
  const uint32_t wr = so + (uint32_t)(r * 128 + 4 * (lane & 3));
  __syncwarp();                                        // the warp's reads of the previous plane are done
#pragma unroll
  for (int j = 0; j < 8; ++j) {
    const uint32_t a = wr + (uint32_t)((j ^ r) * 16);
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a), "r"(v[j]) : "memory");
    asm volatile("st.shared.b32 [%0], %1;" ::"r"(a + 8 * 128), "r"(v[8 + j]) : "memory");
  }
  __syncwarp();
  const int row0 = lane >> 3, ch = lane & 7;           // rows row0 + 4 q: 8 lanes per 128-byte row
  // row row0 + 4 q has (row & 7) = row0 ^ 4 (q & 1)
  const uint32_t rd0 = so + (uint32_t)(row0 * 128 + ((ch ^ row0) * 16)), rd1 = so + (uint32_t)(row0 * 128 + ((ch ^ row0 ^ 4) * 16));
  __nv_bfloat16 *o = out + (size_t)(pix0 + row0) * 64 + ch * 8;
#pragma unroll
  for (int q = 0; q < 4; ++q) {
    uint4 d;
    asm volatile("ld.shared.v4.b32 {%0, %1, %2, %3}, [%4];" : "=r"(d.x), "=r"(d.y), "=r"(d.z), "=r"(d.w)
                 : "r"(((q & 1) ? rd1 : rd0) + (uint32_t)(q * 4 * 128)) : "memory");
    if (pix0 + row0 + 4 * q < pixels) *reinterpret_cast<uint4 *>(o + q * 4 * 64) = d;
  }
}

__global__ void __launch_bounds__(C1_THREADS, 2)
conv1_tc_kernel(const float *__restrict__ x, int N, int H, int W, const float *__restrict__ w, const float *__restrict__ bias,
                int relu, __nv_bfloat16 *__restrict__ out_hi, __nv_bfloat16 *__restrict__ out_lo) {
  extern __shared__ uint8_t smem_raw[];
  uint8_t *smem = reinterpret_cast<uint8_t *>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~(uintptr_t)1023);
  uint8_t *sB = smem + 2 * C1_A_BYTES;
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const uint32_t so = smem_u32(sB + C1_B_BYTES) + (uint32_t)(warp * C1_OUT_WARP);
  const uint32_t b_base = smem_u32(sB);
  const int g = tid >> 7;
  const int pixels = N * H * W;                        // < 2^31 (checked by the launcher): 32-bit index math throughout
  const int total_tiles = (pixels + BM - 1) / BM;
  asm volatile("griddepcontrol.wait;" ::: "memory");
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  const int c0 = 2 * (lane & 3);                       // this thread's fragment channels: 8 j + c0, + 1 (j < 8)
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
  const int brow = tid & 127, bhalf = tid >> 7;          // builder: A row, k columns [16 bhalf, 16 bhalf + 16)
  float in[16];
  conv1_gather(x, (int)blockIdx.x * BM + brow, pixels, H, W, bhalf, in);     // the launcher keeps blockIdx.x < total_tiles
  for (int tile = blockIdx.x, it = 0; tile < total_tiles; tile += gridDim.x, ++it) {
    // ---- im2col of this tile's taps (in registers) into A buffer it & 1. That buffer was last read by the MMAs of tile
    // it - 2, which both warpgroups finished before the barrier of tile it - 1.
    uint8_t *sa = smem + (it & 1) * C1_A_BYTES;
    uint8_t *pa = sa + (size_t)brow * 128;
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
    const uint32_t a_base = smem_u32(sa);
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
    // ---- the next tile's taps: in flight while this tile's MMAs run and its outputs are stored
    const int next = tile + (int)gridDim.x;
    conv1_gather(x, next < total_tiles ? next * BM + brow : pixels, pixels, H, W, bhalf, in);
    wgmma_wait<0>();
    wgmma_fence_acc(acc);
    // ---- epilogue on the fragment: acc[4 j + {0, 1}] = row lane / 4, channels 8 j + c0 + {0, 1}; acc[4 j + {2, 3}] = row
    // lane / 4 + 8 (wgmma m64: warp k of a warpgroup owns rows 16 k .. 16 k + 15)
#pragma unroll
    for (int j = 0; j < 8; ++j) {
      const float2 b = __ldg(reinterpret_cast<const float2 *>(bias + 8 * j + c0));
#pragma unroll
      for (int h = 0; h < 2; ++h) {
        float &f0 = acc[4 * j + 2 * h], &f1 = acc[4 * j + 2 * h + 1];
        f0 += b.x; f1 += b.y;
        if (relu) { f0 = fmaxf(f0, 0.f); f1 = fmaxf(f1, 0.f); }
      }
    }
    const int pix0 = tile * BM + 64 * g + 16 * (warp & 3);
#pragma unroll 1
    for (int plane = 0; plane < 2; ++plane) {          // the split is recomputed per plane: 16 fewer live registers
      uint32_t v[16];
#pragma unroll
      for (int j = 0; j < 8; ++j)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
          uint32_t hi2, lo2;
          split_bf16x2(acc[4 * j + 2 * h], acc[4 * j + 2 * h + 1], hi2, lo2);
          v[8 * h + j] = plane ? lo2 : hi2;
        }
      conv1_store_plane(so, v, plane ? out_lo : out_hi, pix0, pixels, lane);
    }
  }
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

// the operand map of an (N tile, scheme) instantiation: boxes of row_bytes rows (box[0] = stage_k elements) in tiles
// swizzled to match; FP8X1 has 1-byte elements, the other schemes bf16 / fp16
int encode_map(mpn_ctx *ctx, CUtensorMap *tm, const void *base, int rank, const cuuint64_t *dims,
               const cuuint64_t *strides_bytes /* rank-1 */, const cuuint32_t *box, const cuuint32_t *estr, int BN, OperandScheme ops) {
  const bool fp8 = ops == OperandScheme::FP8X1;
  PFN_encodeTiled fn = get_encode_fn();
  if (!fn) return mpn_fail(ctx, MPN_ERR_CUDA, "cuTensorMapEncodeTiled entry point unavailable");
  CUresult r = fn(tm, fp8 ? CU_TENSOR_MAP_DATA_TYPE_UINT8 : CU_TENSOR_MAP_DATA_TYPE_BFLOAT16, (cuuint32_t)rank, const_cast<void *>(base), dims,
                  strides_bytes, box, estr, CU_TENSOR_MAP_INTERLEAVE_NONE, row_bytes(BN, ops) == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_128B,
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

template <int BN, OperandScheme OPS = OperandScheme::BF16X3>
int launch_bn(mpn_ctx *ctx, const ConvPlan &pl, const TcParams &tp) {
  const int smem = tc_smem_bytes(BN, OPS);
  // slots 0-2: BF16X3 by BN, 3: FP16X2, 5-7: BF16X1 by BN, 8-9: FP8X1 by BN (4 is the first-layer kernel)
  constexpr int bslot = BN == 256 ? 2 : (BN == 128 ? 1 : 0);
  constexpr int slot = OPS == OperandScheme::FP16X2 ? 3 : (OPS == OperandScheme::BF16X1 ? 5 + bslot
                                                         : (OPS == OperandScheme::FP8X1 ? 8 + bslot : bslot));
  if (!ctx->tc_attr_set[slot]) {     // per ctx (= per device): the attribute is per device function
    MPN_CUDA(ctx, cudaFuncSetAttribute(conv_gemm_tc_kernel<BN, OPS>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    ctx->tc_attr_set[slot] = 1;
  }
  const long long units = (long long)pl.tiles_img * pl.tiles_h * pl.tiles_w * pl.tiles_n * pl.splitk;
  MPN_CHECK_ARG(ctx, units > 0 && units < (1ll << 31), "conv_tc: grid size out of range");
  TcParams tpu = tp;
  tpu.units = (int)units;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)std::min<long long>(units, ctx->sm_count));     // persistent: one CTA per SM
  cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = (size_t)smem; cfg.stream = ctx->stream;
  cudaLaunchAttribute attr[1];
  int na = 0;
  if (tc_use_pdl()) {
    attr[na].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    attr[na].val.programmaticStreamSerializationAllowed = 1;
    ++na;
  }
  cfg.attrs = attr; cfg.numAttrs = na;
  MPN_CUDA(ctx, cudaLaunchKernelEx(&cfg, conv_gemm_tc_kernel<BN, OPS>, pl.tmA_hi, pl.tmA_lo, pl.tmB_hi, pl.tmB_lo, tpu));
  MPN_LAUNCHED(ctx);
  return MPN_OK;
}

// the kernel instantiation of a plan: (BN, operand scheme)
int launch_ops(mpn_ctx *ctx, const ConvPlan &pl, const TcParams &tp) {
  if (pl.ops == OperandScheme::FP16X2) return launch_bn<256, OperandScheme::FP16X2>(ctx, pl, tp);
  if (pl.ops == OperandScheme::FP8X1)
    return pl.BN == 128 ? launch_bn<128, OperandScheme::FP8X1>(ctx, pl, tp) : launch_bn<64, OperandScheme::FP8X1>(ctx, pl, tp);
  if (pl.ops == OperandScheme::BF16X1) {
    switch (pl.BN) {
      case 256: return launch_bn<256, OperandScheme::BF16X1>(ctx, pl, tp);
      case 128: return launch_bn<128, OperandScheme::BF16X1>(ctx, pl, tp);
      default: return launch_bn<64, OperandScheme::BF16X1>(ctx, pl, tp);
    }
  }
  switch (pl.BN) {
    case 256: return launch_bn<256>(ctx, pl, tp);
    case 128: return launch_bn<128>(ctx, pl, tp);
    default: return launch_bn<64>(ctx, pl, tp);
  }
}

}  // namespace

// first layer on the tensor cores (see conv1_tc_kernel); y: NHWC split planes with 64 channels
// (the caller, conv_direct_nchw_launch, holds the conv_direct profile scope)
int conv1_tc_launch(mpn_ctx *ctx, const float *x_nchw, int N, int H, int W, const float *w_dev, const float *bias_dev, int relu,
                    DTensor &y) {
  MPN_CHECK_ARG(ctx, y.hi && y.lo && y.C == 64 && y.ld % 8 == 0, "conv1_tc: output must be 64-channel split planes");
  MPN_CHECK_ARG(ctx, bias_dev, "conv1_tc: bias missing");
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
  MPN_CUDA(ctx, cudaLaunchKernelEx(&cfg, conv1_tc_kernel, x_nchw, N, H, W, w_dev, bias_dev, relu, y.hi, y.lo));
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
  // BF16X1 reads the hi planes only: a bf16 training step's operands have no lo plane
  MPN_CHECK_ARG(ctx, choose_only || (p.x.hi && (p.x.lo || p.bf16) && ((p.w_hi && (p.w_lo || p.bf16)) || p.w16)),
                "conv_tc: operands must be split-bf16 (or an fp16 weight plane)");
  MPN_CHECK_ARG(ctx, !(p.w16 && p.bf16), "conv_tc: the bf16 numerics do not take an fp16 weight plane");
  MPN_CHECK_ARG(ctx, !(p.fp8 && (p.w16 || p.bf16)), "conv_tc: the fp8 numerics take neither an fp16 weight plane nor the bf16 numerics");
  MPN_CHECK_ARG(ctx, choose_only || !p.fp8 || (p.x8 && p.x8_exp && p.w8 && p.w8_exp), "conv_tc: the fp8 numerics need e4m3 planes and exponents");
  pl.ops = p.w16 ? OperandScheme::FP16X2 : (p.fp8 ? OperandScheme::FP8X1 : (p.bf16 ? OperandScheme::BF16X1 : OperandScheme::BF16X3));
  const bool w16 = pl.ops == OperandScheme::FP16X2, fp8 = pl.ops == OperandScheme::FP8X1;
  MPN_CHECK_ARG(ctx, choose_only || (p.x.fmt == 1) == w16, "conv_tc: fp16 activation planes go with the fp16 weight plane (and only with it)");
  // Cin need not fill the last K block of a tap: the A map's channel extent is Cin, so the TMA zero-fills the block beyond
  // it, and the weights of such a layer are laid out [Cout][kh][kw][conv_k_pad(Cin)] with the pad zero (the K block ->
  // (tap, channel block) mapping is the same as for Cin = 64 k). The fp8 quantizer groups 64 channels, and the fp16-weight
  // Linears are fc6 / fc7 only: neither takes a tail.
  MPN_CHECK_ARG(ctx, p.x.C % 8 == 0, "conv_tc: Cin must be a multiple of 8");
  MPN_CHECK_ARG(ctx, !fp8 || p.x.C % BK == 0, "conv_tc: the fp8 numerics need Cin a multiple of 64 (their quantizer groups are 64 channels wide)");
  MPN_CHECK_ARG(ctx, !w16 || p.x.C % BK == 0, "conv_tc: the fp16-weight path needs Cin a multiple of 64");
  const int cblocks = (int)(conv_k_pad(p.x.C) / BK);
  MPN_CHECK_ARG(ctx, p.x.ld % 8 == 0, "conv_tc: input pixel stride must be a multiple of 8 elements");
  // the TMA's global address: a channel view (a group of a grouped convolution) must start on a multiple of 8 channels
  MPN_CHECK_ARG(ctx, (uintptr_t)p.x.hi % 16 == 0 && (uintptr_t)p.x.lo % 16 == 0, "conv_tc: input planes must start on 16 bytes");
  MPN_CHECK_ARG(ctx, p.stride >= 1 && p.stride <= 2, "conv_tc: stride must be 1 or 2");
  const int Ho = (int)p.y.H, Wo = (int)p.y.W, N = (int)p.y.N;
  pl.flat = (p.kh == 1 && p.kw == 1 && p.stride == 1 && p.pad == 0 && conv_pad_w(p) == 0) ? 1 : 0;
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
    const bool r3_ok = (p.kh == 3 && p.kw == 3 && p.stride == 1 && p.pad == 1 && conv_pad_w(p) == 1);
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
  // ceil(units / SMs) (one CTA per SM). Per K block: the tensor pipe does 3 x 128 x BN x 64 MACs (2 for w16, 1 for bf16)
  // at ~1024 bf16 MACs per cycle per SM (2048 e4m3: half a bf16 product per MAC); the operands are (128 + BN) rows x 128 B
  // per plane (64 B for fp8). FP8X1 tiles are at most 128 wide (the promotion fragment doubles the accumulator registers).
  {
    const int taps = p.kh * p.kw;
    const double kblocks = (double)taps * (double)cblocks;
    double best = 1e300; int best_bn = 64;
    for (int bi = 0; bi < 3; ++bi) {
      const int bn = bi == 0 ? 256 : (bi == 1 ? 128 : 64);
      if (w16 && bn != 256) continue;                             // the fp16-weight kernel exists for the wide tile only
      if (fp8 && bn == 256) continue;
      if (!p.m_invariant && bn > 64 && bn > ((p.Cout + 63) / 64) * 64) continue;   // do not pad N by more than one 64-block
      // per-ROI layers: the N tile is a function of Cout alone, so the plan of a row never depends on the row count
      const int roi_bn = p.Cout > 128 ? 256 : (p.Cout > 64 ? 128 : 64);
      if (p.m_invariant && bn != (fp8 ? std::min(roi_bn, 128) : roi_bn)) continue;
      const long long units = tiles_m * ((p.Cout + bn - 1) / bn);
      const long long rounds = (units + sm_count - 1) / sm_count;
      const double mma = (w16 ? 2.0 : (pl.ops == OperandScheme::BF16X1 ? 1.0 : (fp8 ? 0.5 : 3.0))) * 128.0 * bn * 64.0 / 1024.0;
      const double ingest = ((double)a_planes(pl.ops) * 128 + (double)b_planes(pl.ops) * bn) * (fp8 ? 64.0 : 128.0) / 48.0;
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
    box[0] = (cuuint32_t)stage_k(pl.BN, pl.ops); box[1] = BM; box[2] = 1; box[3] = 1;
    estr[0] = estr[1] = estr[2] = estr[3] = 1;
  } else {
    if (pl.mode == 1) { pl.tn = 1; pl.th = 16; pl.tw = 8; }
    else { pl.tn = gtn; pl.th = gth; pl.tw = gtw; }
    pl.tiles_w = (Wo + pl.tw - 1) / pl.tw; pl.tiles_h = (Ho + pl.th - 1) / pl.th; pl.tiles_img = (N + pl.tn - 1) / pl.tn;
    dims[0] = (cuuint64_t)p.x.C; dims[1] = (cuuint64_t)p.x.W; dims[2] = (cuuint64_t)p.x.H; dims[3] = (cuuint64_t)p.x.N;
    strides[0] = (cuuint64_t)p.x.ld * 2; strides[1] = (cuuint64_t)p.x.W * p.x.ld * 2;
    strides[2] = (cuuint64_t)p.x.H * p.x.W * p.x.ld * 2;
    box[0] = (cuuint32_t)stage_k(pl.BN, pl.ops); box[1] = (cuuint32_t)(pl.tw * p.stride); box[2] = (cuuint32_t)(pl.th * p.stride); box[3] = (cuuint32_t)pl.tn;
    estr[0] = 1; estr[1] = (cuuint32_t)p.stride; estr[2] = (cuuint32_t)p.stride; estr[3] = 1;
  }
  {
    // split-K for GEMMs too small to fill the machine (cls/bbox heads: a handful of tiles, 64 K blocks each,
    // latency-bound): the split count depends on K only (so results do not change with the number of rows, as long as
    // the GEMM stays small); it is either that value or 1
    const long long units = tiles_m * pl.tiles_n;
    const long long num_kb = (long long)p.kh * p.kw * cblocks;
    long long sk = std::min<long long>(num_kb / 8, 8);
    // the M tiles of the 1000 proposals per image the reference tests with (ROI_TILES_REF x 128 rows)
    constexpr long long ROI_TILES_REF = 8;
    if (p.m_invariant && pl.flat && p.Cout <= 128) { if (sk < 2) sk = 1; }       // a function of (Cout, K) only
    // the first factor of an SVD-compressed Linear (p.fill_split): as many splits as fill the SMs with ROI_TILES_REF M
    // tiles, at least 8 K blocks each; fc6's 25088 -> 1024 at 4 N tiles takes 4 splits, fc7's 4096 -> 256 takes 8
    else if (p.m_invariant && pl.flat && p.fill_split)
      sk = std::max<long long>(1, std::min<long long>(sm_count / (ROI_TILES_REF * pl.tiles_n), num_kb / 8));
    else if (p.m_invariant) sk = 1;
    // trunk weight gradients (K = pixels) with K >= 16384: at most 32 K blocks (2048 pixels) per split, and at least as
    // many splits as fill the SMs. The accumulator's error grows with the K one split sums: at 151 K blocks per split
    // (conv3_2 at 600 x 1000 + 600 x 800, 7 splits) dW measured 2.2e-4 normwise against fp64, past the per-GEMM 1e-4
    else if (p.wide_k_split && pl.flat && num_kb >= 256)
      sk = std::max<long long>({1, std::min<long long>(sm_count / units, num_kb / 8), (num_kb + 31) / 32});
    else if (pl.mode == 1 || sk < 2 || units * sk > sm_count) sk = 1;
    const char *env2 = getenv("MPN_TC_SPLITK");
    if (env2 && env2[0] == '0') sk = 1;
    pl.splitk = (int)std::max<long long>(sk, 1);
    pl.kb_per_split = (int)((num_kb + pl.splitk - 1) / pl.splitk);
    pl.splitk = (int)((num_kb + pl.kb_per_split - 1) / pl.kb_per_split);     // no empty splits
  }
  if (choose_only) return MPN_OK;
  const long long Ktot = (long long)p.kh * p.kw * conv_k_pad(p.x.C);
  cuuint64_t bd[2] = {(cuuint64_t)Ktot, (cuuint64_t)p.Cout}, bs[1] = {(cuuint64_t)Ktot * 2};
  cuuint32_t bb[2] = {(cuuint32_t)stage_k(pl.BN, pl.ops), (cuuint32_t)pl.BN}, be[2] = {1, 1};
  if (fp8) {                           // dense 1-byte planes: x8 [pixel][x.C], w8 [Cout][Ktot]
    const cuuint64_t C8 = (cuuint64_t)p.x.C;
    if (pl.flat) { strides[0] = C8; strides[1] = (cuuint64_t)P * C8; strides[2] = strides[1]; }
    else { strides[0] = C8; strides[1] = (cuuint64_t)p.x.W * C8; strides[2] = (cuuint64_t)p.x.H * p.x.W * C8; }
    bs[0] = (cuuint64_t)Ktot;
    MPN_TRY(encode_map(ctx, &pl.tmA_hi, p.x8, 4, dims, strides, box, estr, pl.BN, pl.ops));
    MPN_TRY(encode_map(ctx, &pl.tmB_hi, p.w8, 2, bd, bs, bb, be, pl.BN, pl.ops));
    pl.tmA_lo = pl.tmA_hi; pl.tmB_lo = pl.tmB_hi;
    pl.valid = 1;
    return MPN_OK;
  }
  MPN_TRY(encode_map(ctx, &pl.tmA_hi, p.x.hi, 4, dims, strides, box, estr, pl.BN, pl.ops));
  if (a_planes(pl.ops) == 2) { MPN_TRY(encode_map(ctx, &pl.tmA_lo, p.x.lo, 4, dims, strides, box, estr, pl.BN, pl.ops)); }
  else pl.tmA_lo = pl.tmA_hi;                                            // BF16X1: the lo planes are never read
  if (w16) {
    // split-K partials are scaled by acc_scale in the epilogue, so the reduce sums true values in its fixed order
    MPN_CHECK_ARG(ctx, pl.mode == 0 && pl.flat && pl.BN == 256, "conv_tc: the fp16-weight path is for wide flat GEMMs");
    MPN_TRY(encode_map(ctx, &pl.tmB_hi, p.w16, 2, bd, bs, bb, be, pl.BN, pl.ops));      // 16-bit elements: the TMA only moves bytes
    pl.tmB_lo = pl.tmB_hi;
  } else {
    MPN_TRY(encode_map(ctx, &pl.tmB_hi, p.w_hi, 2, bd, bs, bb, be, pl.BN, pl.ops));
    if (b_planes(pl.ops) == 2) { MPN_TRY(encode_map(ctx, &pl.tmB_lo, p.w_lo, 2, bd, bs, bb, be, pl.BN, pl.ops)); }
    else pl.tmB_lo = pl.tmB_hi;
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
  tp.Cout = p.Cout; tp.kh = p.kh; tp.kw = p.kw; tp.stride = p.stride; tp.pad_h = p.pad; tp.pad_w = conv_pad_w(p);
  tp.cblocks = (int)(conv_k_pad(p.x.C) / BK);
  tp.tn = pl.tn; tp.th = pl.th; tp.tw = pl.tw;
  tp.tiles_img = pl.tiles_img; tp.tiles_h = pl.tiles_h; tp.tiles_w = pl.tiles_w; tp.tiles_n = pl.tiles_n;
  tp.bias = p.bias;
  tp.res_hi = p.res.hi; tp.res_lo = p.res.lo; tp.res_ld = p.res.ld;
  tp.out_hi = p.y.hi; tp.out_lo = p.y.lo; tp.out_ld = p.y.ld;
  tp.out_f32 = p.y.f32; tp.out_f32_ld = p.y_f32_ld;
  tp.relu = p.relu;
  tp.splitk = pl.splitk; tp.kb_per_split = pl.kb_per_split; tp.split_stride = 0;
  tp.acc_scale = pl.ops == OperandScheme::FP16X2 ? p.w16_inv_scale : 1.f;
  tp.out_fmt = p.y.fmt; tp.ovf = nullptr;
  if (p.y.fmt) MPN_TRY(mpn_ovf_flag(ctx, &tp.ovf));
  if (pl.ops == OperandScheme::FP8X1) { tp.a_exp = p.x8_exp; tp.b_exp = p.w8_exp; tp.sample_pix = p.y.H * p.y.W; }
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
    MPN_TRY(launch_ops(ctx, pl, tp));
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
  return launch_ops(ctx, pl, tp);
}

// Host-only view of the planner (no GPU): which engine configuration conv_tc_plan would pick for a layer on a device
// with `sm_count` SMs. out[8] = {mode (bit 0: 16 x 8 patches of the 3x3 / stride 1 convolutions), CTA group (always 1),
// BN, split-K, stream-K (always 0), tn, th, tw}. per_roi: 0 trunk layer, 1 per-ROI layer, 2 per-ROI Linear without a bias
// (the first factor of an SVD-compressed Linear: ConvProblem::fill_split).
extern "C" int mpn_debug_plan(int64_t N, int64_t Cin, int64_t H, int64_t W, int64_t Cout, int32_t k, int32_t stride, int32_t pad,
                              int32_t per_roi, int32_t sm_count, int32_t *out) {
  if (!out || N <= 0 || Cin <= 0 || Cin % 8 || H <= 0 || W <= 0 || Cout <= 0 || k <= 0 || stride < 1 || stride > 2 || pad < 0 || sm_count < 2 ||
      per_roi < 0 || per_roi > 2)
    return MPN_ERR_ARG;
  ConvProblem p;
  p.x.N = N; p.x.H = H; p.x.W = W; p.x.C = Cin; p.x.ld = Cin;
  p.Cout = (int)Cout; p.kh = p.kw = k; p.stride = stride; p.pad = pad; p.m_invariant = per_roi ? 1 : 0;
  p.fill_split = per_roi == 2 ? 1 : 0;
  p.y.N = N; p.y.H = (H + 2 * pad - k) / stride + 1; p.y.W = (W + 2 * pad - k) / stride + 1; p.y.C = Cout; p.y.ld = Cout;
  if (p.y.H <= 0 || p.y.W <= 0) return MPN_ERR_ARG;
  ConvPlan pl;
  const int rc = conv_tc_plan_impl(nullptr, sm_count, p, pl, true);
  if (rc != MPN_OK) return rc;
  out[0] = pl.mode; out[1] = 1; out[2] = pl.BN; out[3] = pl.splitk; out[4] = 0; out[5] = pl.tn; out[6] = pl.th; out[7] = pl.tw;
  return MPN_OK;
}

"""GPU: the wgmma engine's operand ring. The 256-wide tiles of the 16-bit schemes (bf16x3, the bf16 numerics, the fp16
weights of fc6 / fc7) stage half a K block per ring stage, the narrower ones a whole K block. This covers what that
staging can get wrong: K loops that end before, at and past a wrap of the ring (in every N tile width and scheme),
split-K units shorter than the ring, convolutions with many more tiles than SMs, and stride-2 convolutions. Each result
is checked against fp64 at the engine's 1e-4 normwise bar, and a second run must give the same bits."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import multipathnet_b200 as mpn
from conftest import rel_err
from test_engine_gpu import _w16_emulation
import _bf16_oracle as B

pytestmark = pytest.mark.gpu
TOL = 1e-4
SM_COUNT = 132

# (ring depth in stages, stages per K block) by (scheme, N tile): gemm_tc.cu num_stages, kb_steps
DEPTH = {("bf16x3", 64): (4, 1), ("bf16x3", 128): (3, 1), ("bf16x3", 256): (4, 2), ("bf16", 64): (4, 1), ("bf16", 128): (4, 1),
         ("bf16", 256): (8, 2), ("w16", 256): (6, 2)}
N_FOR_BN = {64: 64, 128: 120, 256: 256}       # a GEMM's N tile is a function of its width (per-ROI planning)


@contextlib.contextmanager
def scheme(ctx, name):
    if name == "bf16":
        ctx.set_option("bf16", 1)
    try:
        yield
    finally:
        ctx.set_option("bf16", -1)


def _rn(a):
    return B.rn_bf16(torch.from_numpy(np.ascontiguousarray(a, np.float32))).double()


def plan(N, Cin, H, W, Cout, k, s, p, per_roi=0):
    out = (C.c_int32 * 8)()
    assert mpn.load_library().mpn_debug_plan(N, Cin, H, W, Cout, k, s, p, per_roi, SM_COUNT, out) == 0
    return dict(zip(("mode", "cg", "bn", "splitk", "streamk", "tn", "th", "tw"), out))


def gemm_ref(name, A, Bm, bias):
    if name == "w16":
        return _w16_emulation(A, Bm, bias, True)
    a, b = (_rn(A), _rn(Bm)) if name == "bf16" else (torch.from_numpy(A).double(), torch.from_numpy(Bm).double())
    return torch.relu(a @ b.t() + torch.from_numpy(bias).double()).numpy()


def run_gemm(ctx, name, A, Bm, bias):
    impl = 2 if name == "w16" else 0
    with scheme(ctx, name):
        got = ctx.gemm_check(A, Bm, bias, relu=True, impl=impl)
        again = ctx.gemm_check(A, Bm, bias, relu=True, impl=impl)
    assert np.array_equal(got, again), "two runs differ"
    return got


def _ring_cases():
    for (name, bn), (S, per_kb) in DEPTH.items():
        # K loops of one K block, half the ring, half the ring + 1 stage, the full ring, one stage past it, past the second wrap
        for steps in sorted({per_kb, S // 2, S // 2 + 1, S, S + 1, 2 * S + 1}):
            kblocks = max(1, -(-steps // per_kb))
            yield name, bn, kblocks


@pytest.mark.parametrize("name,bn,kblocks", sorted(set(_ring_cases())))
def test_gemm_ring_wrap(ctx, name, bn, kblocks):
    M, N, K = 300, N_FOR_BN[bn], 64 * kblocks
    assert plan(M, K, 1, 1, N, 1, 1, 0, per_roi=1)["bn"] == bn
    rng = np.random.default_rng(N + K)
    A = np.maximum(rng.standard_normal((M, K)), 0).astype(np.float32)
    Bm = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    got = run_gemm(ctx, name, A, Bm, bias)
    assert rel_err(got, gemm_ref(name, A, Bm, bias)) < TOL


@pytest.mark.parametrize("name", ["bf16x3", "bf16"])
@pytest.mark.parametrize("N", [21, 84, 128])
def test_gemm_split_k_tail_shorter_than_ring(ctx, name, N):
    """K = 65 K blocks: 8 splits of 9 K blocks, the last one only 2 (4 stages, less than the ring holds)"""
    M, K = 200, 64 * 65
    pl = plan(M, K, 1, 1, N, 1, 1, 0, per_roi=1)
    assert pl["splitk"] == 8
    rng = np.random.default_rng(N)
    A = rng.standard_normal((M, K)).astype(np.float32)
    Bm = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    got = run_gemm(ctx, name, A, Bm, bias)
    assert rel_err(got, gemm_ref(name, A, Bm, bias)) < TOL


def _conv(ctx, name, N, Cin, H, W, Cout, k, s, p):
    rng = np.random.default_rng(Cin + H + W + Cout + s)
    x = rng.standard_normal((N, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    with scheme(ctx, name):
        got = ctx.conv_check(x, w, b, stride=s, pad=p, relu=True, impl=0)
        again = ctx.conv_check(x, w, b, stride=s, pad=p, relu=True, impl=0)
    assert np.array_equal(got, again), "two runs differ"
    xr, wr = (_rn(x), _rn(w)) if name == "bf16" else (torch.from_numpy(x).double(), torch.from_numpy(w).double())
    ref = F.relu(F.conv2d(xr, wr, torch.from_numpy(b).double(), stride=s, padding=p)).numpy()
    assert rel_err(got, ref) < TOL


@pytest.mark.parametrize("name", ["bf16x3", "bf16"])
@pytest.mark.parametrize("shape,bn,splitk", [
    ((1, 64, 192, 256, 64, 3, 1, 1), 64, 1),        # 384 tiles of 16 x 8
    ((1, 128, 200, 256, 128, 3, 1, 1), 64, 1),      # 416 tiles x 2 N tiles
    ((1, 64, 60, 80, 256, 3, 1, 1), 128, 1),
    ((1, 128, 150, 200, 256, 3, 1, 1), 256, 1),
    ((2, 64, 30, 34, 64, 3, 2, 1), 64, 1),          # stride 2
    ((1, 128, 28, 36, 256, 1, 2, 0), 64, 1),
    ((2, 128, 60, 64, 256, 3, 2, 1), 64, 2),        # stride 2, split-K
])
def test_conv_ring(ctx, name, shape, bn, splitk):
    if name == "bf16x3":            # (the bf16 numerics' cost model may choose other tiles: they run whatever it picks)
        pl = plan(*shape)
        assert (pl["bn"], pl["splitk"]) == (bn, splitk)
    _conv(ctx, name, *shape)


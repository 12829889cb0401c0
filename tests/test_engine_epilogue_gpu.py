"""GPU: the wgmma engine's persistent tile loop and its epilogue, which finishes each tile straight from the accumulator
fragments (64 channels at a time, split planes through a per-warp shared buffer, fp32 stored directly).

Covers every (scheme, N tile) instantiation that the check entry points reach (bf16x3 and bf16 at 64 / 128 / 256, the
fp16-weight kernel at 256, fp8 at 64 / 128), edge tiles in H, W and N, generic patches with several images per tile,
stride 2, split-K heads, and grids with fewer units than SMs, one more unit than SMs and many more. Each result is
checked against fp64 (fp8: against the CUDA-core check kernel on the same e4m3 operands) at the engine's 1e-4
normwise bar, and a second run must give the same bits. The fused pool, residuals, channel-slice outputs and fp16
output planes run in the whole-model tests."""
import contextlib

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err
from test_engine_ring_gpu import plan, gemm_ref, _rn

pytestmark = pytest.mark.gpu
TOL = 1e-4


@contextlib.contextmanager
def scheme(ctx, name):
    if name in ("bf16", "fp8"):
        ctx.set_option(name, 1)
    try:
        yield
    finally:
        if name in ("bf16", "fp8"):
            ctx.set_option(name, -1)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _conv(ctx, name, N, Cin, H, W, Cout, k, s, p, relu=True):
    rng = np.random.default_rng(N * 7 + Cin + H + W + Cout + s)
    x = rng.standard_normal((N, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    with scheme(ctx, name):
        got = ctx.conv_check(x, w, b, stride=s, pad=p, relu=relu, impl=0)
        again = ctx.conv_check(x, w, b, stride=s, pad=p, relu=relu, impl=0)
        chk = ctx.conv_check(x, w, b, stride=s, pad=p, relu=relu, impl=1) if name == "fp8" else None
    assert np.array_equal(got, again), "two runs differ"
    if name == "fp8":
        assert rel_err(got, chk) < TOL + 2.0 ** -17
        return
    xr, wr = (_rn(x), _rn(w)) if name == "bf16" else (torch.from_numpy(x).double(), torch.from_numpy(w).double())
    ref = F.conv2d(xr, wr, torch.from_numpy(b).double(), stride=s, padding=p)
    ref = (F.relu(ref) if relu else ref).numpy()
    assert rel_err(got, ref) < TOL


# (N, Cin, H, W, Cout, k, s, p): the 16 x 8 patches at odd H / W, a partial last N tile, generic patches with tn > 1,
# stride 2 and 1x1 layers
SHAPES = [(1, 64, 37, 53, 64, 3, 1, 1), (1, 64, 37, 53, 200, 3, 1, 1), (1, 128, 19, 25, 320, 3, 1, 1),
          (3, 64, 5, 7, 128, 3, 1, 1), (4, 64, 3, 5, 64, 3, 2, 1), (2, 64, 15, 17, 136, 3, 2, 1), (3, 128, 9, 11, 256, 1, 1, 0)]


@pytest.mark.parametrize("name", ["bf16x3", "bf16", "fp8"])
@pytest.mark.parametrize("shape", SHAPES)
def test_conv_edge_tiles(ctx, name, shape):
    _conv(ctx, name, *shape)


@pytest.mark.parametrize("name", ["bf16x3", "bf16", "fp8"])
@pytest.mark.parametrize("rel", ["few", "sms+1", "many"])
def test_conv_units_vs_sms(ctx, name, rel):
    """16 x 8 patches, 64 channels: units = tiles. Fewer units than SMs, one more than SMs (one CTA runs two), and about
    five per SM"""
    sms = _sms()
    tiles_w = {"few": 5, "sms+1": sms + 1, "many": 5 * sms + 3}[rel]
    H, W = 16, 8 * tiles_w
    if name == "bf16x3":
        pl = plan(1, 64, H, W, 64, 3, 1, 1)
        assert (pl["bn"], pl["mode"], pl["splitk"]) == (64, 1, 1)
    _conv(ctx, name, 1, 64, H, W, 64, 3, 1, 1)


@pytest.mark.parametrize("relu", [True, False])
def test_conv_no_relu_and_bn256_many_units(ctx, relu):
    """BN = 256 tiles, two and a half waves of them; without ReLU the epilogue's sign handling is exercised too"""
    _conv(ctx, "bf16x3", 1, 128, 150, 200, 256, 3, 1, 1, relu=relu)


def _gemm(ctx, name, M, N, K, seed):
    rng = np.random.default_rng(seed)
    A = rng.standard_normal((M, K)).astype(np.float32)
    Bm = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    impl = 2 if name == "w16" else 0
    with scheme(ctx, name):
        got = ctx.gemm_check(A, Bm, bias, relu=True, impl=impl)
        again = ctx.gemm_check(A, Bm, bias, relu=True, impl=impl)
        chk = ctx.gemm_check(A, Bm, bias, relu=True, impl=1) if name == "fp8" else None
    assert np.array_equal(got, again), "two runs differ"
    if name == "fp8":
        assert rel_err(got, chk) < TOL + 2.0 ** -17
    else:
        assert rel_err(got, gemm_ref(name, A, Bm, bias)) < TOL


# per-ROI GEMMs: the N tile is a function of N (64 / 128 / 256); M rows in units below, just past and well past the SMs
@pytest.mark.parametrize("name,N", [("bf16x3", 64), ("bf16x3", 120), ("bf16x3", 264), ("bf16", 64), ("bf16", 128),
                                    ("bf16", 256), ("w16", 512), ("fp8", 64), ("fp8", 128)])
@pytest.mark.parametrize("M", [300, 128 * 133 - 5, 5000])
def test_gemm_schemes(ctx, name, N, M):
    _gemm(ctx, name, M, N, 64 * 3, N + M)


@pytest.mark.parametrize("name", ["bf16x3", "bf16"])
@pytest.mark.parametrize("M,N", [(1000, 21), (1000, 84), (77, 128)])
def test_gemm_split_k_heads(ctx, name, M, N):
    """the cls / bbox heads: K = 4096 runs as 8 splits whose fp32 partials go straight from the fragments"""
    assert plan(M, 4096, 1, 1, N, 1, 1, 0, per_roi=1)["splitk"] == 8
    _gemm(ctx, name, M, N, 4096, M + N)

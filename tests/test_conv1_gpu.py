"""GPU parity of the first-layer kernel (conv1_tc_kernel: 3x3, pad 1, Cin 3, Cout 64, with a bias) against an fp64
F.conv2d, at the bar of test_engine_gpu.py::test_first_layer_direct_conv. conv_check(..., impl=2) with a bias is the
call that reaches this kernel. The sizes cover the full 600 x 800 image, images smaller than one 128-pixel tile,
sizes that leave a partial last tile, and N = 2 (tiles that straddle two images)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _case(N, H, W, seed):
    rng = np.random.default_rng(seed)
    x = (rng.random((N, 3, H, W)) * 255 - 110).astype(np.float32)
    w = (rng.standard_normal((64, 3, 3, 3)) / 64).astype(np.float32)
    b = rng.standard_normal(64).astype(np.float32)
    return x, w, b


def _ref(x, w, b, relu):
    y = F.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(), padding=1)
    return (F.relu(y) if relu else y).float().numpy()


@pytest.mark.parametrize("relu", [True, False])
@pytest.mark.parametrize("N,H,W", [(1, 600, 800), (1, 1, 1), (1, 7, 5), (1, 37, 53), (1, 601, 799), (2, 37, 53), (2, 600, 800)])
def test_first_layer_kernel(ctx, N, H, W, relu):
    x, w, b = _case(N, H, W, 100 + H + W)
    got = ctx.conv_check(x, w, b, stride=1, pad=1, relu=relu, impl=2)
    assert got.shape == (N, 64, H, W)
    assert rel_err(got, _ref(x, w, b, relu)) < TOL
    if not relu:
        assert (got < 0).any()        # the bias-only path really ran without the clamp


@pytest.mark.parametrize("N,H,W", [(1, 600, 800), (2, 37, 53)])
def test_first_layer_kernel_is_deterministic(ctx, N, H, W):
    x, w, b = _case(N, H, W, 7)
    a = ctx.conv_check(x, w, b, stride=1, pad=1, relu=True, impl=2)
    c = ctx.conv_check(x, w, b, stride=1, pad=1, relu=True, impl=2)
    assert np.array_equal(a, c)

"""GPU: the inn.ROIPooling backward (roi_pool_backward_nchw_kernel through mpn_roi_pool_backward[_dev]) against the
reference scatter of tests/_roi_backward_ref.py, bit for bit: both sum each cell in ascending (roi, ph, pw) order."""
import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import modules, workloads as wl
from oracle import ref as O
from _roi_backward_ref import roi_pool_backward as scatter

pytestmark = pytest.mark.gpu


def _forward_backward(ctx, fm, rois, P, scale, variant, seed=0):
    """device argmax == oracle argmax, then device grad_data == the reference scatter exactly; returns (grad_out, argmax, grad_data)"""
    out, am = ctx.roi_pool(fm, rois, P, P, scale, variant, with_argmax=True)
    _, ra = O.roi_pool(fm, rois, P, P, scale, variant, with_argmax=True)
    assert np.array_equal(am, ra)
    g = np.random.default_rng(seed).standard_normal(out.shape, dtype=np.float32)
    gd = ctx.roi_pool_backward(g, am, rois, fm.shape, P, P, scale, variant)
    assert np.array_equal(gd, scatter(g, ra, rois, fm.shape))
    return g, am, gd


def _add_at(g, am, rois, shape):
    """independent fp64 statement: np.add.at over the argmax"""
    ref = np.zeros(shape, np.float64)
    r, c, _, _ = np.nonzero(am >= 0)
    n = rois[:, 0].astype(np.int64)[r] - 1
    a = am[am >= 0]
    np.add.at(ref.reshape(shape[0], shape[1], -1), (n, c, a), g[am >= 0].astype(np.float64))
    return ref


@pytest.mark.parametrize("variant", [1, 2])
@pytest.mark.parametrize("name", ["S1", "S2", "S3", "S4", "R1000"])
def test_backward_bit_exact_vs_reference(ctx, name, variant):
    fm, rois, P, scale = wl.roi_pool_case(name, foveal=ctx.foveal)
    g, am, gd = _forward_backward(ctx, fm, rois, P, scale, variant)
    if name == "S1":
        assert np.any(am == -1)                                    # inverted / outside rois: empty bins
    ref = _add_at(g, am, rois, fm.shape)
    assert np.max(np.abs(gd - ref)) <= 1e-6 * max(np.max(np.abs(ref)), 1e-30)


@pytest.mark.parametrize("variant", [1, 2])
def test_backward_edge_cases(ctx, variant):
    # all-equal map: every argmax is the first cell of its bin
    fm = np.ones((2, 16, 20, 37), np.float32)
    rois = np.zeros((50, 5), np.float32)
    rois[:, 1:] = wl.random_boxes(50, 320, 592, 3)
    rois[:, 0] = np.arange(50) % 2 + 1
    _, am, gd = _forward_backward(ctx, fm, rois, 7, 1 / 16, variant, seed=1)
    # tiny rois (one pixel: smaller than a bin, so one cell is the argmax of all 49 bins), mixed with ordinary ones
    tiny = np.concatenate([rois[:10], np.array([[1, 40, 40, 40, 40], [2, 600, 300, 600, 300], [1, 1, 1, 1, 1]], np.float32)])
    fm2 = np.random.default_rng(4).standard_normal((2, 16, 20, 37), dtype=np.float32)
    _, am, _ = _forward_backward(ctx, fm2, tiny, 7, 1 / 16, variant, seed=2)
    assert all(len(np.unique(am[i, 0])) == 1 for i in range(10, 13))
    # R = 0: zeros
    gd = ctx.roi_pool_backward(np.zeros((0, 16, 7, 7), np.float32), np.zeros((0, 16, 7, 7), np.int32), np.zeros((0, 5), np.float32),
                               fm.shape, 7, 7, 1 / 16, variant)
    assert gd.shape == fm.shape and np.all(gd == 0) and not np.any(np.signbit(gd))


def test_backward_deterministic_host_and_device_forms_agree(ctx):
    import torch
    fm, rois, P, scale = wl.roi_pool_case("S3")
    out, am = ctx.roi_pool(fm, rois, P, P, scale, 2, with_argmax=True)
    g = np.random.default_rng(9).standard_normal(out.shape, dtype=np.float32)
    ctx.profile_begin()
    a = ctx.roi_pool_backward(g, am, rois, fm.shape, P, P, scale, 2)
    assert ctx.profile_end()["roi_pool"][1] == 1                   # timed under the ROI pooling category
    b = ctx.roi_pool_backward(g, am, rois, fm.shape, P, P, scale, 2)
    assert np.array_equal(a.view(np.uint32), b.view(np.uint32))
    N, C, H, W = fm.shape
    g_d, am_d, r_d = torch.from_numpy(g).cuda(), torch.from_numpy(am).cuda(), torch.from_numpy(rois).cuda()
    gd_d = torch.full((N, C, H, W), float("nan"), dtype=torch.float32, device="cuda")   # every element must be written
    torch.cuda.synchronize()
    ctx.roi_pool_backward_dev(g_d, am_d, N, C, H, W, r_d, rois.shape[0], P, P, scale, 2, gd_d)
    ctx.synchronize()
    d = gd_d.cpu().numpy()
    assert not np.any(np.isnan(d))
    assert np.array_equal(d.view(np.uint32), a.view(np.uint32))


def test_backward_validates_like_the_forward(ctx):
    fm = np.zeros((1, 8, 10, 10), np.float32)
    g, am = np.zeros((1, 8, 2, 2), np.float32), np.zeros((1, 8, 2, 2), np.int32)
    with pytest.raises(mpn.MpnError, match="batch index"):
        ctx.roi_pool_backward(g, am, np.array([[3, 1, 1, 5, 5]], np.float32), fm.shape, 2, 2, 1.0)
    with pytest.raises(mpn.MpnError, match="variant"):
        ctx.roi_pool_backward(g, am, np.array([[1, 1, 1, 5, 5]], np.float32), fm.shape, 2, 2, 1.0, variant=3)


def test_module_update_grad_input(ctx):
    fm, rois, P, scale = wl.roi_pool_case("S2")
    m = modules.ROIPooling(ctx, P, P, scale)
    with pytest.raises(RuntimeError):
        m.updateGradInput((fm, rois), np.zeros((2, 512, 7, 7), np.float32))      # no forward yet: no argmax
    out = m.forward((fm, rois))
    g = np.random.default_rng(3).standard_normal(out.shape, dtype=np.float32)
    gd, gr = m.updateGradInput((fm, rois), g)
    _, ra = O.roi_pool(fm, rois, P, P, scale, 2, with_argmax=True)
    assert np.array_equal(gd, scatter(g, ra, rois, fm.shape))
    assert gr.shape == rois.shape and np.all(gr == 0)
    assert m.gradInput[0] is gd

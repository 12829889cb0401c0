"""CPU suite: the reference inn.ROIPooling backward (tests/_roi_backward_ref.py, a scatter through the forward's argmax)
on hand-computed known answers, on its fp32 summation order and on the adjoint identity of a selection. The device
kernel is checked against it bit for bit in tests/test_roi_backward_gpu.py."""
import numpy as np
import pytest

from _roi_backward_ref import roi_pool_backward as scatter

# 4x4 map, maximum at cell (1,1) = flat 5, every other value distinct and smaller
MAP = np.arange(16, dtype=np.float32).reshape(1, 1, 4, 4)
MAP[0, 0, 1, 1] = 100.0
# the same windows under both end conventions (v2 ends one cell earlier): A = cells [0,2]^2, B = cells [0,1]^2
ROIS = {1: np.array([[1, 1, 1, 3, 3], [1, 1, 1, 2, 2]], np.float32),
        2: np.array([[1, 1, 1, 4, 4], [1, 1, 1, 3, 3]], np.float32)}


@pytest.mark.parametrize("variant", [1, 2])
def test_known_answer_overlapping_rois(oracle_built, variant):
    """2x2 bins at scale 1. A is 3 cells wide, so its bins are [0,2) and [1,3) per axis: cell 5 lies in all four and is
    the argmax of each. B's bins are single cells: they select 0, 1, 4, 5. Cell 5 collects four bins of A and one of B;
    cell 10 lies in A's bins but is never selected; cell 15 is in no bin."""
    O = oracle_built
    rois = ROIS[variant]
    out, am = O.roi_pool(MAP, rois, 2, 2, 1.0, variant, with_argmax=True)
    assert am.reshape(2, 4).tolist() == [[5, 5, 5, 5], [0, 1, 4, 5]]
    g = np.array([[1, 2, 3, 4], [10, 20, 30, 40]], np.float32).reshape(2, 1, 2, 2)
    gd = scatter(g, am, rois, MAP.shape)
    want = np.zeros(16, np.float32)
    want[[0, 1, 4, 5]] = [10, 20, 30, 1 + 2 + 3 + 4 + 40]
    assert np.array_equal(gd.reshape(-1), want)
    assert gd[0, 0, 2, 2] == 0 and gd[0, 0, 3, 3] == 0


@pytest.mark.parametrize("variant", [1, 2])
def test_roi_smaller_than_a_bin(oracle_built, variant):
    """a one-cell ROI pooled 3x3: every bin is that cell, so it receives all nine gradients; a two-cell-wide ROI pooled
    7x7 puts each of its cells in several bins along that axis"""
    O = oracle_built
    fm = np.random.default_rng(0).permutation(30).astype(np.float32).reshape(1, 1, 5, 6)
    x2 = 4 if variant == 1 else 5
    one = np.array([[1, 4, 3, x2, 3 if variant == 1 else 4]], np.float32)      # cell (2, 3)
    out, am = O.roi_pool(fm, one, 3, 3, 1.0, variant, with_argmax=True)
    assert np.all(am == 2 * 6 + 3)
    g = np.arange(1, 10, dtype=np.float32).reshape(1, 1, 3, 3)
    gd = scatter(g, am, one, fm.shape)
    assert gd[0, 0, 2, 3] == 45 and np.count_nonzero(gd) == 1
    two = np.array([[1, 1, 1, 2 if variant == 1 else 3, 5 if variant == 1 else 6]], np.float32)   # cells [0,1] x [0,4]
    out, am = O.roi_pool(fm, two, 7, 7, 1.0, variant, with_argmax=True)
    g = np.ones((1, 1, 7, 7), np.float32)
    gd = scatter(g, am, two, fm.shape)
    cnt = np.bincount(am.reshape(-1), minlength=30).reshape(5, 6)
    assert np.array_equal(gd[0, 0], cnt.astype(np.float32))
    assert cnt[:, :2].sum() == 49 and cnt.max() > 1


def test_empty_bins_and_zero_rois(oracle_built):
    """bins of a ROI outside the map have argmax -1 and contribute nothing; R = 0 gives zeros"""
    O = oracle_built
    rois = np.array([[1, 100, 100, 120, 120]], np.float32)
    out, am = O.roi_pool(MAP, rois, 2, 2, 1.0, 2, with_argmax=True)
    assert np.all(am == -1)
    gd = scatter(np.ones((1, 1, 2, 2), np.float32), am, rois, MAP.shape)
    assert np.array_equal(gd, np.zeros_like(MAP))
    gd = scatter(np.zeros((0, 1, 2, 2), np.float32), np.zeros((0, 1, 2, 2), np.int32), np.zeros((0, 5), np.float32), MAP.shape)
    assert np.array_equal(gd, np.zeros_like(MAP))


def test_summation_order_is_roi_ph_pw_in_fp32():
    """one cell selected by every bin of two ROIs: the fp32 result depends on the order of the additions, and must be
    the sequential sum from +0 in ascending (roi, ph, pw) order"""
    am = np.full((2, 1, 2, 2), 5, np.int32)
    rois = np.array([[1, 1, 1, 3, 3], [1, 1, 1, 2, 2]], np.float32)
    g = np.array([1e8, 1, -1e8, 1, 3, -0.75, 2.5e7, -2.5e7], np.float32).reshape(2, 1, 2, 2)
    want = np.float32(0)
    for v in g.reshape(-1):
        want = np.float32(want + v)
    assert want != np.float32(np.sum(g.astype(np.float64)))          # the order is visible in this sum
    assert scatter(g, am, rois, MAP.shape)[0, 0, 1, 1] == want


@pytest.mark.parametrize("variant,seed", [(1, 0), (2, 1), (2, 2)])
def test_adjoint_identity(oracle_built, variant, seed):
    """the forward is a selection, so <grad_out, out> == <grad_data, data>. Small-integer gradients keep every fp32 cell
    sum exact; distinct map values make the argmax unique"""
    O = oracle_built
    rng = np.random.default_rng(seed)
    N, C, H, W = 2, 3, 19, 25
    data = (rng.permutation(N * C * H * W).astype(np.float32) - 700.0).reshape(N, C, H, W)
    R = 60
    xy = rng.uniform(-40, 420, (R, 2))
    wh = rng.uniform(1, 250, (R, 2))
    rois = np.concatenate([rng.integers(1, N + 1, (R, 1)), xy, xy + wh], 1).astype(np.float32)
    out, am = O.roi_pool(data, rois, 7, 7, 1 / 16, variant, with_argmax=True)
    assert np.any(am == -1) and np.any(am >= 0)
    g = rng.integers(-8, 9, out.shape).astype(np.float32)
    gd = scatter(g, am, rois, data.shape)
    lhs = float(np.sum(g.astype(np.float64) * out.astype(np.float64)))
    rhs = float(np.sum(gd.astype(np.float64) * data.astype(np.float64)))
    assert abs(lhs - rhs) <= 1e-12 * max(abs(lhs), 1.0)
    assert np.sum(gd != 0) > 0

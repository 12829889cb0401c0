"""CPU checks of tests/_detect_tail_ref.py, the references the detect-tail GPU tests hold the device to: the fp32 decode
restatement equals the C oracle (oracle.ref.convert_from / bbox_norm / clamp_boxes) bit for bit where exp is exact, the
fp64 softmax / integral mean is a distribution, and the gather + NMS chain equals a per-class loop over oracle.ref.nms."""
import numpy as np
import pytest

from multipathnet_b200 import workloads as wl
from oracle import ref as O

import _detect_tail_ref as T


@pytest.fixture(scope="module", autouse=True)
def _oracle(oracle_built):
    return oracle_built


def _exact_rows(R, C, seed):
    """deltas with y.z = y.w = 0 (exp exact) and arbitrary centre shifts; boxes of every size, some degenerate"""
    rng = np.random.default_rng(seed)
    boxes = wl.random_boxes(R, 480, 640, seed).astype(np.float32)
    boxes[::9, 2] = boxes[::9, 0]                                        # zero width
    d = (rng.standard_normal((R, C, 4)) * 0.7).astype(np.float32)
    d[..., 2:] = 0
    return d.reshape(R, 4 * C), boxes


@pytest.mark.parametrize("R,C", [(1, 2), (37, 21), (500, 81)])
def test_decode_restatement_equals_oracle_where_exp_is_exact(R, C):
    d, boxes = _exact_rows(R, C, R + C)
    got, wt, ht = T.decode(d, boxes)
    assert np.array_equal(got, O.convert_from(d, boxes))
    assert np.array_equal(wt, np.repeat((boxes[:, 2] - boxes[:, 0])[:, None], C, 1))   # exp(0) * w
    mean, std = np.float32([0.02, -0.01, 0.0, 0.0]), np.float32([0.1, 0.1, 0.2, 0.2])
    W0, H0 = 600.0, 450.0
    got, _, _ = T.decode(d, boxes, True, W0, H0, mean, std)
    want = O.clamp_boxes(O.convert_from(O.bbox_norm(d, mean, std), boxes), W0, H0)
    assert np.array_equal(got, want)
    assert got[:, 0::2].min() >= 1 and got[:, 0::2].max() <= W0 and got[:, 1::2].max() <= H0


def test_decode_restatement_edges():
    """exp overflow: w = 0 times inf is NaN and stays NaN through the clamp; inf coordinates clamp to the image"""
    boxes = np.float32([[10, 10, 10, 50], [10, 10, 60, 50]])           # w = 0, then w = 50
    d = np.zeros((2, 8), np.float32)
    d[:, 2] = 100.0                                                      # exp(100) = inf in fp32
    d[:, 7] = -200.0                                                     # exp(-200) = 0
    raw, wt, _ = T.decode(d, boxes)
    assert np.isnan(raw[0, 0]) and np.isnan(raw[0, 2]) and raw[1, 0] == -np.inf and raw[1, 2] == np.inf
    assert np.isnan(wt[0, 0]) and wt[1, 0] == np.inf
    assert raw[0, 5] == raw[0, 7] == 30.0                                # ht = 0: both y at the centre
    got, _, _ = T.decode(d, boxes, True, 100.0, 80.0)
    assert np.isnan(got[0, 0]) and got[1, 0] == 1.0 and got[1, 2] == 100.0
    assert T.same_nonfinite(got, got.copy()) and not T.same_nonfinite(np.nan_to_num(got), got)


def test_decode_bar_accepts_ulps_and_rejects_a_wrong_class():
    rng = np.random.default_rng(3)
    boxes = wl.random_boxes(200, 480, 640, 3).astype(np.float32)
    d = (rng.standard_normal((200, 4 * 21)) * 0.5).astype(np.float32)
    ref, wt, ht = T.decode(d, boxes)
    nudged = np.nextafter(ref, np.float32(np.inf))
    assert T.decode_ratio(nudged, ref, wt, ht)[0] <= 1
    shifted = np.roll(ref.reshape(200, 21, 4), 1, axis=1).reshape(200, -1)
    assert T.decode_ratio(shifted, ref, wt, ht)[0] > 1


@pytest.mark.parametrize("K,C", [(1, 21), (3, 81), (6, 201)])
def test_softmax_mean_reference(K, C):
    rng = np.random.default_rng(K * C)
    x = (rng.standard_normal((K, 50, C)) * 3).astype(np.float32)
    x[:, 0] *= 1e4 / np.abs(x[:, 0]).max()
    x[:, 1] = 0.5
    x[:, 2, 3] = -np.finfo(np.float32).max
    p = T.softmax_mean(x)
    assert np.allclose(p.sum(1), 1.0, rtol=0, atol=1e-12)
    assert np.allclose(p[1], 1.0 / C, rtol=1e-15) and p[2, 3] == 0.0
    e = np.exp(x.astype(np.float64) - x.max(2, keepdims=True))
    assert np.allclose(p, (e / e.sum(2, keepdims=True)).mean(0), rtol=1e-14, atol=0)
    if K == 1:
        assert np.abs(p - O.softmax(x[0])).max() <= 1e-6                # the C oracle's fp32 softmax is inside the bar too
        assert np.all(np.abs(O.softmax(x[0]) - p) <= T.softmax_bar(x))
    bar = T.softmax_bar(x)
    assert np.all(bar >= 1e-6 * p + T.TINY) and np.all(bar[1] == 1e-6 * p[1] + T.TINY)   # equal logits: x - m = 0 is exact


def test_gather_is_strict_and_in_row_order():
    s = np.float32([[0, 0.5], [0, 0.25], [0, 0.75], [0, 0.5], [0, -1]])
    assert T.gather(s, 1, 0.5).tolist() == [2]
    assert T.gather(s, 1, 0.25).tolist() == [0, 2, 3]
    assert T.gather(s, 1, -1.5).tolist() == [0, 1, 2, 3, 4]
    assert T.gather(s, 1, 0.75).size == 0


@pytest.mark.parametrize("thresh", [-1.5, 0.4])
def test_class_keeps_equal_a_per_class_nms_loop(thresh):
    R, C = 700, 11
    rng = np.random.default_rng(11)
    boxes = wl.random_boxes(R, 300, 400, 11).astype(np.float32)
    scores = rng.random((R, C)).astype(np.float32)
    scores[:, 3] = np.floor(scores[:, 3] * 8) / 8                        # ties
    scores[:, 4] = np.float32(0.4)                                       # every score exactly at the threshold
    scores[::3, 5] = np.float32(0.4)
    bboxes = T.decode((rng.standard_normal((R, 4 * C)) * 0.3).astype(np.float32), boxes, True, 400.0, 300.0)[0]
    got = T.class_keeps(scores, bboxes, thresh, 0.3, 2, 9)
    assert len(got) == 7
    for j, k in zip(range(2, 9), got):
        rows = [r for r in range(R) if scores[r, j] > np.float32(thresh)]
        sb = np.float32([[*bboxes[r, 4 * j:4 * j + 4], scores[r, j]] for r in rows]).reshape(-1, 5)
        want = np.int32(rows)[O.nms(sb, 0.3)] if rows else np.zeros(0, np.int32)
        assert np.array_equal(k, want), j
        if O.ref_built():
            assert np.array_equal(sb[O.nms(sb, 0.3)], O.ref_nms_rows(sb, 0.3))
    if thresh == 0.4:
        assert got[4 - 2].size == 0 and not np.isin(np.arange(0, R, 3), got[5 - 2]).any()


def test_rank_ranges_cover_the_classes_once():
    for world in (1, 2, 3, 4, 7, 8):
        rr = T.rank_ranges(80, world)
        assert rr[0][0] == 1 and rr[-1][1] == 81 and all(a[1] == b[0] for a, b in zip(rr, rr[1:]))
    assert T.rank_ranges(80, 3) == [(1, 27), (27, 54), (54, 81)]

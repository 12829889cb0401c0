"""CPU: the training rules through the product's host views (mpn_debug_dropout / _criteria / _sgd, compiled from
csrc/train_rule.cuh) against numpy restatements and hand-computed answers, and the refusals that need no GPU."""
import ctypes as C

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models, train
from _train_ref import criteria, dropout_keep, philox4x32_10, sgd


def lib():
    return mpn.load_library()


def debug_dropout(seed, step, tower, layer, elem0, n, p):
    out = np.empty(n, np.uint8)
    assert lib().mpn_debug_dropout(seed, step, tower, layer, elem0, n, p, out.ctypes.data) == 0
    return out.astype(bool)


def debug_criteria(x, d, labels, t, w=1.0):
    x, d, t = (np.ascontiguousarray(a, np.float32) for a in (x, d, t))
    lab = np.ascontiguousarray(labels, np.int32)
    gx, gd, L = np.empty_like(x), np.empty_like(d), np.empty(3, np.float32)
    rc = lib().mpn_debug_criteria(x.ctypes.data, d.ctypes.data, lab.ctypes.data, t.ctypes.data, x.shape[0], x.shape[1], w,
                                  gx.ctypes.data, gd.ctypes.data, L.ctypes.data)
    return None if rc != 0 else (L, gx, gd)


def test_philox_known_answer():
    """Random123's published vector for philox4x32-10 with a zero counter and key"""
    out = philox4x32_10([np.zeros(1, np.uint64)] * 4, (0, 0))
    assert [int(o[0]) for o in out] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]


@pytest.mark.parametrize("p", [0.5, 0.1, 0.9, 0.0])
def test_dropout_rule_bit_exact(p):
    seed = 0x1234_5678_9ABC_DEF0
    for step, tower, layer, e0 in [(0, 0, 2, 0), (3, 4, 3, 1 << 33), (7, 1, 1, 12345)]:
        got = debug_dropout(seed, step, tower, layer, e0, 4099, p)
        want = dropout_keep(seed, step, tower, layer, np.arange(e0, e0 + 4099, dtype=np.uint64), p)
        assert np.array_equal(got, want)
    if p > 0:
        frac = debug_dropout(555, 0, 0, 2, 0, 1 << 16, p).mean()
        assert abs(frac - (1 - p)) < 0.01
    else:
        assert debug_dropout(555, 0, 0, 2, 0, 1000, p).all()


def test_cross_entropy_known_answers():
    C_ = 3
    x = np.array([[0.0, 0.0, 0.0], [1.0, 2.0, 3.0]], np.float32)
    d = np.zeros((2, 4 * C_), np.float32)
    L, gx, _ = debug_criteria(x, d, [1, 3], np.zeros_like(d))
    ce0 = np.log(3.0)
    ce1 = np.log(np.exp(1) + np.exp(2) + np.exp(3)) - 3.0
    assert abs(L[1] - (ce0 + ce1) / 2) < 1e-6 and L[2] == 0.0 and abs(L[0] - L[1]) < 1e-7
    np.testing.assert_allclose(gx[0], np.array([1 / 3 - 1, 1 / 3, 1 / 3]) / 2, rtol=1e-6)
    sm = np.exp([1.0, 2.0, 3.0]) / np.exp([1.0, 2.0, 3.0]).sum()
    np.testing.assert_allclose(gx[1], (sm - [0, 0, 1]) / 2, rtol=1e-6)


def test_bbox_regression_known_answers():
    """label 2 (foreground): both SmoothL1 branches and |d| = 1 exactly; label 1 (background): its columns are masked out, so
    a non-zero target there still costs and still has a gradient (BBoxRegressionCriterion.lua:38-41); the last class C"""
    C_ = 3
    x = np.zeros((3, C_), np.float32)
    d = np.zeros((3, 4 * C_), np.float32)
    t = np.zeros_like(d)
    d[0, 4:8] = [0.5, 3.0, -2.0, 1.0]                    # row 0, label 2: diffs 0.5, 3, -2, 1
    d[1, 0:4] = [5.0, 5.0, 5.0, 5.0]                     # row 1, label 1: background, input masked to 0
    t[1, 0] = 0.25                                        # off-mask target: diff -0.25
    d[2, 8:12] = [0.0, 0.0, 0.0, 0.0]                    # row 2, label C = 3
    t[2, 8:12] = [0.0, 1.0, -1.5, 0.0]                   # diffs 0, -1, 1.5, 0
    t[2, 4] = 2.0                                         # off-mask target on a foreground row: diff -2
    L, _, gd = debug_criteria(x, d, [2, 1, 3], t, w=2.0)
    row0 = 0.5 * 0.25 + (3 - 0.5) + (2 - 0.5) + 0.5
    row1 = 0.5 * 0.0625
    row2 = 0.5 + 1.0 + (2 - 0.5)
    assert abs(L[2] - (row0 + row1 + row2) / 3) < 1e-6
    assert abs(L[0] - (L[1] + 2.0 * L[2])) < 1e-6
    np.testing.assert_allclose(gd[0, 4:8], np.array([0.5, 1.0, -1.0, 1.0]) / 3 * 2, rtol=1e-6)
    np.testing.assert_allclose(gd[1, 0:4], np.array([-0.25, 0, 0, 0]) / 3 * 2, rtol=1e-6)
    assert np.all(gd[1, 4:] == 0)
    np.testing.assert_allclose(gd[2, 8:12], np.array([0.0, -1.0, 1.0, 0.0]) / 3 * 2, rtol=1e-6)
    np.testing.assert_allclose(gd[2, 4], -1.0 / 3 * 2, rtol=1e-6)


def test_criteria_all_background_and_random_rows():
    rng = np.random.default_rng(0)
    R, C_ = 64, 21
    x = rng.standard_normal((R, C_)).astype(np.float32) * 3
    d = rng.standard_normal((R, 4 * C_)).astype(np.float32)
    t = np.zeros_like(d)
    L, gx, gd = debug_criteria(x, d, np.ones(R, np.int32), t)
    assert L[2] == 0.0 and not np.any(gd)
    labels = rng.integers(1, C_ + 1, R).astype(np.int32)
    for r in range(R):
        if labels[r] > 1:
            t[r, 4 * labels[r] - 4:4 * labels[r]] = rng.standard_normal(4) * 1.5
    L, gx, gd = debug_criteria(x, d, labels, t, 0.7)
    tot, ce, sl1, rgx, rgd = criteria(x, d, labels, t, 0.7)
    assert abs(L[1] - ce) <= 1e-6 * abs(ce) and abs(L[2] - sl1) <= 1e-6 * abs(sl1) and abs(L[0] - tot) <= 1e-6 * abs(tot)
    np.testing.assert_allclose(gx, rgx, rtol=1e-6, atol=1e-9)
    np.testing.assert_allclose(gd, rgd, rtol=1e-6, atol=1e-9)
    assert debug_criteria(x, d, np.full(R, C_ + 1, np.int32), t) is None           # labels out of 1..C
    assert debug_criteria(x, d, np.zeros(R, np.int32), t) is None


def test_sgd_three_steps_and_decay():
    """the recalled optim.sgd: weight decay into the gradient, the first step's buffer is the gradient, then
    buf = m buf + (1 - damp) g; decay scales lr and the buffer; weight decay 0 for biases"""
    rng = np.random.default_rng(1)
    n = 1000
    w0 = rng.standard_normal(n).astype(np.float32)
    gs = [rng.standard_normal(n).astype(np.float32) for _ in range(3)]
    for wd, damp in [(5e-4, 0.0), (0.0, 0.0), (5e-4, 0.25)]:
        lr, mom = 1e-3, 0.9
        w, buf = w0.copy(), np.zeros(n, np.float32)
        rw, rbuf = w0.copy(), np.zeros(n, np.float32)
        for k in range(3):
            assert lib().mpn_debug_sgd(w.ctypes.data, gs[k].ctypes.data, buf.ctypes.data, n, lr, mom, damp, wd, int(k == 0)) == 0
            rw, rbuf = sgd(rw, gs[k], rbuf, lr, mom, damp, wd, k == 0)
            assert np.array_equal(w, rw) and np.array_equal(buf, rbuf)
            if k == 0:
                np.testing.assert_allclose(buf, (gs[0] + np.float32(wd) * w0) if wd else gs[0], rtol=1e-7, atol=0)
            if k == 1:                                                   # decay between steps 2 and 3 (onEndEpoch)
                lr = float(np.float32(lr) * np.float32(0.1)); buf *= np.float32(0.1); rbuf = buf.copy()
    # plain SGD without momentum: w -= lr * g
    w = w0.copy(); b = np.zeros(n, np.float32)
    lib().mpn_debug_sgd(w.ctypes.data, gs[0].ctypes.data, b.ctypes.data, n, 0.5, 0.0, 0.0, 0.0, 1)
    np.testing.assert_allclose(w, w0 - 0.5 * gs[0], rtol=1e-6, atol=1e-7)


def test_graphs_that_train_and_graphs_that_are_refused():
    train.check_spec(models.vgg16_multipathnet(21, seed=None, width_div=4, fc_dim=256))
    train.check_spec(models.vgg16_fast_rcnn(21, seed=None, width_div=4, fc_dim=256))
    with pytest.raises(mpn.MpnError, match="1x1 convolution"):
        train.check_spec(models.resnet50_fast_rcnn(81, seed=None, integral_k=0))
    with pytest.raises(mpn.MpnError, match="integral head"):
        train.check_spec(models.vgg16_multipathnet(21, seed=None, width_div=4, fc_dim=256, integral_k=2))


def test_step_argument_checks():
    spec = models.vgg16_fast_rcnn(21, seed=None, width_div=4, fc_dim=256)
    lim = (64, 192, 256)
    im = np.zeros((3, 128, 176), np.float32)
    rois = np.array([[1, 1, 50, 60]] * 4, np.float32)
    ok = dict(images=[im], rois_per_image=[rois], labels=np.array([1, 2, 21, 5]), bbox_targets=np.zeros((4, 84), np.float32))
    train.check_step(spec, lim, **ok)
    for k, v, msg in [("labels", np.array([1, 2, 22, 5]), "labels"), ("labels", np.array([0, 2, 3, 5]), "labels"),
                      ("rois_per_image", [np.zeros((0, 4), np.float32)], "R = 0"),
                      ("rois_per_image", [np.zeros((65, 4), np.float32)], "R = 65"),
                      ("images", [np.zeros((3, 200, 176), np.float32)], "larger than max_h"),
                      ("images", [np.zeros((3, 128, 300), np.float32)], "larger than max_h"),
                      ("bbox_targets", np.zeros((4, 80), np.float32), "bbox_targets")]:
        a = dict(ok); a[k] = v
        if k == "rois_per_image" and v[0].shape[0] == 65:
            a["labels"] = np.ones(65); a["bbox_targets"] = np.zeros((65, 84), np.float32)
        with pytest.raises(mpn.MpnError, match=msg):
            train.check_step(spec, lim, **a)


def test_config_struct_layout():
    assert C.sizeof(mpn._lib.CTrainConfig) == 6 * 4 + 8

"""CPU: training with the integral loss (K class heads, one trained per step): the graph checks, the per-step set draw
(mpn_integral_set) against a numpy restatement of Philox4x32-10, the donkey threshold rule, and vgg16_fast_rcnn's
integral_k option (integral_k = 0 draws exactly the single-head model's weights)."""
import copy
import hashlib

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models, train
from multipathnet_b200._lib import Head
from multipathnet_b200.batch_provider import integral_set, integral_thresholds
from _train_ref import philox4x32_10

DRAW_INTEGRAL = 5


def _draw_set(seed, step, n_sets):
    """rand_int(draw_u32(seed, step, slot 0, set 0, DRAW_INTEGRAL, draw 0), n_sets) - 1 in numpy"""
    out = philox4x32_10([np.zeros(1, np.uint64), np.full(1, step, np.uint64), np.zeros(1, np.uint64), np.full(1, DRAW_INTEGRAL, np.uint64)],
                        (seed & 0xFFFFFFFF, seed >> 32))
    return int((np.uint64(out[0][0]) * np.uint64(n_sets)) >> np.uint64(32))


def _sha(spec):
    h = hashlib.sha256()
    for w in spec.weights:
        h.update(np.ascontiguousarray(w, np.float32).tobytes())
    return h.hexdigest()


def test_integral_training_is_opt_in():
    """the plain check refuses an integral head as before; the integral check accepts it and every single-head graph"""
    spec = models.vgg16_multipathnet(21, seed=None, width_div=4, fc_dim=256, integral_k=2)
    with pytest.raises(mpn.MpnError, match="integral head"):
        train.check_spec(spec)
    train.check_spec(spec, integral=True)
    train.check_spec(models.vgg16_multipathnet(21, seed=None, width_div=4, fc_dim=256), integral=True)
    train.check_spec(models.vgg16_fast_rcnn(21, seed=None, width_div=4, fc_dim=256), integral=True)
    with pytest.raises(mpn.MpnError, match="1x1 convolution"):
        train.check_spec(models.resnet50_fast_rcnn(81, seed=None, integral_k=3), integral=True)


@pytest.mark.parametrize("kind", ["mpn", "frcnn"])
@pytest.mark.parametrize("k", [2, 6])
def test_integral_specs_pass_the_training_checks(kind, k):
    if kind == "mpn":
        spec = models.vgg16_multipathnet(21, seed=None, width_div=4, fc_dim=256, integral_k=k)
        train.check_spec(spec, integral=True)
        with pytest.raises(mpn.MpnError, match="exactly one tower"):          # MultiPathNet's trunk stays frozen
            train.check_spec(spec, 6, integral=True)
    else:
        spec = models.vgg16_fast_rcnn(21, seed=None, width_div=4, fc_dim=256, integral_k=k)
        train.check_spec(spec, integral=True)
        train.check_spec(spec, spec.trunk_train_from, integral=True)       # trunk training + integral
    assert len(spec.cls_heads) == k and spec.no_softmax == 1


def test_class_heads_over_different_columns_are_refused():
    spec = models.vgg16_multipathnet(21, seed=None, width_div=4, fc_dim=256, integral_k=3)
    bad = copy.deepcopy(spec)
    h = bad.cls_heads[2]
    bad.cls_heads[2] = Head(h.col_begin + 64, h.col_len - 64, h.cout, h.weight, h.bias)       # towers 1-4 minus 64 columns
    with pytest.raises(mpn.MpnError, match="same columns"):
        train.check_spec(bad, integral=True)
    shared = copy.deepcopy(spec)
    h = shared.cls_heads[1]
    shared.cls_heads[1] = Head(h.col_begin, h.col_len, h.cout, spec.cls_heads[0].weight, h.bias)
    with pytest.raises(mpn.MpnError, match="shared"):
        train.check_spec(shared, integral=True)


def test_integral_set_draw_matches_restatement():
    for seed in (555, 1, 0xFEDCBA9876543210):
        for n in (1, 2, 3, 6, 16):
            got = [integral_set(seed, s, n) for s in range(300)]
            assert got == [_draw_set(seed, s, n) for s in range(300)], (seed, n)
            assert set(got) == set(range(n))                                # every set is drawn
            assert got == [integral_set(seed, s, n) for s in range(300)]   # deterministic
    assert [integral_set(555, s, 6) for s in range(40)] != [integral_set(556, s, 6) for s in range(40)]
    with pytest.raises(mpn.MpnError):
        integral_set(555, 0, 0)


def test_integral_draw_is_disjoint_from_the_sampler_draws():
    """purpose 5 gives other words than the image / flip / bg / fg draws (1-4) of the same (seed, step, slot 0, set 0)"""
    out = [philox4x32_10([np.zeros(1, np.uint64), np.full(1, 9, np.uint64), np.zeros(1, np.uint64), np.full(1, p, np.uint64)],
                         (555, 0))[0][0] for p in range(1, 6)]
    assert len(set(int(v) for v in out)) == 5


def test_integral_thresholds_follow_the_donkey_rule():
    t = integral_thresholds(6)
    assert len(t) == 6
    for i, (fg, lo, hi) in enumerate(t):                                    # donkey.lua:38-45, i = loader - 1
        assert fg == 0.5 + i / 20 and hi == fg and lo == 0.1
    assert integral_thresholds(1) == ((0.5, 0.1, 0.5),)
    assert integral_thresholds(2, bg_lo=0.0, bg_hi=0.4) == ((0.4, 0.0, 0.4), (0.4 + 1 / 20, 0.0, 0.4 + 1 / 20))
    with pytest.raises(mpn.MpnError):
        integral_thresholds(0)


@pytest.mark.parametrize("args,digest", [
    (dict(num_classes=21, seed=5, width_div=4, fc_dim=256), "ae6d18e4a61d8974ad89ce9237c1026586aea8efffb70daf3a6535f0cdca920c"),
    (dict(num_classes=81, seed=1234, width_div=8, fc_dim=512), "2b8b5d7a77452b2ddcbee112f2ec7c81ea17302880cc421ab2b582296c9abdab"),
])
def test_fast_rcnn_without_integral_heads_keeps_its_weights(args, digest):
    """the digests were taken from vgg16_fast_rcnn before it had integral_k"""
    s0 = models.vgg16_fast_rcnn(**args)
    s1 = models.vgg16_fast_rcnn(**args, integral_k=0)
    assert _sha(s0) == digest and _sha(s1) == digest
    assert len(s0.cls_heads) == 1 and s0.no_softmax == 0


def test_fast_rcnn_integral_heads_are_drawn_in_turn():
    """integral_k = 3: the trunk, fc6 / fc7 and head 0 are the single-head model's, heads 1, 2 and the bbox head follow"""
    s0 = models.vgg16_fast_rcnn(21, seed=5, width_div=4, fc_dim=256)
    s3 = models.vgg16_fast_rcnn(21, seed=5, width_div=4, fc_dim=256, integral_k=3)
    assert len(s3.cls_heads) == 3 and s3.no_softmax == 1
    assert len(s3.weights) == len(s0.weights) + 4
    h0 = s0.cls_heads[0]
    for i in range(h0.weight + 1):                                          # everything up to head 0's weight
        assert np.array_equal(s0.weights[i], s3.weights[i])
    for h in s3.cls_heads:
        assert (h.col_begin, h.col_len, h.cout) == (s3.bbox_head.col_begin, s3.bbox_head.col_len, 21)
    ws = [s3.weights[h.weight] for h in s3.cls_heads]
    assert not np.array_equal(ws[0], ws[1]) and not np.array_equal(ws[1], ws[2])
    assert s3.bbox_head.weight > max(h.bias for h in s3.cls_heads)

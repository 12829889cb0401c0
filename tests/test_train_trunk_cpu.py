"""CPU: which trunk layers the model builders train, the library's refusals of trunk training (mpn_train_check),
and the numpy argmax rules the trunk-training oracle restates (max pool and ROI pooling) on hand-made maps."""
import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from multipathnet_b200.train import check_spec
from _train_trunk_ref import FLT_MAX, pool_argmax, roi_argmax, roi_backward, roi_bin_windows


def test_builders_trunk_train_from():
    s = models.vgg16_fast_rcnn(21, seed=None)
    assert s.trunk_train_from == 6
    L = s.trunk_layers[6]
    assert L.kind == mpn._lib.MPN_LAYER_CONV and L.cin == 128 and L.cout == 256          # conv3_1, after conv1_*, pool1, conv2_*, pool2
    assert [l.kind for l in s.trunk_layers[:6]].count(mpn._lib.MPN_LAYER_MAXPOOL) == 2
    assert models.vgg16_multipathnet(81, seed=None).trunk_train_from == 0
    assert models.resnet50_fast_rcnn(81, seed=None).trunk_train_from == 0
    check_spec(s, s.trunk_train_from)
    check_spec(models.vgg16_fast_rcnn(21, seed=None, width_div=4, fc_dim=256), 6)


def test_check_config_refusals():
    s = models.vgg16_fast_rcnn(21, seed=None)
    n = len(s.trunk_layers)
    for k in (-1, n, n + 5):
        with pytest.raises(mpn.MpnError, match="out of range"):
            check_spec(s, k)
    check_spec(s, 0)                                                  # frozen
    with pytest.raises(mpn.MpnError, match="exactly one tower"):
        check_spec(models.vgg16_multipathnet(81, seed=None), 6)
    t = models.vgg16_fast_rcnn(21, seed=None)
    t.towers[0].levels = [(t.taps["conv4"], 1.0 / 8)]                  # pools from a slot below the last trunk layer
    with pytest.raises(mpn.MpnError, match="pool its ROIs from the last trunk layer"):
        check_spec(t, 6)
    r = models.resnet50_fast_rcnn(81, seed=None, integral_k=0)
    with pytest.raises(mpn.MpnError, match="3x3 / stride 1 / pad 1 convolution"):
        check_spec(r, 1)
    # a stride-2 or residual convolution inside the trained range
    for field, val in (("stride", 2), ("residual_slot", 3), ("relu", 0)):
        t = models.vgg16_fast_rcnn(21, seed=None)
        setattr(t.trunk_layers[8], field, val)
        with pytest.raises(mpn.MpnError, match="3x3 / stride 1"):
            check_spec(t, 6)
        check_spec(t, 9)                                              # below the trained range: not trained, not checked
    t = models.vgg16_fast_rcnn(21, seed=None)
    t.trunk_layers[9].kh = 3
    with pytest.raises(mpn.MpnError, match="max pool"):
        check_spec(t, 6)


def test_pool_argmax_ties_and_clipped_windows():
    y = np.array([[[1, 3, 3, 0, 5],
                   [3, 2, 1, 3, 4],
                   [7, 7, 2, 2, 9]]], np.float32)                    # 3 x 5: ceil mode, windows clipped at the edges
    idx = pool_argmax(y)
    assert idx.shape == (1, 2, 3)
    # (0, 0): 1 3 / 3 2 -> the first 3 in row-major order; (0, 1): 3 0 / 1 3 -> the first 3; (0, 2): 5 / 4 -> clipped
    # (1, 0): 7 7 -> the first; (1, 1): 2 2 -> the first; (1, 2): 9 alone
    assert idx.tolist() == [[[1, 2, 4], [10, 12, 14]]]
    z = np.zeros((2, 1, 1), np.float32)
    assert pool_argmax(z).tolist() == [[[0]], [[0]]]
    n = np.full((1, 2, 2), -FLT_MAX, np.float32)
    assert pool_argmax(n).tolist() == [[[-1]]]                       # nothing is > -FLT_MAX


def test_roi_argmax_rules():
    H, W = 4, 6
    f = np.zeros((2, H, W), np.float32)
    f[0] = [[0, 1, 1, 0, 0, 0],
            [1, 1, 0, 0, 2, 2],
            [0, 0, 0, 0, 2, 0],
            [0, 0, 0, 0, 0, 3]]
    f[1] = -1.0
    # one bin over the whole map (scale 1, 1-based boxes, variant 2: ends exclusive of the last pixel)
    am = roi_argmax(f, [(1, 1, 7, 5)], 1.0, 2, 1, 1)
    assert am.shape == (1, 1, 2)
    assert am[0, 0, 0] == 3 * W + 5 and am[0, 0, 1] == 0            # the max; all equal -> the first cell
    # 2 x 2 bins: ties go to the first cell in scan order
    am = roi_argmax(f, [(1, 1, 7, 5)], 1.0, 2, 2, 2)
    win = roi_bin_windows((1, 1, 7, 5), 1.0, 2, 2, 2, H, W)
    assert win == [(0, 2, 0, 3), (0, 2, 3, 6), (2, 4, 0, 3), (2, 4, 3, 6)]
    assert am[0, :, 0].tolist() == [1, 10, 12, 23]
    # a ROI outside the map: every bin empty -> -1; the backward names no cell
    am = roi_argmax(f, [(40, 40, 60, 60)], 1.0, 2, 2, 2)
    assert (am == -1).all()
    assert not roi_backward(np.ones((1, 4, 2), np.float32), am, H, W).any()
    # many bins naming one cell: summed in (r, bin) order
    am = roi_argmax(f, [(5, 2, 7, 5), (5, 2, 7, 5)], 1.0, 2, 2, 2)
    g = np.arange(1, 17, dtype=np.float32).reshape(2, 4, 2)
    got = roi_backward(g, am, H, W)
    want = np.zeros((2, H, W), np.float32)
    for r in range(2):
        for b in range(4):
            for c in range(2):
                if am[r, b, c] >= 0:
                    want[c].flat[am[r, b, c]] += g[r, b, c]
    assert np.array_equal(got, want)
    assert got[0, 1, 4] > 0


def test_t7_readers_take_the_trunk_range_from_the_nobackprop_prefix():
    """utils.disableFeatureBackprop wraps the trunk's first modules in nn.NoBackprop (model_utils.lua:95-103): both
    readers count the trunk layers made inside it (ReLUs fused) as trunk_train_from; a prefix covering the whole trunk
    (multipathnet.lua:60-62) gives 0"""
    from multipathnet_b200 import t7
    from test_t7_cpu import _tiny_fast_rcnn, _roundtrip
    from test_t7_graphs_cpu import _tiny_multipathnet, _tiny_resnet
    model, _ = _tiny_fast_rcnn(np.random.default_rng(5))                # NoBackprop{conv, ReLU, conv, ReLU, pool}, conv, ReLU
    for read in (t7.fast_rcnn_from_t7, t7.model_from_t7):
        spec = read(_roundtrip(model))
        assert [l.kind for l in spec.trunk_layers] == [1, 1, 2, 1] and spec.trunk_train_from == 3
        check_spec(spec, spec.trunk_train_from)
    spec = t7.model_from_t7(_roundtrip(_tiny_multipathnet(np.random.default_rng(1))))
    assert spec.trunk_train_from == 0
    spec = t7.model_from_t7(_roundtrip(_tiny_resnet(np.random.default_rng(2))))   # NoBackprop{conv1, bn, relu, pool, layer1}
    k = spec.trunk_train_from
    assert 0 < k < len(spec.trunk_layers)
    assert k == 2 + 2 * 3 + 1                                             # conv1 (bn folded), pool, 2 bottlenecks of 3 convs + 1 shortcut
    with pytest.raises(mpn.MpnError, match="3x3 / stride 1 / pad 1 convolution"):
        check_spec(spec, k)
    # a trunk without NoBackprop, and the exporter's round trip of the builders' range
    plain = t7.T7Object(model.typename, dict(model.fields))
    par = plain.modules[0]
    dpt = par.modules[0]
    flat = t7.flatten_sequential(dpt)
    plain.fields["modules"] = [t7.T7Object(par.typename, {"modules": [t7.T7Object("nn.Sequential", {"modules": flat}), par.modules[1]]})] + \
        list(model.modules[1:])
    assert t7.fast_rcnn_from_t7(_roundtrip(plain)).trunk_train_from == 0
    s = models.vgg16_fast_rcnn(21, seed=1, width_div=8, fc_dim=64)
    back = t7.model_from_t7(_roundtrip(t7.model_to_t7(s)))
    assert back.trunk_train_from == 6 and t7.fast_rcnn_from_t7(_roundtrip(t7.model_to_t7(s))).trunk_train_from == 6

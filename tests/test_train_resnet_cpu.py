"""CPU: the fixed-batch-norm ResNet builders (models.resnet{18,50}_fast_rcnn(fixed_bn=True)), the ConstAffine records of
model_from_t7, and the host-only graph check mpn_train_check with fixed-batch-norm records (accepts, refusals,
unrecorded models' messages)."""
import hashlib

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models, t7
from multipathnet_b200._lib import MPN_LAYER_AVGPOOL, MPN_LAYER_CONV
from multipathnet_b200.train import check_spec


def _convs(layers):
    return [L for L in layers if L.kind == MPN_LAYER_CONV]


@pytest.mark.parametrize("which", ["r18", "r50"])
def test_builders_record_exactly_layer2_to_layer4(which):
    if which == "r18":
        s = models.resnet18_fast_rcnn(81, seed=None, fixed_bn=True)
        per_block, first_train = (2, 3), 2 + 2 * 2                     # layer1: two basic blocks of two convolutions
        n_trunk = 2 + 2 * 2 + 2 * 5
    else:
        s = models.resnet50_fast_rcnn(81, seed=None, fixed_bn=True)
        per_block, first_train = (3, 4), 2 + 4 + 3 + 3
        n_trunk = 2 + 4 + 3 + 3 + (4 + 3 * 3) + (4 + 5 * 3)
    assert len(s.trunk_layers) == n_trunk and s.trunk_train_from == first_train
    assert s.trunk_layers[first_train].in_slot == s.trunk_layers[first_train - 1].out_slot   # layer2's first reads layer1's output
    trunk_rec = {L.weight for L in _convs(s.trunk_layers[first_train:])}
    tower_rec = {L.weight for L in _convs(s.towers[0].layers)}
    assert set(s.fixed_bn) == trunk_rec | tower_rec
    assert not ({L.weight for L in _convs(s.trunk_layers[:first_train])} & set(s.fixed_bn))
    assert s.towers[0].layers[-1].kind == MPN_LAYER_AVGPOOL
    for i, a in s.fixed_bn.items():
        assert a.shape == (s.weights[i].shape[0],) and a.dtype == np.float32


def test_fixed_bn_weights_are_the_folded_product():
    """W' = fl(a * W) for every record: the builder's draw restated with the same generator"""
    s = models.resnet18_fast_rcnn(5, seed=3, integral_k=0, blocks=(1, 1, 1, 1), fixed_bn=True)
    recs = {}

    class Spy(models._W):
        def conv_fixed_bn(self, cout, cin, kh, kw, gain=1.0):
            std = gain * np.sqrt(2.0 / (cin * kh * kw) / 1.75)
            w = self.rng.standard_normal((cout, cin, kh, kw), dtype=np.float32) * np.float32(std)
            a = self.rng.uniform(0.5, 2.0, cout).astype(np.float32)
            b = self.rng.standard_normal(cout, dtype=np.float32) * np.float32(0.05)
            i = self.add(a[:, None, None, None] * w)
            recs[i] = (w, a)
            return i, self.add(b), a
    orig = models._W
    models._W = Spy
    try:
        s2 = models._resnet_fast_rcnn("x", False, 5, 3, 0, (1, 1, 1, 1), True)
    finally:
        models._W = orig
    assert set(recs) == set(s.fixed_bn)
    for i, (w, a) in recs.items():
        want = (a[:, None, None, None] * w).astype(np.float32)
        assert np.array_equal(s.weights[i].view(np.uint32), want.view(np.uint32)) and np.array_equal(s.fixed_bn[i], a)
    assert all(np.array_equal(x, y) for x, y in zip(s.weights, s2.weights))


def test_fixed_bn_false_builds_the_same_resnet50_as_before():
    """the default draws exactly the weights inference has always run (digest of the parent's builder)"""
    s = models.resnet50_fast_rcnn(num_classes=21, seed=5, integral_k=3, blocks=(1, 1, 1, 1))
    h = hashlib.sha256()
    for w in s.weights:
        h.update(np.ascontiguousarray(w, np.float32).tobytes())
    assert h.hexdigest() == "b416298efe39cd30c14183b45e593b24a968c86da7f7308f1a04b2a5017477f7"
    assert s.fixed_bn == {} and s.trunk_train_from == 0
    s18 = models.resnet18_fast_rcnn(5, seed=None)
    assert s18.fixed_bn == {} and s18.trunk_train_from == 0


def test_check_accepts_the_recorded_resnets():
    for s in (models.resnet18_fast_rcnn(5, seed=None, integral_k=0, fixed_bn=True),
              models.resnet50_fast_rcnn(5, seed=None, integral_k=0, blocks=(1, 1, 1, 1), fixed_bn=True)):
        check_spec(s)
        check_spec(s, s.trunk_train_from)
        with pytest.raises(mpn.MpnError, match="integral"):
            check_spec(models.resnet18_fast_rcnn(5, seed=None, integral_k=3, fixed_bn=True), s.trunk_train_from)
    s = models.resnet18_fast_rcnn(5, seed=None, integral_k=3, fixed_bn=True)
    check_spec(s, s.trunk_train_from, integral=True)


def test_unrecorded_resnets_keep_todays_messages():
    s = models.resnet50_fast_rcnn(5, seed=None, integral_k=0)
    with pytest.raises(mpn.MpnError, match="1x1 convolution"):
        check_spec(s)
    s = models.resnet18_fast_rcnn(5, seed=None, integral_k=0)
    with pytest.raises(mpn.MpnError, match="1x1 convolution"):
        check_spec(s)


def test_refusals_of_the_fixed_bn_check():
    base = models.resnet18_fast_rcnn(5, seed=None, integral_k=0, blocks=(1, 1, 1, 1), fixed_bn=True)
    # trunk_from inside layer1 / at conv1 / at the max pool: an unrecorded layer keeps today's trunk message
    for k in (1, 2, 3):
        with pytest.raises(mpn.MpnError, match="3x3 / stride 1"):
            check_spec(base, k)
    # a recorded 5x5, or stride 3, convolution
    for field, val in (("kh", 5), ("stride", 3)):
        s = models.resnet18_fast_rcnn(5, seed=None, integral_k=0, blocks=(1, 1, 1, 1), fixed_bn=True)
        L = s.towers[0].layers[0]
        setattr(L, field, val)
        if field == "kh":
            L.kw, L.pad = 5, 2
        with pytest.raises(mpn.MpnError, match="fixed-batch-norm layer"):
            check_spec(s)
    # a record that names no convolution
    s = models.resnet18_fast_rcnn(5, seed=None, integral_k=0, blocks=(1, 1, 1, 1), fixed_bn=True)
    s.fixed_bn[s.bbox_head.weight] = np.ones(s.bbox_head.cout, np.float32)
    with pytest.raises(mpn.MpnError, match="names no convolution"):
        check_spec(s)
    # a tower that does not end in an AVGPOOL
    s = models.resnet18_fast_rcnn(5, seed=None, integral_k=0, blocks=(1, 1, 1, 1), fixed_bn=True)
    s.towers[0].layers[-1].kind = MPN_LAYER_CONV
    with pytest.raises(mpn.MpnError):
        check_spec(s)


def test_model_from_t7_records_const_affine_after_a_bias_free_convolution():
    from test_t7_graphs_cpu import _tiny_resnet
    rng = np.random.default_rng(21)
    spec = t7.model_from_t7(_tiny_resnet(rng))
    convs = {L.weight: L for L in spec.trunk_layers + spec.towers[0].layers if L.kind == MPN_LAYER_CONV}
    assert set(spec.fixed_bn) <= set(convs)
    k = spec.trunk_train_from
    trained_trunk = {L.weight for L in _convs(spec.trunk_layers[k:])}
    # _tiny_resnet: conv1 + layer1 and layer4's second block carry ConstAffine, layer2 / layer3 / layer4's first raw BN
    assert not (trained_trunk & set(spec.fixed_bn))
    tw = [L.weight for L in _convs(spec.towers[0].layers)]
    assert set(tw[-3:]) <= set(spec.fixed_bn) and not (set(tw[:-3]) & set(spec.fixed_bn))
    assert {L.weight for L in _convs(spec.trunk_layers[:k])} <= set(spec.fixed_bn)
    # a convolution with its own bias before a ConstAffine gets no record; the folded arrays do not depend on records
    from test_t7_graphs_cpu import O, _seq, _conv
    conv = _conv(np.random.default_rng(1), 8, 64, 3, bias=True)
    aff = O("inn.ConstAffine", a=np.full(64, 2.0, np.float32), b=np.zeros(64, np.float32))
    arrays = []

    def add(a):
        arrays.append(np.ascontiguousarray(a, np.float32))
        return len(arrays) - 1
    ev = t7._Layers(add, arrays, 8, (5, 5))
    ev.run(_seq(conv, aff), 0)
    assert ev.fixed_bn == {} and np.array_equal(arrays[0], (conv.weight * 2.0).astype(np.float32))

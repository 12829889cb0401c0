"""CPU: Network-in-Network Fast R-CNN (models.nin_fast_rcnn, models/nin.lua on imagenet-multiGPU.torch's `ninbn`): the
builder's shapes and FLOP counts, the host view of its plans (the K tail of the 96-channel layers, the 5 x 5), the
description and training checks, and the import of a hand-built nin.lua graph."""
import ctypes

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, t7
from multipathnet_b200._lib import MPN_LAYER_AVGPOOL, MPN_LAYER_CONV, MPN_LAYER_MAXPOOL
from multipathnet_b200.train import check_spec
from oracle import graphs as G
from test_t7_graphs_cpu import O, _bn, _both, _cat, _close, _conv, _ident, _linear, _par, _pool, _relu, _seq


def _geometry(layers):
    return [(L.kind, L.kh, L.kw, L.stride, L.pad, L.relu, L.ceil_mode if L.kind == MPN_LAYER_MAXPOOL else 0) for L in layers]


def test_builder_shapes_at_224():
    spec = models.nin_fast_rcnn(21, seed=3)
    assert len(spec.trunk_layers) == 11 and spec.transformer == "imagenet" and spec.trunk_train_from == 0 and not spec.fixed_bn
    assert [L.cin for L in spec.trunk_layers if L.kind == MPN_LAYER_CONV] == [3, 96, 96, 96, 256, 256, 256, 384, 384]
    img = np.random.default_rng(0).standard_normal((3, 224, 224)).astype(np.float32)
    ts = G.trunk_forward(spec, img)
    top, scale = spec.towers[0].levels[0]
    assert tuple(ts[top].shape) == (1, 384, 14, 14) and scale == 1 / 16 and spec.taps["block3"] == top
    t = spec.towers[0]
    assert (t.pooled_w, t.pooled_h) == (7, 7) and t.layers[-1].kind == MPN_LAYER_AVGPOOL
    slots = G._run_layers(t.layers, {0: torch.zeros(3, 384, 7, 7)}, spec.weights)
    assert tuple(slots[t.out_slot].shape) == (3, 1024)
    assert spec.cls_heads[0].col_len == 1024 and spec.bbox_head.cout == 84


def test_flop_counts():
    spec = models.nin_fast_rcnn(21, seed=None)

    def conv(cin, cout, k, h, w):
        return 2.0 * cin * cout * k * k * h * w

    def trunk(h1, w1, h2, w2, h3, w3):
        return (conv(3, 96, 11, h1, w1) + 2 * conv(96, 96, 1, h1, w1) + conv(96, 256, 5, h2, w2) + 2 * conv(256, 256, 1, h2, w2)
                + conv(256, 384, 3, h3, w3) + 2 * conv(384, 384, 1, h3, w3))
    assert models.trunk_flops(spec, 224, 224) == trunk(56, 56, 28, 28, 14, 14)
    assert models.trunk_flops(spec, 600, 1000) == trunk(150, 250, 75, 125, 38, 63)
    per_roi = conv(384, 1024, 3, 7, 7) + 2 * conv(1024, 1024, 1, 7, 7) + 2.0 * 1024 * (21 + 84)
    assert models.head_flops_per_roi(spec) == per_roi
    assert abs(per_roi * 1000 / 1e12 - 0.553) < 1e-3 and abs(conv(3, 96, 11, 150, 250) / 1e9 - 2.6) < 0.05
    assert models.w16_flops_per_roi(spec) == 0.0                  # no Linear on a 1 x 1 map: the tower keeps BF16X3


def test_build_desc_accepts_both_forms():
    for fb in (False, True):
        spec = models.nin_fast_rcnn(21, seed=None, fixed_bn=fb)
        d, _ = mpn.Model.build_desc(spec)
        assert d.n_trunk_layers == 11 and d.n_towers == 1 and d.n_tower_layers == 4 and d.bbox_head.cout == 84


def test_fixed_bn_form():
    spec = models.nin_fast_rcnn(21, seed=2, fixed_bn=True)
    convs = [L for L in spec.trunk_layers + spec.towers[0].layers if L.kind == MPN_LAYER_CONV]
    assert set(spec.fixed_bn) == {L.weight for L in convs[3:]}         # blocks 2-4 recorded, block 1 folded
    assert spec.trunk_train_from == 4 and spec.trunk_layers[4].kh == 5  # block 2's 5x5 (disableFeatureBackprop(features, 10))
    plain = models.nin_fast_rcnn(21, seed=2)
    assert _geometry(plain.trunk_layers) == _geometry(spec.trunk_layers)


def _plan(lib, N, Cin, H, W, Cout, k, s, p, per_roi=0):
    out = (ctypes.c_int32 * 8)()
    rc = lib.mpn_debug_plan(N, Cin, H, W, Cout, k, s, p, per_roi, 132, out)
    return rc, dict(zip(("mode", "cg", "bn", "splitk", "streamk", "tn", "th", "tw"), out))


def test_planner_choices_for_nin_at_600x1000():
    """host view of conv_tc_plan on a 132-SM device: the tailed layers (block 1's 1x1s and block 2's 5x5 read 96
    channels: two K blocks per tap, the second half zero) and the rest of the graph"""
    lib = mpn.load_library()
    want = {  # layer: (args, mode, bn, splitk, (tn, th, tw))
        "block1 1x1 (96, tail)": ((1, 96, 150, 250, 96, 1, 1, 0), 0, 64, 1, (1, 1, 128)),
        "block2 5x5 (96, tail)": ((1, 96, 75, 125, 256, 5, 1, 2), 0, 64, 1, (1, 1, 128)),
        "block3 3x3": ((1, 256, 38, 63, 384, 3, 1, 1), 1, 128, 1, (1, 16, 8)),
        "block3 1x1": ((1, 384, 38, 63, 384, 1, 1, 0), 0, 64, 1, (1, 1, 128)),
    }
    for name, (args, mode, bn, sk, patch) in want.items():
        rc, pl = _plan(lib, *args)
        assert rc == 0 and (pl["mode"], pl["bn"], pl["splitk"], (pl["tn"], pl["th"], pl["tw"])) == (mode, bn, sk, patch), (name, pl)
    for args, bn in (((1000, 384, 7, 7, 1024, 3, 1, 1), 256), ((1000, 1024, 7, 7, 1024, 1, 1, 0), 256)):
        rc, pl = _plan(lib, *args, per_roi=1)
        assert rc == 0 and pl["bn"] == bn and pl["splitk"] == 1
    # a tail with a 3x3 / stride 1 kernel keeps the 16 x 8 patches (mode 1): the tail lives in the K loop, not in the patch
    rc, pl = _plan(lib, 1, 24, 30, 30, 64, 3, 1, 1)
    assert rc == 0 and pl["mode"] == 1
    # the tail's K blocks are counted: the same layer with Cin rounded up to 128 plans alike
    assert _plan(lib, 1, 96, 75, 125, 256, 5, 1, 2)[1] == _plan(lib, 1, 128, 75, 125, 256, 5, 1, 2)[1]


def test_planner_refuses_cin_not_a_multiple_of_8():
    lib = mpn.load_library()
    for cin in (3, 20, 100):
        assert _plan(lib, 1, cin, 30, 30, 64, 3, 1, 1)[0] != 0


def test_training_checks():
    spec = models.nin_fast_rcnn(5, seed=None, fixed_bn=True)
    check_spec(spec, 0)                                                 # block 4 and the heads, through the fixed-BN path
    check_spec(models.nin_fast_rcnn(5, seed=None, fixed_bn=True, integral_k=2), 0, integral=True)
    with pytest.raises(mpn.MpnError, match="fixed-batch-norm layer"):   # train_trunk: block 2's recorded 5x5
        check_spec(spec, spec.trunk_train_from)


# ---------------------------------------------------------------- nin.lua's graph, hand-built at tiny widths
def _block(rng, cin, cout, k, s, p, fixed):
    """conv -> BN -> ReLU -> (1x1 conv -> BN -> ReLU) x 2; BN raw (under NoBackprop, folded on import) or inn.ConstAffine
    after a bias-free convolution (BNtoFixed)"""
    mods = []
    for ci, kk, ss, pp in ((cin, k, s, p), (cout, 1, 1, 0), (cout, 1, 1, 0)):
        mods += [_conv(rng, ci, cout, kk, ss, pp, bias=not fixed), _bn(rng, cout, fixed), _relu()]
    return mods


def _tiny_nin(rng, C=4, widths=(24, 32, 48, 64)):
    """nin.lua: features 1..29 (block 1 under NoBackprop: disableFeatureBackprop(features, 10)), ROIPooling(7, 7, 1/16),
    classifier 31..40 + View, classAndBBoxLinear. widths[0] = 24 leaves a tail in a 64-channel K block, as 96 does."""
    a, b, c, d = widths
    feats = (_block(rng, 3, a, 11, 4, 5, False) + [_pool(3, 2, 1, ceil=False)] + _block(rng, a, b, 5, 1, 2, True)
             + [_pool(3, 2, 1, ceil=False)] + _block(rng, b, c, 3, 1, 1, True))
    assert len(feats) == 29
    features = _seq(O("nn.NoBackprop", modules=[_seq(*feats[:10])]), *feats[10:])
    classifier = _seq(*_block(rng, c, d, 3, 1, 1, True), O("nn.SpatialAveragePooling", kW=7, kH=7, dW=1, dH=1, padW=0, padH=0),
                      O("nn.View", size=[d], numInputDims=3))
    return _seq(_par(features, _ident()), O("inn.ROIPooling", W=7, H=7, spatial_scale=1 / 16.0), classifier,
                _cat(_linear(rng, C, d, 0.05), _linear(rng, 4 * C, d, 0.02)))


def test_nin_graph_import_matches_the_builder(oracle_built):
    rng = np.random.default_rng(17)
    model = _tiny_nin(rng)
    img = (rng.standard_normal((3, 96, 128)) * 2).astype(np.float32)
    R = 5
    x1, y1 = rng.uniform(1, 60, R), rng.uniform(1, 40, R)
    rois = np.stack([np.ones(R), x1, y1, x1 + rng.uniform(16, 60, R), y1 + rng.uniform(16, 50, R)], 1).astype(np.float32)
    # saved, loaded, imported; vs the modules' own evaluation. nin.lua returns its ImagenetTransformer beside the graph,
    # which holds no transformer, so the caller names it
    spec, (rc, rb), (c, b) = _both(model, img, rois, transformer="imagenet")
    assert _close(c, rc, 5e-5) and _close(b, rb, 5e-5)
    ref = models.nin_fast_rcnn(4, seed=None, fixed_bn=True)
    assert _geometry(spec.trunk_layers) == _geometry(ref.trunk_layers)
    assert _geometry(spec.towers[0].layers) == _geometry(ref.towers[0].layers)
    tw, rt = spec.towers[0], ref.towers[0]
    assert (tw.pooled_w, tw.pooled_h, tw.levels[0][1], tw.normalize) == (rt.pooled_w, rt.pooled_h, rt.levels[0][1], rt.normalize)
    assert tw.levels[0][0] == spec.trunk_layers[-1].out_slot
    assert [L.cin for L in spec.trunk_layers if L.kind == MPN_LAYER_CONV] == [3, 24, 24, 24, 32, 32, 32, 48, 48]
    # the fixed-batch-norm records: every convolution of blocks 2-4, none of block 1; the trunk trains from block 2's 5x5
    convs = [L for L in spec.trunk_layers + spec.towers[0].layers if L.kind == MPN_LAYER_CONV]
    assert set(spec.fixed_bn) == {L.weight for L in convs[3:]}
    assert spec.trunk_train_from == ref.trunk_train_from == 4
    assert spec.transformer == "imagenet" and spec.has_bbox_norm == 0
    mpn.Model.build_desc(spec)
    check_spec(spec, 0)              # the graph rules; a trained layer's width is checked when training begins (GPU)
    with pytest.raises(mpn.MpnError, match="fixed-batch-norm layer"):
        check_spec(spec, spec.trunk_train_from)

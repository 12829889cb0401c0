"""CaffeNet Fast R-CNN on the host: the builder's graph (slot sizes, FLOP counts), its mpn_layer_ext records, the host
build of csrc/lrn_rule.cuh against the numpy restatement and fp64, the .t7 reader and writer on grouped convolutions
and the three LRN modules, the importer's refusals, and the Lua shim."""
import ctypes as C
import io
import os

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, t7
from multipathnet_b200._lib import CLayerExt, MPN_LAYER_CONV, MPN_LAYER_LRN, Model, MpnError

import _caffenet_ref as CR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _shapes(spec, H, W):
    shp = {0: (3, H, W)}
    for L in spec.trunk_layers:
        c, h, w = shp[L.in_slot]
        if L.kind == MPN_LAYER_CONV:
            shp[L.out_slot] = (L.cout, (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1)
        elif L.kind == MPN_LAYER_LRN:
            shp[L.out_slot] = (c, h, w)
        else:
            po = lambda n: -(-(n - L.kh) // L.stride) + 1        # ceil mode, no pad (every window starts inside)
            shp[L.out_slot] = (c, po(h), po(w))
    return shp


def test_builder_slot_shapes_and_flops():
    s = models.alexnet_fast_rcnn(21, seed=None)
    assert _shapes(s, 224, 224)[9] == (256, 13, 13)
    shp = _shapes(s, 600, 1000)
    assert shp[1] == (96, 148, 248) and shp[2] == (96, 74, 124) and shp[3] == (96, 74, 124)
    assert shp[5] == (256, 37, 62) and shp[9] == (256, 37, 62)
    # independent walk: per group Cin / G input channels
    fl = 0.0
    for L in s.trunk_layers:
        if L.kind == MPN_LAYER_CONV:
            _, h, w = shp[L.out_slot]
            fl += 2.0 * (L.cin // L.groups) * L.cout * L.kh * L.kw * h * w
    assert models.trunk_flops(s, 600, 1000) == pytest.approx(fl, rel=1e-12)
    assert abs(fl / 1e9 - 17.33) < 0.01
    assert abs(models.head_flops_per_roi(s) / 1e6 - 109.9) < 0.1


def test_default_weights_unchanged_by_first_gain():
    a, b = models.alexnet_fast_rcnn(21, seed=1), models.alexnet_fast_rcnn(21, seed=1, first_gain=1.0 / 64)
    assert all(np.array_equal(x, y) for x, y in zip(a.weights, b.weights))
    c = models.alexnet_fast_rcnn(21, seed=1, first_gain=0.5)
    assert np.array_equal(c.weights[0], a.weights[0] * np.float32(32)) or np.allclose(c.weights[0], a.weights[0] * 32, rtol=1e-6)
    assert all(np.array_equal(x, y) for x, y in zip(a.weights[1:], c.weights[1:]))


def test_records_groups_only_on_conv2_4_5_and_build_desc_refuses():
    s = models.alexnet_fast_rcnn(21, seed=None)
    recs = Model.layer_ext(s)
    assert [(r.tower, r.layer, r.groups, r.pad_w, r.out_c_total, r.exclude_pad) for r in recs] == \
        [(-1, 3, 2, 2, 0, 0), (-1, 7, 2, 1, 0, 0), (-1, 8, 2, 1, 0, 0)]
    assert [i for i, L in enumerate(s.trunk_layers) if L.kind == MPN_LAYER_LRN] == [2, 5]
    assert all(s.trunk_layers[i].ext(-1, i) is None for i in (2, 5))
    assert C.sizeof(CLayerExt) == 6 * 4
    with pytest.raises(MpnError, match="grouped convolution"):
        Model.build_desc(s)
    d, _ = Model.build_desc(s, grouped=True)
    assert d.n_trunk_layers == 9 and d.trunk_layers[2].kind == MPN_LAYER_LRN and d.trunk_layers[3].cin == 96
    assert models.caffenet_layer(s) == "trunk layer 2 (LRN)" and models.is_inference_only(s) == "trunk layer 2"


def test_training_check_refuses_caffenet_by_name():
    s = models.alexnet_fast_rcnn(21, seed=None)
    with pytest.raises(MpnError, match="CaffeNet.*trunk layer 2 \\(LRN\\)"):
        mpn.train.check_spec(s)
    # the library's own check, on the records (as lua/model_desc.lua would call it)
    from multipathnet_b200._lib import CTrainSpec, load_library
    lib = load_library()
    d, _keep = Model.build_desc(s, grouped=True)
    ext = Model.layer_ext(s)
    recs = (CLayerExt * len(ext))(*ext)
    msg = C.create_string_buffer(512)
    assert lib.mpn_train_check_ext(C.byref(d), recs, len(ext), C.byref(CTrainSpec()), None, msg, len(msg)) != 0
    assert "CaffeNet" in msg.value.decode() and "trunk layer 2 (LRN)" in msg.value.decode()
    # without the LRN layers the first grouped convolution is named
    s2 = models.alexnet_fast_rcnn(21, seed=None)
    for i in (2, 5):
        s2.trunk_layers[i].kind = 2                                  # an identity-shaped stand-in (1 x 1 max pool)
    d2, _k2 = Model.build_desc(s2, grouped=True)
    assert lib.mpn_train_check_ext(C.byref(d2), recs, len(ext), C.byref(CTrainSpec()), None, msg, len(msg)) != 0
    assert "trunk layer 3 (5x5 convolution 96 -> 256 in 2 groups)" in msg.value.decode()


# ---- the LRN rule --------------------------------------------------------------------------------------------------------
def _hd():
    lib = C.CDLL(os.path.join(ROOT, "multipathnet_b200", "liblrn_host.so"))
    lib.hd_lrn.argtypes = [C.c_void_p, C.c_int64, C.c_int, C.c_int64, C.c_void_p]
    lib.hd_lrn.restype = None
    return lib


@pytest.mark.parametrize("Cn", [8, 16, 96, 200, 256, 384])
def test_host_build_of_lrn_rule_is_the_numpy_rule_bit_for_bit(Cn):
    rng = np.random.default_rng(Cn)
    x = CR.lrn_inputs(rng, Cn)
    aS = CR.alpha_s(x)
    assert aS[aS > 0].min() < 1e-2 and aS.max() > 1e2            # a * S spans the range the rule is pinned over
    flat = np.ascontiguousarray(x.reshape(-1, Cn))
    y = np.empty_like(flat)
    _hd().hd_lrn(flat.ctypes.data, flat.shape[0], Cn, Cn, y.ctypes.data)
    ref = CR.lrn_rule(flat)
    assert np.array_equal(y.view(np.uint32), ref.view(np.uint32))
    r64 = CR.lrn64(flat)
    nz = r64 != 0
    assert np.all(y[~nz] == 0)
    assert np.max(np.abs(y[nz] - r64[nz]) / np.abs(r64[nz])) < 2.0 ** -19


# ---- .t7: grouped convolutions and the LRN modules -----------------------------------------------------------------------
def _T(name, **f):
    return t7.T7Object(name, f)


def _tiny_graph(lrn_type, seed=0, lrn=(5, 1e-4, 0.75, 1.0), g2=2):
    """a small CaffeNet-shaped graph as models/alexnet.lua builds it: conv / ReLU / ceil max pool / LRN / grouped conv / ...
    / ROIPooling / View / Linear + ReLU x 2, {class, bbox} Linears"""
    rng = np.random.default_rng(seed)
    Wt = lambda *s: (rng.standard_normal(s) * np.sqrt(2.0 / np.prod(s[1:]))).astype(np.float32)
    Bs = lambda n: (rng.standard_normal(n) * 0.05).astype(np.float32)
    def conv(cin, cout, k, s, p, g=1):
        return _T("cudnn.SpatialConvolution", nInputPlane=cin, nOutputPlane=cout, kW=k, kH=k, dW=s, dH=s, padW=p, padH=p, groups=g,
                  weight=Wt(cout, cin // g, k, k) * (8.0 if cin == 3 else 1.0), bias=Bs(cout))
    relu = lambda: _T("cudnn.ReLU", inplace=True)
    pool = lambda: _T("cudnn.SpatialMaxPooling", kW=3, kH=3, dW=2, dH=2, padW=0, padH=0, ceil_mode=True)
    norm = lambda: _T(lrn_type, size=lrn[0], alpha=lrn[1], beta=lrn[2], k=lrn[3])
    feats = _T("nn.Sequential", modules=[conv(3, 32, 5, 2, 0), relu(), pool(), norm(), conv(32, 48, 5, 1, 2, g=g2), relu(), pool(),
                                         norm(), conv(48, 64, 3, 1, 1), relu(), conv(64, 32, 3, 1, 1, g=2), relu()])
    fc = lambda i, o: _T("nn.Linear", weight=Wt(o, i), bias=Bs(o))
    return _T("nn.Sequential", modules=[_T("nn.ParallelTable", modules=[feats, _T("nn.Identity")]),
                                        _T("inn.ROIPooling", W=3, H=3, spatial_scale=1.0 / 8, v2=True),
                                        _T("nn.View", size=[-1], numInputDims=3), fc(32 * 9, 64), relu(), fc(64, 64), relu(),
                                        _T("nn.ConcatTable", modules=[fc(64, 5), fc(64, 20)])])


def _roundtrip(g):
    buf = io.BytesIO()
    t7.save(buf, g)
    buf.seek(0)
    return t7.load(buf)


@pytest.mark.parametrize("lrn_type", ["nn.SpatialCrossMapLRN", "inn.SpatialCrossResponseNormalization", "cudnn.SpatialCrossMapLRN"])
def test_tiny_graph_through_the_t7_writer_and_reader_matches_module_evaluation(oracle_built, lrn_type):
    g = _roundtrip(_tiny_graph(lrn_type, seed=len(lrn_type)))
    spec = t7.model_from_t7(g)
    assert [L.groups for L in spec.trunk_layers if L.kind == MPN_LAYER_CONV] == [1, 2, 1, 2]
    assert [L.kind for L in spec.trunk_layers].count(MPN_LAYER_LRN) == 2
    assert [r.groups for r in Model.layer_ext(spec)] == [2, 2]
    back = t7.model_from_t7(_roundtrip(t7.model_to_t7(spec)))
    key = lambda L: (L.kind, L.groups, L.cin, L.cout, L.kh, L.stride, L.pad, L.relu, L.ceil_mode)
    assert [key(L) for L in back.trunk_layers] == [key(L) for L in spec.trunk_layers]
    assert all(np.array_equal(a, b) for a, b in zip(spec.weights, back.weights))
    from oracle import graphs as G
    from multipathnet_b200 import workloads as wl
    img = wl.transform(wl.raw_image(61, 77, 3), "ross") / np.float32(16)
    boxes = wl.random_boxes(17, 61, 77, 3)
    from oracle import ref as O
    rois = O.project_rois(boxes, np.float32(1.0))
    trunk = G.trunk_forward(back, img)
    a = CR.alpha_s(trunk[back.trunk_layers[3].in_slot][0].numpy().transpose(1, 2, 0))
    assert np.median(a) > 1e-2                                  # the LRN does something on this input
    cls, bbox = G.heads_forward(back, trunk, rois)
    ncls, nbbox = CR.evaluate_nn(g, [torch.from_numpy(img)[None], torch.from_numpy(rois)])
    assert rel(cls, ncls.numpy()) < 1e-5 and rel(bbox, nbbox.numpy()) < 1e-5


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def test_full_caffenet_graph_round_trips():
    s = models.alexnet_fast_rcnn(21, seed=None)
    back = t7.model_from_t7(_roundtrip(t7.model_to_t7(s)))
    key = lambda L: (L.kind, L.groups, L.cin, L.cout, L.kh, L.kw, L.stride, L.pad, L.relu, L.ceil_mode)
    assert [key(L) for L in back.trunk_layers] == [key(L) for L in s.trunk_layers]
    assert [key(L) for L in back.towers[0].layers] == [key(L) for L in s.towers[0].layers]
    assert (back.towers[0].pooled_h, back.towers[0].pooled_w) == (6, 6) and back.towers[0].levels[0][1] == pytest.approx(1 / 16)
    assert [(r.layer, r.groups) for r in Model.layer_ext(back)] == [(3, 2), (7, 2), (8, 2)]


def test_importer_refusals():
    with pytest.raises(NotImplementedError, match="only CaffeNet's LRN"):
        t7.model_from_t7(_tiny_graph("nn.SpatialCrossMapLRN", lrn=(3, 1e-4, 0.75, 1.0)))
    with pytest.raises(NotImplementedError, match="only CaffeNet's LRN"):
        t7.model_from_t7(_tiny_graph("cudnn.SpatialCrossMapLRN", lrn=(5, 1e-4, 0.75, 2.0)))
    with pytest.raises(NotImplementedError, match="multiple of 8"):
        t7.model_from_t7(_tiny_graph("nn.SpatialCrossMapLRN", g2=4))            # 32 -> 48 in 4 groups: 12 per group
    with pytest.raises(NotImplementedError, match="multiple of 8"):
        t7.model_from_t7(_tiny_graph("nn.SpatialCrossMapLRN", g2=3))            # does not divide
    # loadcaffe's nn.Concat of nn.Narrow branches
    br = lambda i: _T("nn.Sequential", modules=[_T("nn.Narrow", dimension=2, index=i, length=16),
                                                 _T("nn.SpatialConvolution", nInputPlane=16, nOutputPlane=16, kW=1, kH=1, dW=1, dH=1, padW=0,
                                                    padH=0, weight=np.zeros((16, 16, 1, 1), np.float32), bias=np.zeros(16, np.float32))])
    g = _tiny_graph("nn.SpatialCrossMapLRN")
    feats = t7._children(t7._children(g)[0])[0]
    feats.fields["modules"].insert(3, _T("nn.Concat", dimension=2, modules=[br(1), br(17)]))
    with pytest.raises(NotImplementedError, match="Narrow"):
        t7.model_from_t7(g)


def test_lua_shim_builds_groups_records_and_maps_the_lrn_modules():
    src = open(os.path.join(ROOT, "lua", "model_desc.lua")).read()
    assert "d.tower, d.layer, d.pad_w, d.out_c_off, d.out_c_total, d.exclude_pad, d.groups" in src
    assert "MPN_LAYER_LRN = 5" in open(os.path.join(ROOT, "include", "mpn_abi.h")).read()
    for s in ("SpatialCrossMapLRN = true", "SpatialCrossResponseNormalization = true", "LRN = 5", "only CaffeNet's LRN", "groups",
              "Narrow"):
        assert s in src, s
    assert "grouped convolution (CaffeNet) is not on the accelerated path" not in src

"""Inception-v3 Fast R-CNN on the host: the builder's graph (sizes, concatenation offsets, FLOP counts), its mpn_layer_ext
records, the "inception" transformer, and the fp64 restatement the GPU tests compare against (tests/_inception_ref.py)."""
import ctypes as C

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import (CImageTransform, CLayer, CLayerExt, Layer, Model, MPN_LAYER_AVGPOOL, MPN_LAYER_AVGPOOL_WIN,
                                    MPN_LAYER_CONV, MPN_LAYER_MAXPOOL, MpnError)
from multipathnet_b200.modules import ImageTransformer
from multipathnet_b200.train import check_spec

import _inception_ref as IR


@pytest.fixture(scope="module")
def skel():
    return models.inception_v3_fast_rcnn(seed=None)


def _shapes(layers, h, w, cin):
    """slot -> (C, H, W) by a walk independent of the library's: torch on the meta device, concatenations summed per slot"""
    slots = {0: torch.empty((1, cin, h, w), device="meta")}
    parts = {}
    for L in layers:
        x = slots[L.in_slot]
        if L.kind == MPN_LAYER_CONV:
            y = torch.nn.functional.conv2d(x, torch.empty((L.cout, L.cin, L.kh, L.kw), device="meta"), stride=L.stride,
                                           padding=(L.pad, L.padw))
        elif L.kind == MPN_LAYER_MAXPOOL:
            y = torch.nn.functional.max_pool2d(x, L.kh, L.stride, L.pad, ceil_mode=bool(L.ceil_mode))
        elif L.kind == MPN_LAYER_AVGPOOL_WIN:
            y = torch.nn.functional.avg_pool2d(x, L.kh, L.stride, L.pad, ceil_mode=bool(L.ceil_mode))
        else:
            y = x.mean(dim=(2, 3), keepdim=True)
        if L.out_c_total:
            parts.setdefault(L.out_slot, []).append((L.out_c_off, y.shape[1], tuple(y.shape[2:])))
            y = torch.empty((1, L.out_c_total) + tuple(y.shape[2:]), device="meta")
        slots[L.out_slot] = y
    return {k: tuple(v.shape[1:]) for k, v in slots.items()}, parts


def _flops(layers, h, w, cin):
    shp, _ = _shapes(layers, h, w, cin)
    return sum(2.0 * L.cin * L.cout * L.kh * L.kw * shp[L.out_slot][1] * shp[L.out_slot][2] for L in layers if L.kind == MPN_LAYER_CONV)


def test_builder_sizes_and_concatenations_at_299(skel):
    shp, parts = _shapes(skel.trunk_layers, 299, 299, 3)
    assert shp[skel.taps["mixed_6e"]] == (768, 17, 17)
    t = skel.towers[0]
    assert (t.pooled_h, t.pooled_w) == (17, 17) and t.levels[0][1] == 17.0 / 299.0
    tshp, tparts = _shapes(t.layers, 17, 17, 768)
    assert tshp[t.out_slot][0] == 2048 and skel.bbox_head.col_len == 2048
    stem = [L for L in skel.trunk_layers[:7]]
    assert [(L.kind, L.kh, L.stride, L.pad) for L in stem] == [(1, 3, 2, 0), (1, 3, 1, 0), (1, 3, 1, 1), (2, 3, 2, 0), (1, 1, 1, 0),
                                                               (1, 3, 1, 0), (2, 3, 2, 0)]
    want = [[0, 64, 128, 224, 256], [0, 64, 128, 224, 288], [0, 64, 128, 224, 288], [0, 384, 480, 768]] + [[0, 192, 384, 576, 768]] * 4
    got = []
    for slot in sorted(parts):
        p = sorted(parts[slot])
        assert len({s for _, _, s in p}) == 1                           # branches share the map size
        got.append([o for o, _, _ in p] + [p[-1][0] + p[-1][1]])
    assert got == want
    sizes = [shp[s][1:] for s in sorted(parts)]
    assert sizes == [(35, 35)] * 3 + [(17, 17)] * 5
    tg = [sorted(tparts[s]) for s in sorted(tparts)]
    assert [[o for o, _, _ in p] + [p[-1][0] + p[-1][1]] for p in tg] == [[0, 320, 512, 1280],
                                                                         [0, 320, 704, 1088, 1472, 1856, 2048],
                                                                         [0, 320, 704, 1088, 1472, 1856, 2048]]
    assert [p[0][2] for p in tg] == [(8, 8)] * 3
    for L in skel.trunk_layers + t.layers:                           # every offset 16-aligned, every Cin / Cout 8-aligned
        assert L.out_c_off % 16 == 0 and L.cin % 8 == 0 and L.cout % 8 == 0 or L.in_slot == 0
    asym = {(L.kh, L.kw, L.pad, L.padw) for L in skel.trunk_layers + t.layers if L.kh != L.kw}
    assert asym == {(1, 7, 0, 3), (7, 1, 3, 0), (1, 3, 0, 1), (3, 1, 1, 0)}


@pytest.mark.parametrize("H,W", [(299, 299), (600, 1000), (413, 331)])
def test_flop_counts_match_the_layer_table(skel, H, W):
    assert models.trunk_flops(skel, H, W) == _flops(skel.trunk_layers, H, W, 3)
    t = skel.towers[0]
    heads = sum(2.0 * h.col_len * h.cout for h in skel.cls_heads + [skel.bbox_head])
    assert models.head_flops_per_roi(skel) == _flops(t.layers, 17, 17, 768) + heads


def test_existing_builders_carry_no_ext_records():
    for spec in (models.vgg16_fast_rcnn(seed=None), models.vgg16_multipathnet(seed=None), models.resnet50_fast_rcnn(seed=None),
                 models.nin_fast_rcnn(seed=None), models.resnet18_fast_rcnn(seed=None, fixed_bn=True)):
        assert Model.layer_ext(spec) == [] and models.is_inference_only(spec) == ""
    assert C.sizeof(CLayer) == 14 * 4 and C.sizeof(CLayerExt) == 6 * 4


def test_inception_ext_records(skel):
    recs = Model.layer_ext(skel)
    t = skel.towers[0]
    odd = [L for L in skel.trunk_layers + t.layers if L.out_c_total or L.exclude_pad or L.padw != L.pad]
    assert len(recs) == len(odd) == len({(r.tower, r.layer) for r in recs}) > 0
    for r in recs:
        L = skel.trunk_layers[r.layer] if r.tower < 0 else t.layers[r.layer]
        assert (r.pad_w, r.out_c_off, r.out_c_total, r.exclude_pad) == (L.padw, L.out_c_off, L.out_c_total, L.exclude_pad)
    d, _ = Model.build_desc(skel)                                     # the description itself is the 14-field layer table
    assert d.n_trunk_layers == len(skel.trunk_layers) and d.trunk_layers[12].kind == MPN_LAYER_CONV
    assert all(L.kind == MPN_LAYER_AVGPOOL for L in t.layers[-1:])
    assert Layer(MPN_LAYER_CONV, 0, 1, kh=1, kw=7, pad=0, pad_w=3).ext(-1, 0).pad_w == 3
    assert Layer(MPN_LAYER_CONV, 0, 1, kh=3, kw=3, pad=1).ext(-1, 0) is None


def test_training_is_refused_by_name(skel):
    with pytest.raises(MpnError, match="Inception-v3.*trunk layer 7"):
        check_spec(skel)


def test_inception_transformer_host_and_device_arithmetic(oracle_built, monkeypatch):
    im = wl.raw_image(13, 17, 5)
    out = ImageTransformer("inception").forward(im)
    assert np.array_equal(out, im * np.float32(2) - np.float32(1))
    t = CImageTransform.of("inception")
    assert list(t.swap) == [1, 2, 3] and t.scale == 2.0 and list(t.mean) == [1, 1, 1] and t.has_std == 0
    # the product's per-pixel getImages code (csrc/image_scale.cuh, built for the host) with the same plain data
    monkeypatch.setitem(oracle_built._TRANSFORMERS, "inception", ((1.0, 1.0, 1.0), None, 2.0, (1, 2, 3)))
    assert np.array_equal(oracle_built.image_transform(im, "inception"), out)
    for h, w in [(13, 17), (20, 31), (7, 9)]:
        assert np.array_equal(oracle_built.hd_get_images(im, "inception", h, w), oracle_built.image_scale(out, h, w))


def test_reference_restatement_against_module_by_module_torch(oracle_built):
    """the fp64 restatement's concatenation slots equal torch.cat of the branches run one by one"""
    spec = IR.tiny_spec()
    img = wl.transform(wl.raw_image(40, 48, 1), "inception")
    slots = IR.trunk_forward(spec, img)
    f = lambda L, x: IR.layer(L, x, spec.weights)
    L = spec.trunk_layers
    x = slots[L[1].out_slot]
    b0 = f(L[2], x); b1 = f(L[4], f(L[3], x)); b2 = f(L[6], f(L[5], x)); b3 = f(L[8], f(L[7], x))
    cat = torch.cat([b0, b1, b2, b3], 1)
    assert torch.equal(slots[L[2].out_slot], cat)
    top = torch.cat([f(L[9], cat), f(L[10], cat)], 1)
    assert torch.equal(slots[spec.taps["top"]], top) and not torch.isnan(top).any()
    pooled = IR.pooled_rows(spec, slots, np.array([[1, 1, 1, 40, 30], [1, 5, 9, 21, 17]], np.float32))
    assert pooled.shape == (2, 96, 5, 5)


# ---- import / export: t7.model_from_t7 / model_to_t7 and the Lua shim ---------------------------------------------------
def _roundtrip(spec):
    import io
    from multipathnet_b200 import t7
    g = t7.model_to_t7(spec)
    buf = io.BytesIO()
    t7.save(buf, g)
    buf.seek(0)
    g2 = t7.load(buf)
    return g2, t7.model_from_t7(g2, name="inceptionv3.t7")


@pytest.mark.parametrize("xp", [1, 0])
def test_tiny_inception_graph_through_the_t7_writer_and_reader(oracle_built, xp):
    """a hand-built inceptionv3.lua graph at narrow widths (one block of each kind, a nested concat, K-tail Cin 40 / 24,
    include- and exclude-pad pools) -> model_to_t7 -> .t7 bytes -> model_from_t7: the oracle's detect equals a
    module-by-module evaluation of the graph"""
    spec = IR.tiny_spec(seed=9 + xp, xp=xp)
    g, back = _roundtrip(spec)
    assert back.transformer == "inception" and len(back.trunk_layers) == len(spec.trunk_layers)
    key = lambda L: (L.kind, L.cin, L.cout, L.kh, L.kw, L.stride, L.pad, L.padw, L.relu, L.ceil_mode,
                     L.out_c_off, L.out_c_total, L.exclude_pad)
    assert [key(L) for L in back.trunk_layers] == [key(L) for L in spec.trunk_layers]
    assert [key(L) for L in back.towers[0].layers] == [key(L) for L in spec.towers[0].layers]
    assert Model.layer_ext(back) and len(Model.layer_ext(back)) == len(Model.layer_ext(spec))
    img = wl.transform(wl.raw_image(44, 52, 3), "inception")
    boxes = wl.random_boxes(17, 44, 52, 3)
    rois = np.concatenate([np.ones((17, 1), np.float32), boxes], 1)
    s_ref, b_ref = IR.detect(back, img, boxes, 1.0)
    cls, bbox = IR.evaluate_nn(g, [torch.from_numpy(img)[None], torch.from_numpy(rois)])
    s_nn = oracle_built.softmax(cls.numpy())
    b_nn = oracle_built.convert_from(bbox.numpy(), boxes)
    assert np.abs(s_ref - s_nn).max() < 1e-5 and np.abs(b_ref - b_nn).max() / np.abs(b_nn).max() < 1e-5


def test_full_inception_graph_round_trips(skel):
    _, back = _roundtrip(skel)
    key = lambda L: (L.kind, L.cin, L.cout, L.kh, L.kw, L.stride, L.pad, L.padw, L.out_c_off, L.out_c_total,
                     L.exclude_pad)
    assert [key(L) for L in back.trunk_layers] == [key(L) for L in skel.trunk_layers]
    assert [key(L) for L in back.towers[0].layers] == [key(L) for L in skel.towers[0].layers]
    assert (back.towers[0].pooled_h, back.towers[0].pooled_w) == (17, 17) and back.towers[0].levels[0][1] == pytest.approx(17 / 299)


def _graph(branches, dim=2, kind="nn.Concat", stride=(1, 1)):
    from multipathnet_b200.t7 import T7Object as T
    conv = lambda cin, cout, kh, kw, ph, pw, s=(1, 1): T("cudnn.SpatialConvolution", dict(
        nInputPlane=cin, nOutputPlane=cout, kH=kh, kW=kw, dH=s[0], dW=s[1], padH=ph, padW=pw,
        weight=np.zeros((cout, cin, kh, kw), np.float32), bias=np.zeros(cout, np.float32)))
    seq = lambda *ms: T("nn.Sequential", dict(modules=list(ms)))
    br = [seq(conv(16, 16, k[0], k[1], k[2], k[3], stride if i == 0 else (1, 1))) for i, k in enumerate(branches)]
    trunk = seq(conv(3, 16, 3, 3, 1, 1), T(kind, dict(dimension=dim, modules=br)))
    lin = lambda o, i: T("nn.Linear", dict(weight=np.zeros((o, i), np.float32), bias=np.zeros(o, np.float32)))
    return T("nn.Sequential", dict(modules=[T("nn.ParallelTable", dict(modules=[trunk, T("nn.Identity", {})])),
                                            T("inn.ROIPooling", dict(W=2, H=2, spatial_scale=1.0)),
                                            T("nn.View", dict(size=[-1], numInputDims=3)),
                                            T("nn.ConcatTable", dict(modules=[lin(3, 128), lin(12, 128)]))]))


def test_importer_refusals_by_message():
    from multipathnet_b200 import t7
    ok = t7.model_from_t7(_graph([(1, 7, 0, 3), (7, 1, 3, 0)]))
    assert [L.out_c_off for L in ok.trunk_layers[1:]] == [0, 16] and ok.trunk_layers[1].padw == 3
    with pytest.raises(NotImplementedError, match="anisotropic stride"):
        t7.model_from_t7(_graph([(3, 3, 1, 1), (1, 1, 0, 0)], stride=(1, 2)))
    with pytest.raises(NotImplementedError, match="along dimension 1"):
        t7.model_from_t7(_graph([(1, 1, 0, 0), (1, 1, 0, 0)], dim=1))
    with pytest.raises(NotImplementedError, match="different map sizes"):
        t7.model_from_t7(_graph([(1, 1, 0, 0), (3, 3, 0, 0)], kind="nn.DepthConcat"))


def test_lua_shim_builds_ext_records_for_mpn_model_create_ext():
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    src = open(os.path.join(root, "lua", "model_desc.lua")).read()
    hdr = open(os.path.join(root, "include", "mpn_abi.h")).read()
    cdef = re.search(r"MPN_CDEF_BEGIN \*/(.*?)/\* MPN_CDEF_END", hdr, re.S).group(1)
    fields = re.search(r"typedef struct mpn_layer_ext \{(.*?)\} mpn_layer_ext;", cdef, re.S).group(1)
    names = re.findall(r"\b(tower|layer|pad_w|out_c_off|out_c_total|exclude_pad)\b", re.sub(r"/\*.*?\*/", "", fields, flags=re.S))
    assert names == ["tower", "layer", "pad_w", "out_c_off", "out_c_total", "exclude_pad"]
    assert "ffi.new('mpn_layer_ext[?]'" in src and "C.mpn_model_create_ext(ctx, desc, ea, #ext, wp, ne, #wts, out)" in src
    assert "d.tower, d.layer, d.pad_w, d.out_c_off, d.out_c_total, d.exclude_pad" in src
    assert "AVGPOOL_WIN = 1, 2, 3, 4, 6" in src and "MPN_LAYER_AVGPOOL_WIN = 6" in hdr
    for mod in ("'Concat'", "'DepthConcat'", "count_include_pad", "anisotropic stride"):
        assert mod in src

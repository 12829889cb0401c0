"""Inception-v3 Fast R-CNN on the device against the fp64 restatement (tests/_inception_ref.py): every layer on its own
device inputs (1 x n / n x 1 kernels, windowed average pools, branches written into concatenation slots), ROI pooling at
17 x 17 on 768 channels, detect + NMS at 600 x 1000 with 1000 ROIs, a long-lived model across shapes, and the refusals."""
import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import MPN_LAYER_AVGPOOL, MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_CONV, MPN_LAYER_MAXPOOL, MpnError
from oracle import ref as O

import _bf16_oracle as B
import _inception_ref as IR
from conftest import rel_err

pytestmark = pytest.mark.gpu

TOL, TOL_BF16, SPLIT = 1e-4, 1e-5, 2.0 ** -17       # the engine tests' bars (test_engine_gpu.py, test_bf16_gpu.py, NIN)


def _rn(a):
    return B.rn_bf16(torch.as_tensor(np.ascontiguousarray(a, np.float32))).double()


def _planes(pl):
    """slot planes (bf16 hi / lo bit patterns) -> (hi + lo, hi) as fp32 N x C x H x W"""
    f = lambda a: np.ascontiguousarray((a.astype(np.uint32) << 16).view(np.float32).transpose(0, 3, 1, 2))
    hi = f(pl["hi"])
    return hi + f(pl["lo"]), hi


def _check_layers(m, spec, layers, get, bar, tag, bf16):
    """each layer's device output (its channel slice) against fp64 of the layer on the device's input planes; bf16: a
    convolution against the fp64 product of the hi plane it reads and the bf16-rounded weights (tests/_layer_ref.py's rule)"""
    worst = {}
    for i, L in enumerate(layers):
        if L.kind == MPN_LAYER_AVGPOOL or L.in_slot == 0 and layers is spec.trunk_layers:
            continue
        val, hi = get(L.in_slot)
        x = torch.as_tensor(val, dtype=torch.float64, device="cuda")
        w = spec.weights
        if bf16 and L.kind == MPN_LAYER_CONV:
            x = torch.as_tensor(hi, dtype=torch.float64, device="cuda")
            w = {L.weight: _rn(spec.weights[L.weight]).numpy(), L.bias: spec.weights[L.bias]}
        ref = IR.layer(L, x, w).cpu().numpy()
        y = get(L.out_slot)[0][:, L.out_c_off:L.out_c_off + ref.shape[1]]
        err = rel_err(y, ref)
        if L.kind == MPN_LAYER_MAXPOOL:
            assert np.array_equal(y, ref.astype(np.float32)), f"{tag} layer {i}: max pool into a slice is not the dense max"
        else:
            assert err < bar[L.kind], f"{tag} layer {i} ({L.kh}x{L.kw}, pad {L.pad}/{L.padw}, {L.cin}->{L.cout}): {err:.2e}"
        worst[L.kind] = max(worst.get(L.kind, 0.0), err)
    return worst


@pytest.mark.parametrize("numerics", ["default", "bf16"])
def test_every_layer_against_fp64(numerics):
    ctx = mpn.Context(0)
    if numerics == "bf16":
        ctx.set_option("bf16", 1)
    spec = models.inception_v3_fast_rcnn(seed=7)
    m = mpn.Model(ctx, spec, max_rois=64, max_h=360, max_w=420)
    img = wl.transform(wl.raw_image(331, 413, 2), "inception")
    boxes = wl.random_boxes(40, 331, 413, 2)
    m.detect(img, boxes, 1.0)
    bf16 = numerics == "bf16"
    bar = {MPN_LAYER_CONV: TOL_BF16 + SPLIT if bf16 else TOL,
           MPN_LAYER_AVGPOOL_WIN: 2 * SPLIT}                   # the pool sums in fp32; its split-plane store keeps 16 bits
    tw = _check_layers(m, spec, spec.trunk_layers, lambda s: _planes(m.slot_planes(-1, s)), bar, "trunk", bf16)
    t = spec.towers[0]
    pw = _check_layers(m, spec, t.layers, lambda s: _planes(m.slot_planes(0, s)), bar, "tower", bf16)
    print(numerics, "trunk", tw, "tower", pw)
    m.close(); ctx.close()


def test_roi_pooling_17x17_on_768_channels_matches_the_module_op():
    ctx = mpn.Context(0)
    spec = models.inception_v3_fast_rcnn(seed=3)
    m = mpn.Model(ctx, spec, max_rois=300, max_h=600, max_w=1000)
    img = wl.transform(wl.raw_image(600, 1000, 4), "inception")
    boxes = wl.random_boxes(300, 600, 1000, 4)
    m.detect(img, boxes, 1.0)
    fm = m.trunk_slot(spec.taps["mixed_6e"])
    assert fm.shape[1:] == (768, 35, 60)
    rois = O.project_rois(boxes, np.float32(1.0))
    ref = ctx.roi_pool(fm, rois, 17, 17, 17.0 / 299.0)              # mpn_roi_pool, the module op
    got = m.pooled(0).reshape(300, 17, 17, 768).transpose(0, 3, 1, 2)
    assert np.array_equal(got, ref)
    m.close(); ctx.close()


def test_tiny_graphs_detect_and_nms_against_fp64():
    ctx = mpn.Context(0)
    for xp in (1, 0):
        spec = IR.tiny_spec(seed=5 + xp, xp=xp)
        m = mpn.Model(ctx, spec, max_rois=128, max_h=128, max_w=160)
        H, W, R = 97, 131, 70
        img = wl.transform(wl.raw_image(H, W, xp), "inception")
        boxes = wl.random_boxes(R, H, W, xp)
        s, b, keeps = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        rs, rb, _ = IR.test_one(spec, img, boxes, 1.0, W, H)
        assert np.abs(s - rs).max() / np.abs(rs).max() < 1e-3 and np.abs(b - rb).max() / np.abs(rb).max() < 1e-3
        for j in range(1, spec.num_classes):
            sb = np.concatenate([b[:, 4 * j:4 * j + 4], s[:, j:j + 1]], 1).astype(np.float32)
            assert np.array_equal(keeps[j - 1], O.nms(sb, 0.3))
        m.close()
    ctx.close()


def test_full_size_detect_nms_600x1000_with_1000_rois():
    ctx = mpn.Context(0)
    spec = models.inception_v3_fast_rcnn(seed=11)
    m = mpn.Model(ctx, spec, max_rois=1000, max_h=600, max_w=1000)
    raw = wl.raw_image(600, 1000, 9)
    img = wl.transform(raw, "inception")
    boxes = wl.random_boxes(1000, 600, 1000, 9)
    s, b, keeps = m.detect_nms(img, boxes, 1.0, 1000, 600, -1.5, 0.3)
    rs, rb, _ = IR.test_one(spec, img, boxes, 1.0, 1000, 600)
    es, eb = np.abs(s - rs).max() / np.abs(rs).max(), np.abs(b - rb).max() / np.abs(rb).max()
    print(f"600x1000 R=1000: scores {es:.2e} boxes {eb:.2e}")
    assert es < 1e-3 and eb < 1e-3
    for j in range(1, spec.num_classes):
        sb = np.concatenate([b[:, 4 * j:4 * j + 4], s[:, j:j + 1]], 1).astype(np.float32)
        assert np.array_equal(keeps[j - 1], O.nms(sb, 0.3))
    # Tester.testOne with iterative localisation, rbox scores and voting runs the same graph
    s2, b2, k2, v2 = m.test_one(img, boxes[:200], 1.0, 1000, 600, num_iter=2, use_rbox_scores=True, bbox_voting=True)
    assert s2.shape == (200, spec.num_classes) and len(k2) == spec.num_classes - 1 and all(np.isfinite(v).all() for v in v2)
    # getImages on the device with the "inception" transformer equals the host transformer + trunk
    sc, h, w = m.trunk_image(raw, "inception", 600, 1000)
    dev_map = m.trunk_slot(spec.taps["mixed_6e"])
    m.trunk(wl.transform(raw, "inception"))
    assert (h, w, sc) == (600, 1000, 1.0) and np.array_equal(dev_map, m.trunk_slot(spec.taps["mixed_6e"]))
    m.close(); ctx.close()


@pytest.mark.parametrize("numerics", ["default", "bf16"])
def test_shape_sequence_matches_fresh_models(numerics):
    ctx = mpn.Context(0)
    if numerics == "bf16":
        ctx.set_option("bf16", 1)
    spec = models.inception_v3_fast_rcnn(seed=5)
    live = mpn.Model(ctx, spec, max_rois=130, max_h=400, max_w=520)
    for H, W, R in [(299, 299, 65), (250, 400, 1), (380, 512, 129), (299, 299, 64), (331, 211, 130)]:
        img = wl.transform(wl.raw_image(H, W, H + R), "inception")
        boxes = wl.random_boxes(R, H, W, W + R)
        a = live.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        fresh = mpn.Model(ctx, spec, max_rois=130, max_h=400, max_w=520)
        f = fresh.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        fresh.close()
        assert np.array_equal(a[0], f[0]) and np.array_equal(a[1], f[1]) and all(np.array_equal(x, y) for x, y in zip(a[2], f[2]))
    live.close(); ctx.close()


def test_fp8_and_training_refuse_by_name_and_the_model_still_detects():
    ctx = mpn.Context(0)
    spec = models.inception_v3_fast_rcnn(seed=2)
    m = mpn.Model(ctx, spec, max_rois=32, max_h=320, max_w=320)
    img = wl.transform(wl.raw_image(299, 299, 1), "inception")
    boxes = wl.random_boxes(16, 299, 299, 1)
    ctx.set_option("fp8", 1)
    with pytest.raises(MpnError, match="fp8.*Inception-v3"):
        m.detect(img, boxes, 1.0)
    ctx.set_option("fp8", 0)
    with pytest.raises(MpnError, match="Inception-v3"):
        mpn.Trainer(m)
    # the library refuses too, before it allocates anything, for callers of the C ABI (lua/model_desc.lua)
    from multipathnet_b200._lib import CTrainConfig, CTrainSpec
    cfg, ts = CTrainConfig(1e-3, 0.9, 0.0, 5e-4, 0.5, 1.0, 1), CTrainSpec()
    assert ctx.lib.mpn_model_train_begin(m.h, cfg, ts) != 0
    msg = ctx.lib.mpn_last_error(ctx.h).decode()
    assert "Inception-v3" in msg and "trunk layer 7" in msg, msg
    s, b = m.detect(img, boxes, 1.0)
    rs, rb = IR.detect(spec, img, boxes, 1.0)
    assert np.abs(s - rs).max() / np.abs(rs).max() < 1e-3
    m.close(); ctx.close()


# ---- the engine and the pools on their own ---------------------------------------------------------------------------
KERNELS = [(1, 7, 1, 0, 3), (7, 1, 1, 3, 0), (1, 3, 1, 0, 1), (3, 1, 1, 1, 0), (3, 3, 2, 0, 0)]   # kh, kw, stride, pad_h, pad_w
MAPS = [(1, 35, 60), (12, 17, 17), (12, 8, 8)]             # a trunk map at 600 x 1000; R per-ROI maps before / after Mixed_7a


@pytest.mark.parametrize("cin", [32, 48, 80, 160, 192, 448, 768])
def test_engine_1xn_nx1_and_strided_valid_into_a_slice(cin):
    """the wgmma engine and its check kernel on Inception's kernels, each writing a channel slice of a NaN-filled row:
    BF16X3 within 1e-4 of fp64, BF16X1 within 1e-5 + 2^-17 of the fp64 product of bf16 operands, the neighbours NaN"""
    ctx = mpn.Context(0)
    rng = np.random.default_rng(cin)
    Cout, off, ld = 96, 16, 128
    worst = {}
    for N, H, W in MAPS:
        x = rng.standard_normal((N, cin, H, W)).astype(np.float32)
        for kh, kw, st, ph, pw in KERNELS:
            w = (rng.standard_normal((Cout, cin, kh, kw)) / np.sqrt(cin * kh * kw)).astype(np.float32)
            b = rng.standard_normal(Cout).astype(np.float32)
            Ho, Wo = (H + 2 * ph - kh) // st + 1, (W + 2 * pw - kw) // st + 1
            y0 = np.full((N, Ho, Wo, ld), np.nan, np.float32)
            xd, wd, bd = (torch.as_tensor(a, dtype=torch.float64, device="cuda") for a in (x, w, b))
            ref = torch.relu(torch.nn.functional.conv2d(xd, wd, bd, stride=st, padding=(ph, pw))).permute(0, 2, 3, 1).cpu().numpy()
            refb = torch.relu(torch.nn.functional.conv2d(_rn(x).cuda(), _rn(w).cuda(), bd, stride=st, padding=(ph, pw)))
            refb = refb.permute(0, 2, 3, 1).cpu().numpy()
            for impl in (0, 1):
                y = ctx.conv_check_slice(x, w, y0, off, b, stride=st, pad_h=ph, pad_w=pw, relu=True, impl=impl)
                assert np.isnan(y[..., :off]).all() and np.isnan(y[..., off + Cout:]).all(), "a slice write touched its neighbours"
                e = rel_err(y[..., off:off + Cout], ref)
                assert e < TOL, (N, H, W, kh, kw, st, impl, e)
                worst[("bf16x3", impl)] = max(worst.get(("bf16x3", impl), 0), e)
            try:
                ctx.set_option("bf16", 1)
                y = ctx.conv_check_slice(x, w, y0, off, b, stride=st, pad_h=ph, pad_w=pw, relu=True, impl=0)
            finally:
                ctx.set_option("bf16", -1)
            eb = rel_err(y[..., off:off + Cout], refb)
            assert np.isnan(y[..., :off]).all() and eb <= TOL_BF16 + SPLIT, (N, H, W, kh, kw, st, eb)
            worst["bf16x1"] = max(worst.get("bf16x1", 0), eb)
    print(cin, worst)
    ctx.close()


@pytest.mark.parametrize("H,W", [(17, 17), (8, 8), (35, 60), (9, 14)])
def test_pools_into_a_slice(H, W):
    """avgpool_win_kernel, include- and exclude-pad, floor and ceil mode, against fp64 of its split-plane input within the
    store's 2^-16; the max pool written into a slice equals the dense max pool bit for bit; NaN neighbours untouched"""
    ctx = mpn.Context(0)
    rng = np.random.default_rng(H * 100 + W)
    N, C, off, ld = 3, 40, 24, 72
    x = rng.standard_normal((N, H, W, C)).astype(np.float32) * 4
    # the input as the planes hold it (an identity max pool round-trips through split hi / lo)
    xr = ctx.pool_check(x, MPN_LAYER_MAXPOOL, 1, 1, 0, np.zeros((N, H, W, C), np.float32))
    xt = torch.as_tensor(xr, dtype=torch.float64).permute(0, 3, 1, 2)
    worst = 0.0
    for k, st, p, ceil in [(3, 1, 1, False), (3, 2, 1, True), (3, 2, 0, False), (2, 2, 0, True), (5, 3, 2, True)]:
        for xp in (0, 1):
            ref = torch.nn.functional.avg_pool2d(xt, k, st, p, ceil_mode=ceil, count_include_pad=not xp).permute(0, 2, 3, 1).numpy()
            y0 = np.full((N,) + ref.shape[1:3] + (ld,), np.nan, np.float32)
            y = ctx.pool_check(x, MPN_LAYER_AVGPOOL_WIN, k, st, p, y0, off, ceil_mode=ceil, exclude_pad=xp)
            assert np.isnan(y[..., :off]).all() and np.isnan(y[..., off + C:]).all()
            e = rel_err(y[..., off:off + C], ref)
            assert e < 2 * SPLIT, (k, st, p, ceil, xp, e)
            worst = max(worst, e)
        if p < k:
            dense = ctx.pool_check(x, MPN_LAYER_MAXPOOL, k, st, p, np.zeros((N,) + ref.shape[1:3] + (C,), np.float32), 0, ceil_mode=ceil)
            y = ctx.pool_check(x, MPN_LAYER_MAXPOOL, k, st, p, np.full((N,) + ref.shape[1:3] + (ld,), np.nan, np.float32), off, ceil_mode=ceil)
            assert np.array_equal(y[..., off:off + C].view(np.uint32), dense.view(np.uint32))
            assert np.isnan(y[..., :off]).all() and np.isnan(y[..., off + C:]).all()
            mref = torch.nn.functional.max_pool2d(xt, k, st, p, ceil_mode=ceil).permute(0, 2, 3, 1).numpy()
            assert np.array_equal(dense, mref.astype(np.float32))
    print(H, W, worst)
    ctx.close()


def test_image_detect_on_device_equals_the_host_path():
    from multipathnet_b200.image_detect import ImageDetect
    from multipathnet_b200.modules import ImageTransformer
    ctx = mpn.Context(0)
    spec = models.inception_v3_fast_rcnn(seed=4)
    m = mpn.Model(ctx, spec, max_rois=64, max_h=600, max_w=1000)
    raw = wl.raw_image(375, 500, 6)
    boxes = wl.random_boxes(50, 375, 500, 6)
    host = ImageDetect(m, ImageTransformer("inception")).detect(raw, boxes)
    dev = ImageDetect(m, ImageTransformer("inception"), on_device=True).detect(raw, boxes)
    assert np.array_equal(host[0], dev[0]) and np.array_equal(host[1], dev[1])
    img, s = ImageDetect(m, ImageTransformer("inception")).getImages(raw)
    rs, rb = IR.detect(spec, img, boxes, s)
    assert rel_err(host[0], rs) < 1e-3 and rel_err(host[1], rb) < 1e-3
    m.close(); ctx.close()


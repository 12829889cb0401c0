"""CaffeNet Fast R-CNN on the device: grouped convolutions on the wgmma engine (one problem per group, on channel views),
the cross-map LRN kernel bit for bit against the restatement of csrc/lrn_rule.cuh, every layer of the model against fp64
on its own device inputs, detect + NMS at 600 x 1000 against the CPU oracle and nms.c, the entry points, a long-lived model
across shapes, and the refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import MPN_LAYER_CONV, MPN_LAYER_LRN, MPN_LAYER_MAXPOOL, MpnError
from oracle import graphs as G

import _bf16_oracle as B
import _caffenet_ref as CR
from conftest import rel_err
from test_model_gpu import assert_nms_every_class

pytestmark = pytest.mark.gpu

TOL, TOL_BF16, SPLIT = 1e-4, 1e-5, 2.0 ** -17       # the engine tests' bars (NIN, Inception)
GAIN = 1.0          # conv1's gain for the LRN tests: a * S of order 1 at norm1 / norm2 (asserted below)


def _rn(a):
    return B.rn_bf16(torch.as_tensor(np.ascontiguousarray(a, np.float32))).double()


def _planes(pl):
    """slot planes (bf16 hi / lo bit patterns) -> (hi + lo, hi) as fp32 N x H x W x C"""
    f = lambda a: np.ascontiguousarray((a.astype(np.uint32) << 16).view(np.float32))
    hi = f(pl["hi"])
    return hi + f(pl["lo"]), hi


# ---- the engine on grouped convolutions ----------------------------------------------------------------------------------
CAFFENET = [(96, 256, 2, 5, 1, 2, 1, 37, 62), (384, 384, 2, 3, 1, 1, 1, 37, 62), (384, 256, 2, 3, 1, 1, 1, 37, 62)]
SMALL = [(cg * G, co * G, G, k, st, k // 2, N, 13, 17)
         for cg, co, G, k, st, N in [(8, 16, 2, 3, 1, 1), (24, 32, 4, 5, 2, 3), (48, 64, 2, 5, 1, 3), (64, 64, 4, 1, 1, 1),
                                     (136, 72, 2, 3, 2, 1), (48, 48, 4, 3, 1, 1), (24, 24, 2, 1, 2, 3)]]


@pytest.mark.parametrize("cin,cout,groups,k,stride,pad,N,H,W", CAFFENET + SMALL)
def test_grouped_convolution_against_fp64(cin, cout, groups, k, stride, pad, N, H, W):
    """BF16X3 within 1e-4 of fp64, BF16X1 within 1e-5 + 2^-17 of the fp64 product of bf16 operands; the input is wider
    than Cin with NaN beyond it, the output row wider than Cout with NaN beyond it: no NaN is read or overwritten; the same
    weights with the groups swapped are outside the bar"""
    ctx = mpn.Context(0)
    rng = np.random.default_rng(cin * 7 + cout + k)
    x_ld, y_ld = cin + 16, cout + 8
    x = np.full((N, H, W, x_ld), np.nan, np.float32)
    x[..., :cin] = rng.standard_normal((N, H, W, cin))
    w = (rng.standard_normal((cout, cin // groups, k, k)) / np.sqrt(cin // groups * k * k)).astype(np.float32)
    b = rng.standard_normal(cout).astype(np.float32)
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    y0 = np.full((N, Ho, Wo, y_ld), np.nan, np.float32)
    xn = np.ascontiguousarray(x[..., :cin].transpose(0, 3, 1, 2))
    ref = CR.grouped_conv64(xn, w, b, groups, stride, pad).transpose(0, 2, 3, 1)
    refb = torch.relu(torch.nn.functional.conv2d(_rn(xn), _rn(w), torch.as_tensor(b, dtype=torch.float64), stride=stride,
                                                 padding=pad, groups=groups)).permute(0, 2, 3, 1).numpy()
    for impl in (0, 1):
        y = ctx.conv_check_grouped(x, cin, w, groups, y0, b, stride=stride, pad=pad, relu=True, impl=impl)
        assert np.isnan(y[..., cout:]).all() and not np.isnan(y[..., :cout]).any()
        e = rel_err(y[..., :cout], ref)
        assert e < TOL, (impl, e)
    # negative control: the group order swapped
    half = cout // groups
    wsw = np.concatenate([w[(g + 1) % groups * half:((g + 1) % groups + 1) * half] for g in range(groups)])
    ysw = ctx.conv_check_grouped(x, cin, wsw, groups, y0, b, stride=stride, pad=pad, relu=True)
    assert rel_err(ysw[..., :cout], ref) > 10 * TOL
    try:
        ctx.set_option("bf16", 1)
        y = ctx.conv_check_grouped(x, cin, w, groups, y0, b, stride=stride, pad=pad, relu=True, impl=0)
    finally:
        ctx.set_option("bf16", -1)
    eb = rel_err(y[..., :cout], refb)
    assert np.isnan(y[..., cout:]).all() and eb <= TOL_BF16 + SPLIT, eb
    print((cin, cout, groups, k, stride, N), e, eb)
    ctx.close()


# ---- the LRN kernel ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Cn", [8, 16, 96, 200, 256, 384])
def test_lrn_kernel_bit_for_bit_and_against_fp64(Cn):
    ctx = mpn.Context(0)
    rng = np.random.default_rng(Cn)
    x0 = CR.lrn_inputs(rng, Cn)
    ld = Cn + 24
    x = np.full(x0.shape[:3] + (ld,), np.nan, np.float32)
    x[..., :Cn] = x0
    y = ctx.lrn_check(x, Cn)
    xin = CR.split_planes(x0)                                    # the kernel reads hi + lo of the split input
    exp = CR.split_planes(CR.lrn_rule(xin))
    assert np.array_equal(y.view(np.uint32), exp.view(np.uint32))
    r64 = CR.lrn64(xin)
    nz = r64 != 0
    assert np.all(y[~nz] == 0) and np.max(np.abs(y[nz] - r64[nz]) / np.abs(r64[nz])) < 2.0 ** -16
    ctx.close()


# ---- every layer of the model against fp64 on its own device inputs -------------------------------------------------------
@pytest.mark.parametrize("numerics", ["default", "bf16"])
def test_every_layer_against_fp64(numerics):
    ctx = mpn.Context(0)
    bf16 = numerics == "bf16"
    if bf16:
        ctx.set_option("bf16", 1)
    spec = models.alexnet_fast_rcnn(21, seed=5, first_gain=GAIN)
    m = mpn.Model(ctx, spec, max_rois=64, max_h=320, max_w=420)
    H, W = 300, 400
    img = wl.transform(wl.raw_image(H, W, 1), spec.transformer)
    boxes = wl.random_boxes(40, H, W, 1)
    m.detect(img, boxes, 1.0)
    # the LRN is not the identity on this image: a * S from the oracle's trunk
    slots = G.trunk_forward(spec, img)
    for i in (2, 5):
        a = CR.alpha_s(slots[spec.trunk_layers[i].in_slot][0].numpy().transpose(1, 2, 0))
        assert 0.1 < np.median(a) < 10, (i, np.median(a))
    get = lambda s: _planes(m.slot_planes(-1, s))
    worst = {}
    for i, L in enumerate(spec.trunk_layers):
        if L.in_slot == 0:
            continue                                             # conv1: the first-layer kernel (test_layers_gpu.py)
        val, hi = get(L.in_slot)
        y = get(L.out_slot)[0]
        if L.kind == MPN_LAYER_LRN:
            exp = CR.split_planes(CR.lrn_rule(val))
            assert np.array_equal(y.view(np.uint32), exp.view(np.uint32)), f"layer {i}: LRN is not the rule"
            assert rel_err(val, CR.lrn64(val)) > 1e-2               # negative control: the layer left out
            continue
        if L.kind == MPN_LAYER_MAXPOOL:
            ref = torch.nn.functional.max_pool2d(torch.as_tensor(val).permute(0, 3, 1, 2), L.kh, L.stride, L.pad, ceil_mode=True)
            assert np.array_equal(y, ref.permute(0, 2, 3, 1).numpy()), f"layer {i}"
            continue
        x = torch.as_tensor(hi if bf16 else val, dtype=torch.float64).permute(0, 3, 1, 2)
        w = spec.weights[L.weight].reshape(L.cout, L.cin // L.groups, L.kh, L.kw)
        wd = _rn(w) if bf16 else torch.as_tensor(w, dtype=torch.float64)
        ref = torch.relu(torch.nn.functional.conv2d(x, wd, torch.as_tensor(spec.weights[L.bias], dtype=torch.float64),
                                                    stride=L.stride, padding=L.pad, groups=L.groups)).permute(0, 2, 3, 1).numpy()
        e = rel_err(y, ref)
        assert e < (TOL_BF16 + SPLIT if bf16 else TOL), f"{numerics} layer {i} ({L.kh}x{L.kw}, {L.groups} groups): {e:.2e}"
        worst[i] = e
    print(numerics, worst)
    m.close(); ctx.close()


# ---- detect + NMS and the entry points -----------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1000, 2000])
def test_detect_nms_600x1000_against_the_oracle_and_nms_c(R):
    ctx = mpn.Context(0)
    spec = models.alexnet_fast_rcnn(21, seed=11)      # the default gain: O(1) activations, well-conditioned end-to-end parity
    m = mpn.Model(ctx, spec, max_rois=R, max_h=600, max_w=1000)
    img = wl.transform(wl.raw_image(600, 1000, 9), spec.transformer)
    boxes = wl.random_boxes(R, 600, 1000, 9)
    img_d, boxes_d = torch.as_tensor(img).cuda(), torch.as_tensor(boxes).cuda()
    s_d = torch.empty((R, 21), device="cuda"); b_d = torch.empty((R, 84), device="cuda")
    k_d = torch.empty((20, R), dtype=torch.int32, device="cuda"); c_d = torch.empty(20, dtype=torch.int32, device="cuda")
    m.detect_nms_dev(img_d, 600, 1000, boxes_d, R, 1.0, 1000, 600, -1.5, 0.3, s_d, b_d, k_d, c_d)
    torch.cuda.synchronize()
    s, b = s_d.cpu().numpy(), b_d.cpu().numpy()
    counts, kk = c_d.cpu().numpy(), k_d.cpu().numpy()
    keeps = [kk[j, :counts[j]] for j in range(20)]
    rs, rb, _ = G.test_one(spec, img, boxes, 1.0, 1000, 600)
    es, eb = rel_err(s, rs), rel_err(b, rb)
    print(f"600x1000 R={R}: scores {es:.2e} boxes {eb:.2e}")
    assert es < 1e-3 and eb < 1e-3
    assert_nms_every_class(s, b, keeps)
    tf, _ = m.last_flops()
    assert abs(tf - models.trunk_flops(spec, 600, 1000)) < 1e-6 * tf
    m.close(); ctx.close()


def test_entry_points_tester_image_detect_and_batch():
    ctx = mpn.Context(0)
    spec = models.alexnet_fast_rcnn(21, seed=4)
    m = mpn.Model(ctx, spec, max_rois=300, max_h=1000, max_w=1000)
    tf = mpn.modules.ImageTransformer(spec.transformer)
    raw = wl.raw_image(375, 500, 6)
    boxes = wl.random_boxes(120, 375, 500, 6)
    t = mpn.Tester(m, tf)
    img_boxes = t.testOne(raw, boxes)
    oracle = mpn.Tester(m, tf, backend=_OracleBackend(spec), device_tail=False).testOne(raw, boxes)
    assert len(img_boxes) == 20
    for a, o in zip(img_boxes, oracle):
        assert a.shape[1] == 5 and abs(a.shape[0] - o.shape[0]) <= max(2, o.shape[0] // 50)
    host = mpn.ImageDetect(m, tf).detect(raw, boxes)
    dev = mpn.ImageDetect(m, tf, on_device=True).detect(raw, boxes)
    assert np.array_equal(host[0], dev[0]) and np.array_equal(host[1], dev[1])
    img, sc = mpn.ImageDetect(m, tf).getImages(raw)
    rs, rb = G.detect(spec, img, boxes, sc)
    assert rel_err(host[0], rs) < 1e-3 and rel_err(host[1], rb) < 1e-3
    # detect_nms_batch over 4 images of different sizes equals per-image calls bit for bit
    ims = [wl.raw_image(h, w, h) for h, w in [(375, 500), (480, 360), (333, 640), (500, 500)]]
    bl = [wl.random_boxes(r, im.shape[1], im.shape[2], r) for r, im in zip((60, 1, 150, 89), ims)]
    batch = m.detect_nms_batch(ims, bl, spec.transformer)
    for im, bx, got in zip(ims, bl, batch):
        one = m.detect_nms_batch([im], [bx], spec.transformer)[0]
        assert np.array_equal(got[0], one[0]) and np.array_equal(got[1], one[1]) and all(np.array_equal(x, y) for x, y in zip(got[2], one[2]))
    m.close(); ctx.close()


class _OracleBackend:
    """the CPU oracle behind Tester (oracle/graphs.py), as tests/test_tester_cpu.py injects it"""
    def __init__(self, spec):
        self.spec = spec

    def detect_nms(self, img, boxes, im_scale, W0, H0, thresh, nms_thresh):
        return G.test_one(self.spec, img, boxes, im_scale, W0, H0, thresh, nms_thresh)

    def detect(self, img, boxes, im_scale, recompute_features):
        return G.detect(self.spec, img, boxes, im_scale)


@pytest.mark.parametrize("numerics", ["default", "bf16"])
def test_shape_sequence_matches_fresh_models(numerics):
    ctx = mpn.Context(0)
    if numerics == "bf16":
        ctx.set_option("bf16", 1)
    spec = models.alexnet_fast_rcnn(21, seed=5, first_gain=GAIN)
    live = mpn.Model(ctx, spec, max_rois=300, max_h=600, max_w=1000)
    for H, W, R, how in [(600, 1000, 300, "nms"), (224, 224, 1, "detect"), (375, 500, 129, "nms"), (600, 1000, 64, "test_one"),
                         (331, 211, 300, "nms")]:
        img = wl.transform(wl.raw_image(H, W, H + R), spec.transformer)
        boxes = wl.random_boxes(R, H, W, W + R)
        fresh = mpn.Model(ctx, spec, max_rois=300, max_h=600, max_w=1000)
        for mm in (live, fresh):
            if how == "detect":
                out = mm.detect(img, boxes, 1.0)
            elif how == "test_one":
                out = mm.test_one(img, boxes, 1.0, W, H, num_iter=2, use_rbox_scores=True)[:2]
            else:
                out = mm.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
            if mm is live:
                a = out
        fresh.close()
        f = out
        assert np.array_equal(a[0], f[0]) and np.array_equal(a[1], f[1])
        if how == "nms":
            assert all(np.array_equal(x, y) for x, y in zip(a[2], f[2]))
    live.close(); ctx.close()


def test_fp8_and_training_refuse_by_name_and_the_model_still_detects():
    ctx = mpn.Context(0)
    spec = models.alexnet_fast_rcnn(21, seed=2)
    m = mpn.Model(ctx, spec, max_rois=32, max_h=320, max_w=320)
    img = wl.transform(wl.raw_image(224, 224, 1), spec.transformer)
    boxes = wl.random_boxes(16, 224, 224, 1)
    ctx.set_option("fp8", 1)
    try:
        with pytest.raises(MpnError, match="fp8.*CaffeNet"):
            m.detect(img, boxes, 1.0)
    finally:
        ctx.set_option("fp8", 0)
    with pytest.raises(MpnError, match="CaffeNet"):
        mpn.Trainer(m)
    from multipathnet_b200._lib import CTrainConfig, CTrainSpec
    cfg, ts = CTrainConfig(1e-3, 0.9, 0.0, 5e-4, 0.5, 1.0, 1), CTrainSpec()
    assert ctx.lib.mpn_model_train_begin(m.h, cfg, ts) != 0
    msg = ctx.lib.mpn_last_error(ctx.h).decode()
    assert "CaffeNet" in msg and "trunk layer 2 (LRN)" in msg, msg
    s, b = m.detect(img, boxes, 1.0)
    rs, rb = G.detect(spec, img, boxes, 1.0)
    assert rel_err(s, rs) < 1e-3 and rel_err(b, rb) < 1e-3
    m.close(); ctx.close()

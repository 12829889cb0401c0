"""GPU: the training step with the VGG-16 Fast R-CNN trunk training from conv3_1 (Trainer(train_trunk=True)) against
fp64 torch autograd from each image's stored pool2 output, fed the device's ReLU sides, max-pool and ROI argmaxes,
dropout masks and per-ROI gates; momentum; determinism; the frozen forward unchanged; inference after a step; refusals."""
import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from conftest import rel_err, record_parity
from _train_trunk_ref import pool_argmax, roi_argmax, roi_backward, trunk_step_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda" if torch.cuda.is_available() else "cpu"


def _spec(seed=21):
    return models.vgg16_fast_rcnn(21, seed=seed, width_div=4, fc_dim=256)


def _batch(spec, sizes=((128, 176), (160, 208)), per_image=(40, 56), seed=0):
    rng = np.random.default_rng(seed)
    ims = [wl.transform(wl.raw_image(h, w, seed + i), spec.transformer) for i, (h, w) in enumerate(sizes)]
    rois = [wl.random_boxes(n, h, w, seed + i).astype(np.float32) for i, ((h, w), n) in enumerate(zip(sizes, per_image))]
    R, C = sum(per_image), spec.num_classes
    labels = rng.integers(1, C + 1, R).astype(np.int32)
    labels[:5] = 1
    tg = np.zeros((R, 4 * C), np.float32)
    for r in range(R):
        if labels[r] > 1:
            tg[r, 4 * labels[r] - 4:4 * labels[r]] = rng.standard_normal(4) * 0.8
    return ims, rois, labels, tg


def _trunk_params(spec):
    out = []
    for L in spec.trunk_layers[spec.trunk_train_from:]:
        if L.kind == mpn._lib.MPN_LAYER_CONV:
            out += [L.weight, L.bias]
    return out


def _oracle(tr, spec, weights, rois, labels, tg, p):
    k0 = spec.trunk_train_from
    slots = {spec.trunk_layers[k0].in_slot} | {L.out_slot for L in spec.trunk_layers[k0:]}
    stored = [{s: tr.trunk_slot(i, s) for s in slots} for i in range(len(rois))]
    gates = {}
    T = spec.towers[0]
    for li, L in enumerate(T.layers):
        if L.kind == mpn._lib.MPN_LAYER_CONV and L.relu:
            gates[(0, li)] = tr.relu_gate(0, li)
    return trunk_step_oracle(spec, k0, stored, rois, labels, tg, weights, gates, p, dev=DEV)


def test_trunk_step_losses_and_gradients_vs_fp64(ctx):
    spec = _spec()
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m, seed=7, train_trunk=True)
    assert set(_trunk_params(spec)) <= set(tr.trained) and len(_trunk_params(spec)) == 18
    ims, rois, labels, tg = _batch(spec)
    L = tr.step(ims, rois, labels, tg)
    (rl, rce, rsl), grads = _oracle(tr, spec, spec.weights, rois, labels, tg, 0.5)
    el = [abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl))]
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    assert set(grads) == set(tr.trained)
    record_parity("train_trunk_step", loss=el[0], cls=el[1], bbox=el[2], grad_max=max(eg.values()),
                  trunk_grad_max=max(eg[i] for i in _trunk_params(spec)))
    assert max(el) < 1e-4, (L, (rl, rce, rsl))
    assert max(eg.values()) < 1e-3, eg
    tr.close(); m.close()


def test_trunk_three_steps_with_momentum_and_decay_vs_fp64(ctx):
    spec = _spec(seed=5)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    lr, mom, wd = 1e-2, 0.9, 5e-4
    tr = mpn.Trainer(m, lr=lr, momentum=mom, weight_decay=wd, seed=3, train_trunk=True)
    ims, rois, labels, tg = _batch(spec, seed=4)
    w = {i: np.array(spec.weights[i], np.float64) for i in tr.trained}
    buf = {}
    biases = {L.bias for L in spec.towers[0].layers} | {spec.cls_heads[0].bias, spec.bbox_head.bias} | \
             {L.bias for L in spec.trunk_layers}
    for k in range(3):
        tr.step(ims, rois, labels, tg)
        cur = [w[i] if i in w else spec.weights[i] for i in range(len(spec.weights))]
        _, grads = _oracle(tr, spec, cur, rois, labels, tg, 0.5)
        for i, g in grads.items():
            g = g + (0.0 if i in biases else wd) * w[i]
            buf[i] = g if k == 0 else mom * buf[i] + g
            w[i] = w[i] - lr * buf[i]
        if k == 0:
            tr.decay(0.5); lr *= 0.5
            for i in buf:
                buf[i] = buf[i] * 0.5
    got = tr.weights()
    errs = {i: rel_err(got[i] - spec.weights[i], w[i] - spec.weights[i]) for i in w}
    record_parity("train_trunk_three_steps", delta_max=max(errs.values()))
    assert max(errs.values()) < 1e-3, errs
    tr.close(); m.close()


def test_trunk_two_trainers_same_bits(ctx):
    spec = _spec(seed=13)
    ims, rois, labels, tg = _batch(spec, seed=6)
    outs = []
    for _ in range(2):
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        tr = mpn.Trainer(m, seed=99, train_trunk=True)
        ls = [tr.step(ims, rois, labels, tg) for _ in range(2)]
        outs.append((ls, [tr.gradient(i) for i in tr.trained], tr.weights()))
        tr.close(); m.close()
    assert outs[0][0] == outs[1][0]
    for k in (1, 2):
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(outs[0][k], outs[1][k]))


def test_first_step_frozen_and_trained_trunk_agree(ctx):
    """the forward is the same until the update: losses, logits and per-ROI gradients bit-equal; a frozen trunk keeps
    its weights"""
    spec = _spec(seed=31)
    ims, rois, labels, tg = _batch(spec, seed=3)
    res = []
    for trunk in (False, True):
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        tr = mpn.Trainer(m, seed=4, train_trunk=trunk)
        L = tr.step(ims, rois, labels, tg)
        per_roi = [i for i in tr.trained if i not in _trunk_params(spec)]
        res.append((L, tr.outputs(), {i: tr.gradient(i) for i in per_roi}, tr.weights()))
        tr.close(); m.close()
    (l0, o0, g0, w0), (l1, o1, g1, w1) = res
    assert l0 == l1
    assert all(np.array_equal(a, b) for a, b in zip(o0, o1))
    assert g0.keys() == g1.keys() and all(np.array_equal(g0[i], g1[i]) for i in g0)
    for i in _trunk_params(spec):
        assert np.array_equal(w0[i], spec.weights[i])
    assert any(not np.array_equal(w1[i], spec.weights[i]) for i in _trunk_params(spec))


@pytest.mark.parametrize("w16", [0, 1])
def test_trunk_inference_after_a_step_equals_a_model_built_from_the_weights(ctx, w16):
    spec = _spec(seed=17)
    ims, rois, labels, tg = _batch(spec, seed=8)
    img, H, W = ims[1], ims[1].shape[1], ims[1].shape[2]
    boxes = wl.random_boxes(64, H, W, 11)
    ctx.set_option("fc_w16", w16)
    try:
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        tr = mpn.Trainer(m, seed=1, train_trunk=True)
        tr.step(ims, rois, labels, tg)
        got = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        spec2 = models.ModelSpec(**{**spec.__dict__, "weights": tr.weights()})
        fresh = mpn.Model(ctx, spec2, max_rois=128, max_h=192, max_w=256)
        want = fresh.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        tr.step(ims, rois, labels, tg)                               # and training continues after an inference call
        fresh.close()
    finally:
        ctx.set_option("fc_w16", -1)
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
    assert all(np.array_equal(a, b) for a, b in zip(got[2], want[2]))
    tr.close(); m.close()


def test_trunk_refusals(ctx):
    with pytest.raises(mpn.MpnError, match="trunk_train_from is 0"):
        mpn.Trainer(mpn.Model(ctx, models.vgg16_multipathnet(21, seed=1, width_div=4, fc_dim=256), max_rois=64, max_h=192, max_w=256),
                    train_trunk=True)
    spec = _spec(seed=2)
    spec.trunk_train_from = 6
    m = mpn.Model(ctx, models.vgg16_multipathnet(21, seed=1, width_div=4, fc_dim=256), max_rois=64, max_h=192, max_w=256)
    m.spec.trunk_train_from = 6
    with pytest.raises(mpn.MpnError, match="exactly one tower"):
        mpn.Trainer(m, train_trunk=True)
    m.close()
    m = mpn.Model(ctx, spec, max_rois=64, max_h=192, max_w=256)
    m.trunk(_batch(spec)[0][0])                                       # a trunk call released the trunk's fp32 weights
    with pytest.raises(mpn.MpnError, match="first trunk call"):
        mpn.Trainer(m, train_trunk=True)
    m.close()
    for opt in ("bf16", "fp8"):
        ctx.set_option(opt, 1)
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        try:
            with pytest.raises(mpn.MpnError, match="bf16"):
                mpn.Trainer(m, train_trunk=True)
        finally:
            m.close()
            ctx.set_option(opt, 0)


def test_full_size_fast_rcnn_trunk_step(ctx):
    """vgg16_fast_rcnn(21) at 600 x 1000 and 600 x 800, 128 ROIs each, training from conv3_1: finite losses; head
    gradients against fp64 in full; 16 sampled output rows of conv5_3's and conv3_1's weight gradients; all at 1e-3. The
    oracle's forward starts nine convolutions below the loss (at pool2), where each device layer stores its output as
    split planes: at this size the loss lands within 2e-4 of it, not within the 1e-4 of the small graph."""
    spec = models.vgg16_fast_rcnn(21, seed=1234)
    m = mpn.Model(ctx, spec, max_rois=256, max_h=608, max_w=1008)
    tr = mpn.Trainer(m, seed=555, train_trunk=True)
    ims, rois, labels, tg = _batch(spec, sizes=((600, 1000), (600, 800)), per_image=(128, 128), seed=3)
    L = tr.step(ims, rois, labels, tg)
    assert all(np.isfinite(L))
    (rl, _, _), grads = _oracle(tr, spec, spec.weights, rois, labels, tg, 0.5)
    heads = [spec.cls_heads[0].weight, spec.cls_heads[0].bias, spec.bbox_head.weight, spec.bbox_head.bias]
    eh = max(rel_err(tr.gradient(i), grads[i]) for i in heads)
    rng = np.random.default_rng(0)
    convs = [L_ for L_ in spec.trunk_layers[spec.trunk_train_from:] if L_.kind == mpn._lib.MPN_LAYER_CONV]
    er = {}
    for name, Ly in (("conv3_1", convs[0]), ("conv5_3", convs[-1])):
        rows = rng.choice(Ly.cout, 16, replace=False)
        er[name] = rel_err(tr.gradient(Ly.weight).reshape(Ly.cout, -1)[rows], grads[Ly.weight].reshape(Ly.cout, -1)[rows])
    el = abs(L[0] - rl) / abs(rl)
    record_parity("train_trunk_full_size", loss=el, heads=eh, **er)
    assert el < 1e-3 and eh < 1e-3 and max(er.values()) < 1e-3, (L, rl, eh, er)
    tr.close(); m.close()


# ---- kernel level: the trunk backward's kernels through their test hooks (mpn_debug_*), on host-made split planes

def _bf16_bits(v):
    """round-to-nearest-even bf16 of fp32 v, as raw bits"""
    u = np.ascontiguousarray(v, np.float32).view(np.uint32).astype(np.uint64)
    return ((u + 0x7FFF + ((u >> 16) & 1)) >> 16).astype(np.uint16)


def _planes(v):
    """fp32 -> split planes (hi, lo bits) and the value they hold, hi + lo in fp32 (what the kernels join)"""
    hi = _bf16_bits(v)
    hf = (hi.astype(np.uint32) << 16).view(np.float32)
    lo = _bf16_bits(np.asarray(v, np.float32) - hf)
    lf = (lo.astype(np.uint32) << 16).view(np.float32)
    return hi, lo, (hf + lf).astype(np.float32)


def test_roi_backward_kernel_bit_exact(ctx):
    """roi_argmax_nhwc_kernel + roi_backward_nhwc_kernel against the numpy argmax rule and an in-order scatter: a map of
    few distinct values (ties everywhere, some broken only by the lo plane), many ROIs on the same cells, empty bins"""
    rng = np.random.default_rng(3)
    H, W, C, PW, PH, scale = 9, 13, 64, 7, 7, 0.25
    v = rng.integers(0, 4, (H, W, C)).astype(np.float32)
    v += (rng.random((H, W, C)) < 0.2) * np.float32(2.0 ** -12)       # below hi's precision: lives in the lo plane
    hi, lo, val = _planes(v)
    boxes = [wl.random_boxes(1, 4 * H, 4 * W, s)[0] for s in range(30)]
    boxes += [(5.0, 5.0, 30.0, 22.0)] * 12                               # the same ROI twelve times: its cells named 12 x
    boxes += [(1.0, 1.0, 6.0, 6.0), (45.0, 30.0, 52.0, 36.0), (200.0, 200.0, 260.0, 240.0)]   # tiny, edge, outside: empty bins
    boxes = np.asarray(boxes, np.float32)
    R = len(boxes)
    rois = np.concatenate([np.ones((R, 1), np.float32), boxes], 1)
    g = rng.standard_normal((R, PH * PW, C)).astype(np.float32)
    out = np.empty((H, W, C), np.float32)
    ctx.check(ctx.lib.mpn_debug_roi_backward_nhwc(ctx.h, hi.ctypes.data, lo.ctypes.data, H, W, C, rois.ctypes.data, R, PW, PH, scale, 2,
                                                  g.ctypes.data, out.ctypes.data), "roi backward hook")
    am = roi_argmax(val.transpose(2, 0, 1), boxes, scale, 2, PW, PH)
    assert (am == -1).any() and np.bincount(am[am >= 0].ravel()).max() > 12
    want = roi_backward(g, am, H, W).transpose(1, 2, 0)
    assert np.array_equal(out.view(np.uint32), want.view(np.uint32))


@pytest.mark.parametrize("H,W", [(7, 9), (75, 125), (8, 6)])
def test_pool_backward_kernel_bit_exact(ctx, H, W):
    """pool_gate_split_kernel: odd sizes clip the last window row / column (ceil mode); ties go to the first cell in
    row-major order on hi + lo; cells at or below 0 are gated"""
    rng = np.random.default_rng(H * W)
    C = 32
    y = rng.integers(-1, 3, (H, W, C)).astype(np.float32)
    y += (rng.random((H, W, C)) < 0.2) * np.float32(2.0 ** -12)
    hi, lo, val = _planes(y)
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    gp = rng.standard_normal((Ho, Wo, C)).astype(np.float32)
    out = np.empty((H, W, C), np.float32)
    ctx.check(ctx.lib.mpn_debug_pool_backward(ctx.h, hi.ctypes.data, lo.ctypes.data, H, W, C, gp.ctypes.data, out.ctypes.data), "pool hook")
    idx = pool_argmax(val.transpose(2, 0, 1))                            # C x Ho x Wo
    hh, ww = np.meshgrid(np.arange(H), np.arange(W), indexing="ij")
    named = idx[:, hh // 2, ww // 2] == (hh * W + ww)[None]
    want = np.where(named & (val.transpose(2, 0, 1) > 0), gp.transpose(2, 0, 1)[:, hh // 2, ww // 2], np.float32(0)).transpose(1, 2, 0)
    assert np.array_equal(out.view(np.uint32), want.astype(np.float32).view(np.uint32))


@pytest.mark.parametrize("name,cin,cout,sizes", [
    ("conv3_2", 256, 256, ((150, 250), (150, 200))),
    ("conv4_1", 256, 512, ((75, 125), (75, 100))),
    ("conv5_3", 512, 512, ((38, 63), (38, 50)))])
def test_dgrad_wgrad_3x3_single_layer_vs_fp64(ctx, name, cin, cout, sizes):
    """one trained 3x3 / stride 1 layer's wgrad (ONE GEMM over both images' pixels, split-K plan) and per-image dgrad at
    full-size shapes, through the graph backward's conv backward, against an fp64 product of the same gradient and
    activations: 1e-4 normwise (the per-GEMM bar)"""
    rng = np.random.default_rng(cin + cout)
    P = sum(h * w for h, w in sizes)
    x = np.maximum(rng.standard_normal((P, cin)), 0).astype(np.float32)
    hi, lo, xv = _planes(x)
    g = (rng.standard_normal((P, cout)) * (rng.random((P, cout)) < 0.5)).astype(np.float32)
    w = (rng.standard_normal((cout, cin, 3, 3)) * np.sqrt(2.0 / (9 * cin))).astype(np.float32)
    hw = np.array([s for hw_ in sizes for s in hw_], np.int32)
    dw = np.empty_like(w)
    dx = np.empty((P, cin), np.float32)
    ctx.check(ctx.lib.mpn_debug_conv_backward(ctx.h, len(sizes), hw.ctypes.data_as(mpn._lib._i32p), cin, cout, 3, 1, hi.ctypes.data,
                                              lo.ctypes.data, g.ctypes.data, w.ctypes.data, dw.ctypes.data, dx.ctypes.data), "conv backward hook")
    wt = torch.tensor(w, dtype=torch.float64, device=DEV)
    dw_ref = torch.zeros_like(wt)
    dx_ref = []
    off = 0
    for h, ww in sizes:
        xi = torch.tensor(xv[off:off + h * ww], dtype=torch.float64, device=DEV).reshape(1, h, ww, cin).permute(0, 3, 1, 2)
        gi = torch.tensor(g[off:off + h * ww], dtype=torch.float64, device=DEV).reshape(1, h, ww, cout).permute(0, 3, 1, 2)
        dw_ref += torch.nn.grad.conv2d_weight(xi, wt.shape, gi, padding=1)
        dx_ref.append(torch.nn.grad.conv2d_input(xi.shape, wt, gi, padding=1)[0].permute(1, 2, 0).reshape(-1, cin))
        off += h * ww
    ew = rel_err(dw, dw_ref.cpu().numpy())
    ex = rel_err(dx, torch.cat(dx_ref).cpu().numpy())
    record_parity(f"trunk_backward_{name}", wgrad=ew, dgrad=ex)
    assert ew < 1e-4 and ex < 1e-4, (ew, ex)

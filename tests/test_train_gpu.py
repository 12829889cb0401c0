"""GPU: the per-ROI training step (mpn_model_train_step) against fp64 torch autograd of the per-ROI graph, fed the device's
pooled rows and dropout masks; determinism; the trained model's inference paths; refusals."""
import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from conftest import rel_err, record_parity
from _train_ref import dropout_keep, step_oracle

pytestmark = pytest.mark.gpu
DEV = "cuda" if torch.cuda.is_available() else "cpu"


def _spec(kind, seed=21, **kw):
    if kind == "mpn":
        return models.vgg16_multipathnet(21, seed=seed, width_div=4, fc_dim=256, **kw)
    return models.vgg16_fast_rcnn(21, seed=seed, width_div=4, fc_dim=256, **kw)


def _batch(spec, sizes=((128, 176), (160, 208)), per_image=(40, 56), seed=0):
    rng = np.random.default_rng(seed)
    ims = [wl.transform(wl.raw_image(h, w, seed + i), spec.transformer) for i, (h, w) in enumerate(sizes)]
    rois = [wl.random_boxes(n, h, w, seed + i).astype(np.float32) for i, ((h, w), n) in enumerate(zip(sizes, per_image))]
    R, C = sum(per_image), spec.num_classes
    labels = rng.integers(1, C + 1, R).astype(np.int32)
    labels[:5] = 1
    labels[5] = C
    tg = np.zeros((R, 4 * C), np.float32)
    for r in range(R):
        if labels[r] > 1:
            tg[r, 4 * labels[r] - 4:4 * labels[r]] = rng.standard_normal(4) * 0.8
    tg[7, 0] = 0.3                                                    # an off-mask target: still costs (reference semantics)
    return ims, rois, labels, tg


def _masks(tr, spec, p):
    out = {}
    if p == 0:
        return out
    for t, T in enumerate(spec.towers):
        for li, L in enumerate(T.layers):
            if L.kind == mpn._lib.MPN_LAYER_CONV and L.relu:            # the per-ROI Linears (fc6, fc7)
                out[(t, li)] = tr.dropout_mask(t, li)
    return out


def _gates(tr, spec, masks):
    """the device's backward gates through the ReLUs of the per-ROI Linears; each lies inside its dropout mask"""
    out = {}
    for t, T in enumerate(spec.towers):
        for li, L in enumerate(T.layers):
            if L.kind == mpn._lib.MPN_LAYER_CONV and L.relu:
                out[(t, li)] = tr.relu_gate(t, li)
                if (t, li) in masks:
                    assert not np.any(out[(t, li)] & (1 - masks[(t, li)]))
    return out


def _oracle(m, tr, spec, weights, labels, tg, p):
    """fp64 autograd of the per-ROI graph on the device's pooled rows, dropout masks and ReLU sides"""
    pooled = {t: m.pooled(t) for t in range(len(spec.towers))}
    masks = _masks(tr, spec, p)
    return step_oracle(spec, pooled, masks, p, weights, labels, tg, dev=DEV, gates=_gates(tr, spec, masks))


@pytest.mark.parametrize("kind", ["mpn", "frcnn"])
def test_step_losses_and_gradients_vs_fp64(ctx, kind):
    spec = _spec(kind)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m, seed=7)
    ims, rois, labels, tg = _batch(spec)
    w0 = [np.array(w) for w in spec.weights]
    L = tr.step(ims, rois, labels, tg)
    (rl, rce, rsl), grads, _ = _oracle(m, tr, spec, w0, labels, tg, 0.5)
    el = [abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl))]
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    record_parity(f"train_step_{kind}", loss=el[0], cls=el[1], bbox=el[2], grad_max=max(eg.values()))
    assert max(el) < 1e-4, (L, (rl, rce, rsl))
    assert max(eg.values()) < 1e-3, eg
    # the masks really are the product rule
    mk = tr.dropout_mask(0, len(spec.towers[0].layers) - 1)
    want = dropout_keep(7, 0, 0, len(spec.towers[0].layers) - 1, np.arange(mk.size, dtype=np.uint64), 0.5).reshape(mk.shape)
    assert np.array_equal(mk.astype(bool), want)
    tr.close(); m.close()


def test_three_steps_with_momentum_and_decay_vs_fp64(ctx):
    spec = _spec("mpn", seed=5)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    lr, mom, wd = 1e-2, 0.9, 5e-4
    tr = mpn.Trainer(m, lr=lr, momentum=mom, weight_decay=wd, seed=3)
    ims, rois, labels, tg = _batch(spec, seed=4)
    w = {i: np.array(spec.weights[i], np.float64) for i in tr.trained}
    buf = {}
    biases = {L.bias for T in spec.towers for L in T.layers} | {spec.cls_heads[0].bias, spec.bbox_head.bias}
    for k in range(3):
        tr.step(ims, rois, labels, tg)
        cur = [w[i] if i in w else spec.weights[i] for i in range(len(spec.weights))]
        _, grads, _ = _oracle(m, tr, spec, cur, labels, tg, 0.5)
        for i, g in grads.items():
            g = g + (0.0 if i in biases else wd) * w[i]
            buf[i] = g if k == 0 else mom * buf[i] + g
            w[i] = w[i] - lr * buf[i]
        if k == 0:
            tr.decay(0.5); lr *= 0.5
            for i in buf:
                buf[i] = buf[i] * 0.5
    errs = {i: rel_err(tr.weights()[i] - spec.weights[i], w[i] - spec.weights[i]) for i in w}
    record_parity("train_three_steps", delta_max=max(errs.values()))
    assert max(errs.values()) < 1e-3, errs
    tr.close(); m.close()


@pytest.mark.parametrize("kind", ["mpn", "frcnn"])
def test_p0_forward_equals_heads_per_image(ctx, kind):
    spec = _spec(kind, seed=9)
    spec.bbox_mean, spec.bbox_std = (0.0, 0.0, 0.0, 0.0), (1.0, 1.0, 1.0, 1.0)
    ims, rois, labels, tg = _batch(spec, seed=2)
    ctx.set_option("fc_w16", 0)
    try:
        ref = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        per = []
        for im, r in zip(ims, rois):
            ref.trunk(im)
            per.append(ref.heads(np.concatenate([np.ones((len(r), 1), np.float32), r], 1)))
        ref.close()
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        tr = mpn.Trainer(m, dropout=0.0)
        tr.step(ims, rois, labels, tg)
        cls, bbox = tr.outputs()
        # the second step's forward reads the planes the fused update wrote: the same bits as a model built from the weights
        spec1 = models.ModelSpec(**{**spec.__dict__, "weights": tr.weights()})
        tr.step(ims, rois, labels, tg)
        cls2, bbox2 = tr.outputs()
        ref = mpn.Model(ctx, spec1, max_rois=128, max_h=192, max_w=256)
        per2 = []
        for im, r in zip(ims, rois):
            ref.trunk(im)
            per2.append(ref.heads(np.concatenate([np.ones((len(r), 1), np.float32), r], 1)))
        ref.close()
    finally:
        ctx.set_option("fc_w16", -1)
    for (cc, bb), pp in [((cls, bbox), per), ((cls2, bbox2), per2)]:
        off = 0
        for (c, b), r in zip(pp, rois):
            assert np.array_equal(cc[off:off + len(r)], c) and np.array_equal(bb[off:off + len(r)], b)
            off += len(r)
    ms = np.zeros(4, np.float32)
    ctx.check(ctx.lib.mpn_model_train_phase_ms(m.h, ms.ctypes.data_as(mpn._lib._f32p)), "phase_ms")
    assert np.all(ms > 0)
    tr.close(); m.close()


def test_two_trainers_same_bits(ctx):
    spec = _spec("mpn", seed=13)
    ims, rois, labels, tg = _batch(spec, seed=6)
    outs = []
    for _ in range(2):
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        tr = mpn.Trainer(m, seed=99)
        ls = [tr.step(ims, rois, labels, tg) for _ in range(2)]
        outs.append((ls, tr.weights()))
        tr.close(); m.close()
    assert outs[0][0] == outs[1][0]
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(outs[0][1], outs[1][1]))


@pytest.mark.parametrize("kind", ["mpn", "frcnn"])
@pytest.mark.parametrize("w16", [0, 1])
def test_inference_after_a_step_equals_a_model_built_from_the_weights(ctx, kind, w16):
    spec = _spec(kind, seed=17)
    ims, rois, labels, tg = _batch(spec, seed=8)
    img, H, W = ims[1], ims[1].shape[1], ims[1].shape[2]
    boxes = wl.random_boxes(64, H, W, 11)
    ctx.set_option("fc_w16", w16)
    try:
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        tr = mpn.Trainer(m, seed=1)
        tr.step(ims, rois, labels, tg)
        with pytest.raises(mpn.MpnError, match="cached trunk features"):     # the step's last image is not a cached trunk
            m.detect(None, boxes, 1.0, recompute_features=False)
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
    assert not np.array_equal(tr.weights()[spec.bbox_head.weight], spec.weights[spec.bbox_head.weight])
    tr.close(); m.close()


def test_refusals(ctx):
    spec = _spec("frcnn", seed=3)
    ims, rois, labels, tg = _batch(spec, seed=1)
    with pytest.raises(mpn.MpnError, match="1x1 convolution"):
        mpn.Trainer(mpn.Model(ctx, models.resnet50_fast_rcnn(81, seed=1, integral_k=0), max_rois=64, max_h=128, max_w=128))
    with pytest.raises(mpn.MpnError, match="integral head"):
        mpn.Trainer(mpn.Model(ctx, _spec("mpn", integral_k=2), max_rois=64, max_h=192, max_w=256))
    for opt in ("bf16", "fp8"):
        ctx.set_option(opt, 1)
        try:
            with pytest.raises(mpn.MpnError, match="bf16"):
                mpn.Trainer(mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256))
        finally:
            ctx.set_option(opt, 0)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m)
    bad = labels.copy(); bad[3] = 22
    with pytest.raises(mpn.MpnError, match="labels"):
        tr.step(ims, rois, bad, tg)
    with pytest.raises(mpn.MpnError, match="R = 0"):
        tr.step(ims, [r[:0] for r in rois], labels[:0], tg[:0])
    with pytest.raises(mpn.MpnError, match="max_rois"):
        tr.step(ims, [np.tile(r, (2, 1)) for r in rois], np.tile(labels, 2), np.tile(tg, (2, 1)))      # R = 192 > 128
    with pytest.raises(mpn.MpnError, match="max_h"):
        tr.step([np.zeros((3, 200, 176), np.float32)], rois[:1], labels[:40], tg[:40])     # 200 > max_h = 192
    # the C entry refuses what the Python checks refuse
    import ctypes as C
    lab = np.full(4, 99, np.int32); L3 = np.zeros(3, np.float32)
    hw = np.array([128, 176], np.int32); cnt = np.array([4], np.int32)
    ptrs = (C.c_void_p * 1)(ims[0].ctypes.data)
    rc = ctx.lib.mpn_model_train_step(m.h, 1, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
                                      rois[0][:4].ctypes.data, lab.ctypes.data, tg[:4].ctypes.data, L3.ctypes.data)
    assert rc != 0 and b"label" in ctx.lib.mpn_last_error(ctx.h)
    tr.close(); m.close()


def test_full_size_multipathnet_step(ctx):
    """vgg16_multipathnet(81) at 600 x 800 and 600 x 900, 128 ROIs each: finite losses; head gradients against fp64 in full,
    fc6 / fc7 / conv_mix gradients on 8 sampled output rows per tower"""
    spec = models.vgg16_multipathnet(81, seed=1234)
    m = mpn.Model(ctx, spec, max_rois=256, max_h=608, max_w=912)
    tr = mpn.Trainer(m, seed=555)
    ims, rois, labels, tg = _batch(spec, sizes=((600, 800), (600, 900)), per_image=(128, 128), seed=3)
    L = tr.step(ims, rois, labels, tg)
    assert all(np.isfinite(L))
    (rl, _, _), grads, _ = _oracle(m, tr, spec, spec.weights, labels, tg, 0.5)
    heads = [spec.cls_heads[0].weight, spec.cls_heads[0].bias, spec.bbox_head.weight, spec.bbox_head.bias]
    eh = max(rel_err(tr.gradient(i), grads[i]) for i in heads)
    rng = np.random.default_rng(0)
    er = 0.0
    for T in spec.towers:
        for Ly in T.layers:
            if Ly.kind != mpn._lib.MPN_LAYER_CONV:
                continue
            rows = rng.choice(Ly.cout, 8, replace=False)
            g = tr.gradient(Ly.weight).reshape(Ly.cout, -1)[rows]
            er = max(er, rel_err(g, grads[Ly.weight].reshape(Ly.cout, -1)[rows]))
    record_parity("train_full_size_mpn", loss=abs(L[0] - rl) / abs(rl), heads=eh, tower_rows=er)
    assert abs(L[0] - rl) / abs(rl) < 1e-4 and eh < 1e-3 and er < 1e-3, (L, rl, eh, er)
    tr.close(); m.close()

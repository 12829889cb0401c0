"""GPU: training with the integral loss (train.lua:288-294): a step trains the selected class head against fp64 autograd
of the single-head graph, the idle heads take a zero gradient and optim.sgd's zero-gradient step (bit for bit the host
rule), momentum and decay over a head switch, bits against a single-head model, inference after training, step_batch on
sample_integral's sets, the trunk training under an integral head, the recipe-sized step, and the refusals."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200.batch_provider import integral_set, integral_thresholds
from conftest import rel_err, record_parity
from _train_ref import step_oracle
from _train_trunk_ref import trunk_step_oracle
import _batch_provider_ref as bref

pytestmark = pytest.mark.gpu
DEV = "cuda" if torch.cuda.is_available() else "cpu"
K = 3


def _spec(kind, seed=21, integral_k=K):
    if kind == "mpn":
        return models.vgg16_multipathnet(21, seed=seed, width_div=4, fc_dim=256, integral_k=integral_k)
    return models.vgg16_fast_rcnn(21, seed=seed, width_div=4, fc_dim=256, integral_k=integral_k)


def _one_head(spec, k):
    """the single-head graph that step k of an integral model trains: class head k, the same towers and bbox head"""
    return dataclasses.replace(spec, cls_heads=[spec.cls_heads[k]], no_softmax=0)


def _batch(spec, sizes=((128, 176), (160, 208)), per_image=(40, 56), seed=0):
    rng = np.random.default_rng(seed)
    ims = [wl.transform(wl.raw_image(h, w, seed + i), spec.transformer) for i, (h, w) in enumerate(sizes)]
    rois = [wl.random_boxes(n, h, w, seed + i).astype(np.float32) for i, ((h, w), n) in enumerate(zip(sizes, per_image))]
    R, C_ = sum(per_image), spec.num_classes
    labels = rng.integers(1, C_ + 1, R).astype(np.int32)
    labels[:5] = 1
    tg = np.zeros((R, 4 * C_), np.float32)
    for r in range(R):
        if labels[r] > 1:
            tg[r, 4 * labels[r] - 4:4 * labels[r]] = rng.standard_normal(4) * 0.8
    return ims, rois, labels, tg


def _gates(tr, spec):
    out = {}
    for t, T in enumerate(spec.towers):
        for li, L in enumerate(T.layers):
            if L.kind == mpn._lib.MPN_LAYER_CONV and L.relu:
                out[(t, li)] = tr.relu_gate(t, li)
    return out


def _oracle(m, tr, spec, k, weights, labels, tg, p):
    """fp64 autograd of the single-head graph of head k on the device's pooled rows, dropout masks and ReLU sides"""
    pooled = {t: m.pooled(t) for t in range(len(spec.towers))}
    masks = {key: tr.dropout_mask(*key) for key in _gates(tr, spec)} if p > 0 else {}
    return step_oracle(_one_head(spec, k), pooled, masks, p, weights, labels, tg, dev=DEV, gates=_gates(tr, spec))


def _head_tensors(spec, k):
    return [spec.cls_heads[k].weight, spec.cls_heads[k].bias]


def _idle_sgd_bits(tr, spec, idle, before, lr, mom, damp, wd, first):
    """each idle head's weight and buffer after the step equal mpn_debug_sgd with g = 0 on their values before it"""
    lib = mpn.load_library()
    for k in idle:
        for i in _head_tensors(spec, k):
            w, buf = (a.copy().reshape(-1) for a in before[i])
            g = np.zeros_like(w)
            is_bias = i == spec.cls_heads[k].bias
            assert lib.mpn_debug_sgd(w.ctypes.data, g.ctypes.data, buf.ctypes.data, w.size, lr, mom, damp, 0.0 if is_bias else wd,
                                     1 if first else 0) == 0
            assert np.array_equal(tr._get(i, 0).reshape(-1).view(np.uint32), w.view(np.uint32)), (k, i)
            assert np.array_equal(tr.momentum_buffer(i).reshape(-1).view(np.uint32), buf.view(np.uint32)), (k, i)


@pytest.mark.parametrize("kind", ["mpn", "frcnn"])
def test_each_head_vs_fp64_and_idle_heads_zero(ctx, kind):
    spec = _spec(kind)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m, seed=7, integral=True)
    assert all(i in tr.trained for k in range(K) for i in _head_tensors(spec, k))
    ims, rois, labels, tg = _batch(spec)
    cfg = tr.cfg
    worst = {"loss": 0.0, "grad": 0.0, "logits": 0.0}
    for step, k in enumerate((1, 0, 2)):
        w0 = tr.weights()
        before = {i: (tr._get(i, 0), tr.momentum_buffer(i)) for j in range(K) if j != k for i in _head_tensors(spec, j)}
        tr.select_head(k)
        L = tr.step(ims, rois, labels, tg)
        (rl, rce, rsl), grads, (rlog, _) = _oracle(m, tr, spec, k, w0, labels, tg, 0.5)
        el = max(abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl)))
        eg = max(rel_err(tr.gradient(i), g) for i, g in grads.items())
        elog = rel_err(tr.outputs()[0], rlog)
        assert el < 1e-4 and eg < 1e-3 and elog < 1e-3, (k, L, (rl, rce, rsl), eg, elog)
        assert set(grads) | {i for j in range(K) if j != k for i in _head_tensors(spec, j)} == set(tr.trained)
        for j in range(K):
            if j != k:
                assert all(not tr.gradient(i).any() for i in _head_tensors(spec, j)), (k, j)
        assert tr.gradient(spec.cls_heads[k].weight).any()
        _idle_sgd_bits(tr, spec, [j for j in range(K) if j != k], before, cfg.lr, cfg.momentum, cfg.dampening, cfg.weight_decay, step == 0)
        worst = {"loss": max(worst["loss"], el), "grad": max(worst["grad"], eg), "logits": max(worst["logits"], elog)}
    record_parity(f"train_integral_{kind}", **worst)
    tr.close(); m.close()


@pytest.mark.parametrize("kind", ["mpn", "frcnn"])
def test_three_steps_heads_0_2_0_with_momentum_and_decay_vs_fp64(ctx, kind):
    spec = _spec(kind, seed=5)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    lr, mom, wd = 1e-2, 0.9, 5e-4
    tr = mpn.Trainer(m, lr=lr, momentum=mom, weight_decay=wd, seed=3, integral=True)
    ims, rois, labels, tg = _batch(spec, seed=4)
    w = {i: np.array(spec.weights[i], np.float64) for i in tr.trained}
    buf = {}
    biases = {L.bias for T in spec.towers for L in T.layers} | {h.bias for h in spec.cls_heads} | {spec.bbox_head.bias}
    # head 1 never trains: its masters follow the fp32 rule exactly (mpn_debug_sgd with g = 0, decay in fp32)
    never = {i: (np.array(spec.weights[i], np.float32), np.zeros(np.shape(spec.weights[i]), np.float32)) for i in _head_tensors(spec, 1)}
    lr32 = np.float32(lr)
    lib = mpn.load_library()
    for step, k in enumerate((0, 2, 0)):
        tr.select_head(k)
        tr.step(ims, rois, labels, tg)
        cur = [w[i] if i in w else spec.weights[i] for i in range(len(spec.weights))]
        _, grads, _ = _oracle(m, tr, spec, k, cur, labels, tg, 0.5)
        for i in w:                                                   # optim.sgd on every tensor, idle heads with g = 0
            g = grads.get(i, 0.0) + (0.0 if i in biases else wd) * w[i]
            buf[i] = g if step == 0 else mom * buf[i] + g
            w[i] = w[i] - lr * buf[i]
        for i, (a, b) in never.items():
            a, b = a.reshape(-1), b.reshape(-1)
            z = np.zeros_like(a)
            assert lib.mpn_debug_sgd(a.ctypes.data, z.ctypes.data, b.ctypes.data, a.size, float(lr32), mom, 0.0,
                                     0.0 if i in biases else wd, 1 if step == 0 else 0) == 0
        if step == 0:
            tr.decay(0.5); lr *= 0.5; lr32 = np.float32(lr32 * np.float32(0.5))
            for i in buf:
                buf[i] = buf[i] * 0.5
            never = {i: (a, (b * np.float32(0.5)).astype(np.float32)) for i, (a, b) in never.items()}
    got = tr.weights()
    moved = [i for i in w if i not in never]
    errs = {i: rel_err(got[i] - spec.weights[i], w[i] - spec.weights[i]) for i in moved}
    record_parity(f"train_integral_three_steps_{kind}", delta_max=max(errs.values()))
    assert max(errs.values()) < 1e-3, errs
    for i, (a, b) in never.items():
        assert np.array_equal(got[i].reshape(-1).view(np.uint32), a.reshape(-1).view(np.uint32)), i
        assert rel_err(got[i], w[i]) < 1e-6, i
    assert not np.array_equal(got[spec.cls_heads[1].weight], spec.weights[spec.cls_heads[1].weight])   # weight decay moved it
    tr.close(); m.close()


def test_idle_head_moves_without_weight_decay(ctx):
    """recipe's weightDecay = 0: head 0 trains, then idles and still moves by lr x its decaying momentum"""
    spec = _spec("mpn", seed=9)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m, lr=1e-2, momentum=0.9, weight_decay=0.0, seed=3, integral=True)
    ims, rois, labels, tg = _batch(spec, seed=6)
    tr.step(ims, rois, labels, tg)                                    # head 0
    w1 = tr._get(spec.cls_heads[0].weight, 0)
    b1 = tr.momentum_buffer(spec.cls_heads[0].weight)
    never = tr._get(spec.cls_heads[2].weight, 0)
    before = {i: (tr._get(i, 0), tr.momentum_buffer(i)) for j in (0, 2) for i in _head_tensors(spec, j)}
    tr.select_head(1)
    tr.step(ims, rois, labels, tg)
    w2 = tr._get(spec.cls_heads[0].weight, 0)
    assert not np.array_equal(w1, w2) and b1.any()
    np.testing.assert_allclose(w2, w1 - np.float32(1e-2) * (np.float32(0.9) * b1), rtol=1e-6, atol=1e-9)
    assert np.array_equal(tr._get(spec.cls_heads[2].weight, 0), never)   # never trained, no decay: stays put
    _idle_sgd_bits(tr, spec, [0, 2], before, 1e-2, 0.9, 0.0, 0.0, False)
    tr.close(); m.close()


@pytest.mark.parametrize("kind", ["mpn", "frcnn"])
def test_head0_bits_equal_a_single_head_model(ctx, kind):
    spec = _spec(kind, seed=13)
    one = _one_head(spec, 0)
    ims, rois, labels, tg = _batch(spec, seed=2)
    outs = []
    for s in (spec, spec, one):
        m = mpn.Model(ctx, s, max_rois=128, max_h=192, max_w=256)
        tr = mpn.Trainer(m, seed=11, integral=len(s.cls_heads) > 1)     # the K = 1 model takes the plain entry
        L = [tr.step(ims, rois, labels, tg) for _ in range(2)]
        shared = [i for i in tr.trained if i not in {t for j in range(1, len(s.cls_heads)) for t in _head_tensors(s, j)}]
        outs.append((L, {i: (tr._get(i, 0), tr.gradient(i), tr.momentum_buffer(i)) for i in shared}, tr.outputs()))
        tr.close(); m.close()
    for o in outs[1:]:
        assert o[0] == outs[0][0]
        assert o[1].keys() == outs[0][1].keys()
        for i in o[1]:
            assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(o[1][i], outs[0][1][i])), i
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(o[2], outs[0][2]))


def test_inference_after_training_sees_every_head(ctx):
    spec = _spec("mpn", seed=17)
    ims, rois, labels, tg = _batch(spec, seed=8)
    img, H, W = ims[1], ims[1].shape[1], ims[1].shape[2]
    boxes = wl.random_boxes(64, H, W, 11)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m, lr=0.05, seed=1, integral=True)
    for k in (0, 1, 2):
        tr.select_head(k)
        tr.step(ims, rois, labels, tg)
    s, b = m.detect(img, boxes, 1.0)
    trained = tr.weights()
    fresh = mpn.Model(ctx, dataclasses.replace(spec, weights=trained), max_rois=128, max_h=192, max_w=256)
    s2, b2 = fresh.detect(img, boxes, 1.0)
    stale = mpn.Model(ctx, dataclasses.replace(spec, weights=[trained[i] if i not in _head_tensors(spec, 1) else spec.weights[i]
                                                              for i in range(len(trained))]), max_rois=128, max_h=192, max_w=256)
    s3, _ = stale.detect(img, boxes, 1.0)
    assert np.array_equal(s, s2) and np.array_equal(b, b2)
    np.testing.assert_allclose(s.sum(1), 1.0, atol=1e-5)                   # the mean of K softmaxes
    assert not np.array_equal(s, s3)                                         # head 1's training reaches the scores
    tr.select_head(2)
    tr.step(ims, rois, labels, tg)                                           # and training continues after inference
    fresh.close(); stale.close(); tr.close(); m.close()


NCLS = 6
SCALE, MAX_SIZE = 160, 256


@pytest.fixture(scope="module")
def feed():
    gt, props, sizes = bref.synthetic_coco(40, NCLS, 11)
    return gt, props, sizes


def _image(sizes):
    def get(i):
        H, W = sizes[i]
        return np.random.default_rng(100 + i).integers(0, 256, (H, W, 3), dtype=np.uint8)
    return get


def test_step_batch_trains_the_head_of_the_sampled_set(ctx, feed):
    gt, props, sizes = feed
    spec = models.vgg16_fast_rcnn(NCLS + 1, seed=4, width_div=4, fc_dim=256, integral_k=3)
    db = mpn.RoiDB(ctx, gt, props, NCLS, integral_thresholds(3), best_number=45)
    prov = mpn.BatchProviderROI(db, _image(sizes), spec.transformer, scale=SCALE, max_size=MAX_SIZE, seed=31)
    prov.setup_data()
    ma = mpn.Model(ctx, spec, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
    mb = mpn.Model(ctx, spec, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
    ta, tb = mpn.Trainer(ma, seed=9, integral=True), mpn.Trainer(mb, seed=9, integral=True)
    sets = []
    for step in range(6):
        batch = prov.sample_integral(step)
        assert batch.set == integral_set(31, step, 3)
        sets.append(batch.set)
        ims, boxes, labels, targets = batch.to_host()
        la = ta.step_batch(batch)
        assert ta.head == batch.set
        tb.select_head(batch.set)                                            # the same step, the head chosen by hand
        lb = tb.step(ims, np.split(boxes, np.cumsum(batch.rois_per_image)[:-1]), labels, targets)
        assert la == lb, (step, la, lb)
        assert all(np.array_equal(a, b) for a, b in zip(ta.outputs(), tb.outputs()))
        for j in range(3):
            g = ta.gradient(spec.cls_heads[j].weight)
            assert g.any() == (j == batch.set), (step, j)
    assert len(set(sets)) > 1, sets
    for i in ta.trained:
        assert np.array_equal(ta._get(i, 0), tb._get(i, 0)), i
    # a RoiDB with another number of sets than class heads is refused, by the Python check and by the C entry
    db2 = mpn.RoiDB(ctx, gt, props, NCLS, integral_thresholds(2), best_number=45)
    prov2 = mpn.BatchProviderROI(db2, _image(sizes), spec.transformer, scale=SCALE, max_size=MAX_SIZE, seed=31)
    prov2.setup_data()
    batch = prov2.sample_integral(0)
    with pytest.raises(mpn.MpnError, match="2 threshold sets and the model 3 class heads"):
        ta.step_batch(batch)
    losses = np.zeros(3, np.float32)
    assert ctx.lib.mpn_model_train_step_batch(ma.h, db2.h, losses.ctypes.data) != 0
    assert b"2 threshold sets and the model 3 class heads" in ctx.lib.mpn_last_error(ctx.h)
    ta.close(); tb.close(); ma.close(); mb.close(); db.close(); db2.close()


def test_trunk_training_under_an_integral_head_vs_fp64(ctx):
    spec = models.vgg16_fast_rcnn(21, seed=21, width_div=4, fc_dim=256, integral_k=3)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m, seed=7, train_trunk=True, integral=True)
    ims, rois, labels, tg = _batch(spec)
    tr.select_head(1)
    L = tr.step(ims, rois, labels, tg)
    k0 = spec.trunk_train_from
    slots = {spec.trunk_layers[k0].in_slot} | {Ly.out_slot for Ly in spec.trunk_layers[k0:]}
    stored = [{s: tr.trunk_slot(i, s) for s in slots} for i in range(len(rois))]
    gates = {key: v for key, v in _gates(tr, spec).items()}
    (rl, rce, rsl), grads = trunk_step_oracle(_one_head(spec, 1), k0, stored, rois, labels, tg, spec.weights, gates, 0.5, dev=DEV)
    el = [abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl))]
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    idle = [i for j in (0, 2) for i in _head_tensors(spec, j)]
    assert set(grads) | set(idle) == set(tr.trained)
    record_parity("train_integral_trunk", loss=el[0], grad_max=max(eg.values()))
    assert max(el) < 1e-4, (L, (rl, rce, rsl))
    assert max(eg.values()) < 1e-3, eg
    assert all(not tr.gradient(i).any() for i in idle)
    tr.close(); m.close()


def test_full_size_integral_multipathnet_step(ctx):
    """the recipe's minibatch on vgg16_multipathnet(81, integral_k=6): 4 images at 800 x 1000, 64 ROIs each"""
    spec = models.vgg16_multipathnet(81, seed=1234, integral_k=6)
    m = mpn.Model(ctx, spec, max_rois=256, max_h=800, max_w=1000)
    tr = mpn.Trainer(m, seed=555, integral=True)
    ims, rois, labels, tg = _batch(spec, sizes=((800, 1000), (800, 1000), (600, 1000), (800, 900)), per_image=(64, 64, 64, 64), seed=3)
    tr.select_head(5)
    L = tr.step(ims, rois, labels, tg)
    assert all(np.isfinite(L)), L
    assert tr.gradient(spec.cls_heads[5].weight).any()
    assert all(not tr.gradient(spec.cls_heads[j].weight).any() for j in range(5))
    tr.close(); m.close()


def test_integral_spec_is_opt_in_and_head_selection_is_checked(ctx):
    """an integral model is refused without the integral loss (as before) and trains through Trainer(integral=True); select_head
    refuses heads outside 0..K-1, and a single-head model has head 0 only"""
    spec = _spec("mpn")
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    with pytest.raises(mpn.MpnError, match="integral head"):
        mpn.Trainer(m)
    cfg = mpn._lib.CTrainConfig(1e-3, 0.9, 0.0, 5e-4, 0.5, 1.0, 555)
    assert ctx.lib.mpn_model_train_begin(m.h, C.byref(cfg), C.byref(mpn._lib.CTrainSpec())) != 0      # integral = 0
    assert b"integral head" in ctx.lib.mpn_last_error(ctx.h)
    for opt in ("bf16", "fp8"):
        ctx.set_option(opt, 1)
        try:
            with pytest.raises(mpn.MpnError, match="bf16"):
                mpn.Trainer(m, integral=True)
        finally:
            ctx.set_option(opt, 0)
    tr = mpn.Trainer(m, integral=True)
    for k in (-1, K):
        with pytest.raises(mpn.MpnError, match=f"class head {k} out of range 0..{K - 1}"):
            tr.select_head(k)
    tr.select_head(K - 1)
    ims, rois, labels, tg = _batch(spec, seed=1)
    assert all(np.isfinite(tr.step(ims, rois, labels, tg)))
    tr.close(); m.close()
    one = _spec("frcnn", seed=3, integral_k=0)
    m1 = mpn.Model(ctx, one, max_rois=128, max_h=192, max_w=256)
    t1 = mpn.Trainer(m1, integral=True)                                     # K = 1 through the integral entry: head 0 only
    with pytest.raises(mpn.MpnError, match="class head 1 out of range 0..0"):
        t1.select_head(1)
    t1.close(); m1.close()

"""GPU: MultiPathNet's phase 2 (Trainer(phase2=True), set_phase2): the towers' ROI pooling backward (foveal regions,
several levels, the L2 normalisation) bit for bit against its in-order numpy restatement; the phase-2 step of
vgg16_multipathnet against fp64 torch autograd from each image's stored pool2 output, fed the device's ReLU sides, max
pool and ROI argmaxes, dropout masks and per-ROI gates; three steps across the switch against optim.sgd; phase 1 equal to
Trainer(model); determinism; inference after phase 2; an integral model; refusals; the COCO recipe's minibatch."""
import dataclasses

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import _ptr, _vp, _i32p, _i64p, _f32p
from conftest import rel_err, record_parity
from _train_phase2_ref import gather, norm_ab, phase2_step_oracle, roi_argmax

pytestmark = pytest.mark.gpu
DEV = "cuda" if torch.cuda.is_available() else "cpu"


# ------------------------------------------------------------------------------------------------ kernel level
def _split(x):
    """fp32 -> (hi, lo) bf16 bit planes with hi + lo close to x (bf16 by truncation of the bits)"""
    x = np.ascontiguousarray(x, np.float32)
    hi = (x.view(np.uint32) >> 16).astype(np.uint16)
    rest = x - (hi.astype(np.uint32) << 16).view(np.float32)
    lo = (rest.astype(np.float32).view(np.uint32) >> 16).astype(np.uint16)
    return hi, lo


def _join(hi, lo):
    return (hi.astype(np.uint32) << 16).view(np.float32) + (lo.astype(np.uint32) << 16).view(np.float32)


def _jobs_hook(ctx, hi, lo, rois, jobs, PW=7, PH=7, variant=2):
    H, W, C = hi.shape
    R, n = rois.shape[0], len(jobs)
    region = np.array([j["region"] for j in jobs], np.int32)
    scale = np.array([j["scale"] for j in jobs], np.float32)
    norm = np.array([j["normalize"] for j in jobs], np.int32)
    ld = np.array([j["g"].shape[-1] for j in jobs], np.int64)
    off = np.array([j["ch_off"] for j in jobs], np.int32)
    gs = [np.ascontiguousarray(j["g"], np.float32) for j in jobs]
    ptrs = (_vp * n)(*[g.ctypes.data for g in gs])
    grad = np.empty((H, W, C), np.float32)
    ab = np.empty((n, R, 2), np.float64)
    am = np.empty((n, R, PH * PW, C), np.int32)
    rc = ctx.lib.mpn_debug_roi_backward_jobs(ctx.h, _ptr(hi), _ptr(lo), H, W, C, _ptr(rois), R, PW, PH, variant, n,
                                              region.ctypes.data_as(_i32p), scale.ctypes.data_as(_f32p), norm.ctypes.data_as(_i32p),
                                              ld.ctypes.data_as(_i64p), off.ctypes.data_as(_i32p), ptrs, _ptr(grad), _ptr(ab), _ptr(am))
    ctx.check(rc, "mpn_debug_roi_backward_jobs")
    return grad, ab, am


def test_roi_backward_jobs_bits_vs_numpy(ctx):
    """five towers' jobs on one map: regions x1 .. x4 (x4 boxes clipped at the border), normalised and not, ties in hi
    and in lo, empty bins, one cell named by several jobs; the gather bit for bit, the argmaxes exactly, (a, b) within
    1e-12 of a double restatement from the device's argmaxes"""
    rng = np.random.default_rng(3)
    H, W, C, R, P = 23, 31, 64, 24, 7
    x = np.maximum(rng.standard_normal((H, W, C)).astype(np.float32), 0)
    x[5:9, 5:9, :8] = 1.5                                       # ties in hi (equal values)
    base = np.float32(2.0)
    x[12:15, 10:14, 8:16] = base                                # ties in lo: equal hi, different / equal lo
    x[12, 11, 8:16] = np.nextafter(base, np.float32(3))
    x[13, 12, 8:16] = np.nextafter(base, np.float32(3))
    hi, lo = _split(x)
    xj = _join(hi, lo)
    boxes = np.zeros((R, 5), np.float32)
    boxes[:, 0] = 1
    for r in range(R):
        w, h = rng.uniform(2, 200), rng.uniform(2, 150)
        x1, y1 = rng.uniform(-20, 8 * W), rng.uniform(-20, 8 * H)
        boxes[r, 1:] = (x1, y1, x1 + w, y1 + h)
    boxes[0, 1:] = (1, 1, 8 * W, 8 * H)                         # whole image: x4 leaves it on every side
    boxes[1, 1:] = (30, 30, 30.5, 30.5)                         # tiny ROI: empty bins at large regions
    boxes[2, 1:] = boxes[3, 1:]                                 # the same ROI twice: one cell named twice
    specs = [(0, 1, 0), (1, 1, 64), (2, 1, 128), (3, 0, 0), (1, 0, 64)]   # (region, normalize, ch_off)
    jobs = []
    for region, nm, off in specs:
        g = rng.standard_normal((R, P * P, 192)).astype(np.float32)
        jobs.append(dict(region=region, scale=1.0 / 8, normalize=nm, ch_off=off, g=g))
    grad, ab, am = _jobs_hook(ctx, hi, lo, boxes, jobs)
    xc = np.ascontiguousarray(xj.transpose(2, 0, 1))
    ref_jobs = []
    for k, j in enumerate(jobs):
        ram = roi_argmax(xc, boxes[:, 1:], j["region"], j["scale"], 2, P, P)
        assert np.array_equal(am[k], ram), k
        gsl = j["g"][:, :, j["ch_off"]:j["ch_off"] + C]
        jab = None
        if j["normalize"]:
            xv = np.where(ram >= 0, xj.reshape(H * W, C)[np.maximum(ram, 0), np.arange(C)], 0)
            ref = np.array([norm_ab(xv[r], gsl[r]) for r in range(R)])
            assert np.max(np.abs(ab[k] - ref) / np.maximum(np.abs(ref), 1e-300)) < 1e-12
            jab = ab[k]
        else:
            assert np.all(ab[k] == 0)
        ref_jobs.append(dict(argmax=ram, g=gsl, ab=jab))
    assert (ram < 0).any() and len({int(v) for v in am[:, 0].ravel()}) > 1
    want = gather(xj, ref_jobs)
    assert np.array_equal(grad.view(np.uint32), want.view(np.uint32))
    # one unnormalised region-0 job is the Fast R-CNN trunk path's kernel, bit for bit
    g1 = rng.standard_normal((R, P * P, C)).astype(np.float32)
    one, _, _ = _jobs_hook(ctx, hi, lo, boxes, [dict(region=0, scale=1.0 / 8, normalize=0, ch_off=0, g=g1)])
    old = np.empty((H, W, C), np.float32)
    ctx.check(ctx.lib.mpn_debug_roi_backward_nhwc(ctx.h, _ptr(hi), _ptr(lo), H, W, C, _ptr(boxes), R, P, P, np.float32(1.0 / 8), 2,
                                                   _ptr(g1), _ptr(old)), "mpn_debug_roi_backward_nhwc")
    assert np.array_equal(one.view(np.uint32), old.view(np.uint32))


# ------------------------------------------------------------------------------------------------ small graph
def _spec(seed=21, integral_k=0):
    return models.vgg16_multipathnet(21, seed=seed, width_div=4, fc_dim=256, integral_k=integral_k)


def _batch(spec, sizes=((128, 176), (160, 208)), per_image=(32, 32), seed=0):
    rng = np.random.default_rng(seed)
    ims = [wl.transform(wl.raw_image(h, w, seed + i), spec.transformer) for i, (h, w) in enumerate(sizes)]
    rois = [wl.random_boxes(n, h, w, seed + i).astype(np.float32) for i, ((h, w), n) in enumerate(zip(sizes, per_image))]
    for r, (h, w) in zip(rois, sizes):
        r[0] = (1, 1, w, h)                                      # the x4 region leaves the image
        r[1] = (w / 4, h / 4, 3 * w / 4, 3 * h / 4)
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
    for L in spec.trunk_layers[spec.phase2_from:]:
        if L.kind == mpn._lib.MPN_LAYER_CONV:
            out += [L.weight, L.bias]
    return out


def _oracle(tr, spec, weights, rois, labels, tg, p, head=0):
    k0 = spec.phase2_from
    slots = {spec.trunk_layers[k0].in_slot} | {L.out_slot for L in spec.trunk_layers[k0:]}
    stored = [{s: tr.trunk_slot(i, s) for s in slots} for i in range(len(rois))]
    gates = {}
    for t, T in enumerate(spec.towers):
        for li, L in enumerate(T.layers):
            if L.kind == mpn._lib.MPN_LAYER_CONV and L.relu:
                gates[(t, li)] = tr.relu_gate(t, li)
    return phase2_step_oracle(spec, k0, stored, rois, labels, tg, weights, gates, p, head=head, dev=DEV)


def _check_step(tr, spec, L, rois, labels, tg, name, head=0):
    (rl, rce, rsl), grads = _oracle(tr, spec, spec.weights if tr.steps == 1 else tr.weights(), rois, labels, tg, 0.5, head)
    el = [abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl))]
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    assert set(grads) <= set(tr.trained)
    for i in set(tr.trained) - set(grads):                      # idle class heads
        assert not np.any(tr.gradient(i))
    record_parity(name, loss=el[0], cls=el[1], bbox=el[2], grad_max=max(eg.values()),
                  trunk_grad_max=max(eg[i] for i in _trunk_params(spec)))
    assert max(el) < 1e-4, (L, (rl, rce, rsl))
    assert max(eg.values()) < 1e-3, {i: e for i, e in eg.items() if e >= 1e-3}


def test_phase2_step_losses_and_gradients_vs_fp64(ctx):
    spec = _spec()
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m, seed=7, phase2=True)
    tr.set_phase2()
    assert set(_trunk_params(spec)) <= set(tr.trained) and len(_trunk_params(spec)) == 18
    ims, rois, labels, tg = _batch(spec)
    L = tr.step(ims, rois, labels, tg)
    _check_step(tr, spec, L, rois, labels, tg, "train_phase2_step")
    tr.close(); m.close()


def test_phase2_three_steps_across_the_switch_vs_fp64(ctx):
    """phase 1, set_phase2(lr) (rate changed, every buffer zeroed), two phase-2 steps: optim.sgd in fp64 with the trunk
    joining with zero buffers and the ordinary update"""
    spec = _spec(seed=5)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    lr, mom, wd, lr2 = 1e-2, 0.9, 5e-4, 4e-3
    tr = mpn.Trainer(m, lr=lr, momentum=mom, weight_decay=wd, seed=3, phase2=True)
    ims, rois, labels, tg = _batch(spec, seed=4)
    trunk = set(_trunk_params(spec))
    w = {i: np.array(spec.weights[i], np.float64) for i in set(tr.trained) | trunk}
    buf = {}
    biases = {L.bias for T in spec.towers for L in T.layers} | {spec.cls_heads[0].bias, spec.bbox_head.bias} | \
             {L.bias for L in spec.trunk_layers}
    for k in range(3):
        if k == 1:
            tr.set_phase2(lr2)
            lr = lr2
            buf = {i: np.zeros_like(b) for i, b in buf.items()}
        tr.step(ims, rois, labels, tg)
        cur = [w[i] if i in w else spec.weights[i] for i in range(len(spec.weights))]
        if k == 0:
            assert not (trunk & set(tr.trained))
            _, grads = _oracle_phase1(tr, spec, cur, rois, labels, tg)
        else:
            _, grads = _oracle(tr, spec, cur, rois, labels, tg, 0.5)
        for i, g in grads.items():
            g = g + (0.0 if i in biases else wd) * w[i]
            buf[i] = g if (k == 0 and i not in buf) else mom * buf.get(i, 0 * g) + g
            w[i] = w[i] - lr * buf[i]
    got = tr.weights()
    errs = {i: rel_err(got[i] - spec.weights[i], w[i] - spec.weights[i]) for i in w}
    record_parity("train_phase2_three_steps", delta_max=max(errs.values()))
    assert max(errs.values()) < 1e-3, {i: e for i, e in errs.items() if e >= 1e-3}
    tr.close(); m.close()


def _oracle_phase1(tr, spec, weights, rois, labels, tg):
    """phase 1's gradients: the same oracle with the trunk frozen (its tensors' gradients dropped); the kept slots of a
    phase-1 step do not exist, so the trunk maps come from a frozen trunk call with the same weights"""
    frozen = mpn.Model(tr.ctx, dataclasses.replace(spec, weights=list(weights)), max_rois=128, max_h=192, max_w=256)
    k0 = spec.phase2_from
    slots = {spec.trunk_layers[k0].in_slot} | {L.out_slot for L in spec.trunk_layers[k0:]}
    stored = []
    for i, im in enumerate(_batch(spec, seed=4)[0]):
        frozen.trunk(im)
        stored.append({s: frozen.trunk_slot(s)[0] for s in slots})
    frozen.close()
    gates = {(t, li): tr.relu_gate(t, li) for t, T in enumerate(spec.towers) for li, L in enumerate(T.layers)
             if L.kind == mpn._lib.MPN_LAYER_CONV and L.relu}
    (l, ce, sl), grads = phase2_step_oracle(spec, k0, stored, rois, labels, tg, weights, gates, 0.5, dev=DEV)
    return (l, ce, sl), {i: g for i, g in grads.items() if i not in set(_trunk_params(spec))}


def test_phase2_without_switch_is_trainer_bit_for_bit(ctx):
    spec = _spec(seed=13)
    ims, rois, labels, tg = _batch(spec, seed=6)
    outs = []
    for phase2 in (False, True):
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        tr = mpn.Trainer(m, seed=99, phase2=phase2)
        ls = [tr.step(ims, rois, labels, tg) for _ in range(2)]
        outs.append((ls, tr.weights()))
        tr.close(); m.close()
    assert outs[0][0] == outs[1][0]
    assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(outs[0][1], outs[1][1]))


def test_phase2_two_trainers_same_bits(ctx):
    spec = _spec(seed=17)
    ims, rois, labels, tg = _batch(spec, seed=8)
    outs = []
    for _ in range(2):
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        tr = mpn.Trainer(m, seed=5, phase2=True)
        ls = [tr.step(ims, rois, labels, tg)]
        tr.set_phase2(2e-3)
        ls += [tr.step(ims, rois, labels, tg) for _ in range(2)]
        outs.append((ls, [tr.gradient(i) for i in tr.trained], tr.weights()))
        tr.close(); m.close()
    assert outs[0][0] == outs[1][0]
    for k in (1, 2):
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(outs[0][k], outs[1][k]))


def test_phase2_inference_equals_model_from_weights(ctx):
    spec = _spec(seed=23)
    ims, rois, labels, tg = _batch(spec, seed=9)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m, lr=1e-2, seed=2, phase2=True)
    tr.set_phase2()
    tr.step(ims, rois, labels, tg)
    trained = tr.weights()
    assert any(not np.array_equal(trained[i], spec.weights[i]) for i in _trunk_params(spec))
    r5 = np.concatenate([np.ones((len(rois[0]), 1), np.float32), rois[0]], 1)
    m.trunk(ims[0])
    s1, b1 = m.heads(r5)
    fresh = mpn.Model(ctx, dataclasses.replace(spec, weights=trained), max_rois=128, max_h=192, max_w=256)
    fresh.trunk(ims[0])
    s2, b2 = fresh.heads(r5)
    assert np.array_equal(s1, s2) and np.array_equal(b1, b2)
    tr.close(); m.close(); fresh.close()


def test_phase2_integral_vs_fp64(ctx):
    spec = _spec(seed=29, integral_k=3)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    tr = mpn.Trainer(m, seed=11, phase2=True, integral=True)
    tr.set_phase2()
    tr.select_head(2)
    ims, rois, labels, tg = _batch(spec, seed=10)
    L = tr.step(ims, rois, labels, tg)
    _check_step(tr, spec, L, rois, labels, tg, "train_phase2_integral", head=2)
    tr.close(); m.close()


def test_phase2_refusals(ctx):
    spec = _spec(seed=1)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    with pytest.raises(mpn.MpnError, match="trunk_train_from is 0"):
        mpn.Trainer(m, train_trunk=True)
    with pytest.raises(mpn.MpnError, match="exclude each other"):
        mpn.Trainer(m, train_trunk=True, phase2=True)
    with pytest.raises(mpn.MpnError, match="not made with phase2"):
        tr = mpn.Trainer(m)
        try:
            tr.set_phase2()
        finally:
            tr.close()
    tr = mpn.Trainer(m, phase2=True)
    tr.set_phase2()
    with pytest.raises(mpn.MpnError, match="already made"):
        tr.set_phase2()
    tr.close(); m.close()
    fr = models.vgg16_fast_rcnn(21, seed=1, width_div=4, fc_dim=256)
    m = mpn.Model(ctx, fr, max_rois=128, max_h=192, max_w=256)
    with pytest.raises(mpn.MpnError, match="phase2_from is 0"):
        mpn.Trainer(m, phase2=True)
    m.close()
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    m.trunk(_batch(spec)[0][0])                                 # a trunk call releases the trunk's fp32 weights
    with pytest.raises(mpn.MpnError, match="before its first trunk call"):
        mpn.Trainer(m, phase2=True)
    m.close()
    for opt in ("bf16", "fp8"):
        ctx.set_option(opt, 1)
        m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
        try:
            with pytest.raises(mpn.MpnError, match="bf16"):
                mpn.Trainer(m, phase2=True)
        finally:
            m.close()
            ctx.set_option(opt, 0)


# ------------------------------------------------------------------------------------------------ full size
def test_phase2_coco_recipe_minibatch_vs_fp64(ctx):
    """train_multipathnet_coco.sh: four images (800 x 1000, 800 x 1000, 666 x 1000, 800 x 800), 64 ROIs each, integral
    K = 6, in phase 2: loss, head gradients and 16 sampled rows of conv3_1's, conv4_1's and conv5_3's weight gradients"""
    spec = models.vgg16_multipathnet(81, seed=41, integral_k=6)
    sizes = ((800, 1000), (800, 1000), (666, 1000), (800, 800))
    m = mpn.Model(ctx, spec, max_rois=256, max_h=1000, max_w=1000)
    tr = mpn.Trainer(m, seed=4, phase2=True, integral=True)
    tr.set_phase2()
    tr.select_head(4)
    ims, rois, labels, tg = _batch(spec, sizes=sizes, per_image=(64,) * 4, seed=12)
    L = tr.step(ims, rois, labels, tg)
    (rl, rce, rsl), grads = _oracle(tr, spec, spec.weights, rois, labels, tg, 0.5, head=4)
    el = max(abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl)))
    heads = [spec.cls_heads[4].weight, spec.cls_heads[4].bias, spec.bbox_head.weight, spec.bbox_head.bias]
    eh = max(rel_err(tr.gradient(i), grads[i]) for i in heads)
    convs = [L_ for L_ in spec.trunk_layers[spec.phase2_from:] if L_.kind == mpn._lib.MPN_LAYER_CONV]
    rng = np.random.default_rng(0)
    et = {}
    for name, L_ in (("conv3_1", convs[0]), ("conv4_1", convs[3]), ("conv5_3", convs[-1])):
        rows = rng.choice(L_.cout, 16, replace=False)
        et[name] = rel_err(tr.gradient(L_.weight)[rows], grads[L_.weight][rows])
    record_parity("train_phase2_coco", loss=el, head_grad=eh, **et)
    # as for the full-size Fast R-CNN trunk step, the oracle starts nine convolutions below the loss, where each device
    # layer stores its output as split planes: the loss is held to 2e-4 at this size
    assert el < 2e-4 and eh < 1e-3 and max(et.values()) < 1e-3, (el, eh, et)
    tr.close(); m.close()

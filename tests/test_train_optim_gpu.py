"""GPU: train.lua's other optim methods on the device. After every step each trained master and state equals the numpy
fp32 restatement of csrc/train_rule.cuh (tests/test_train_optim_cpu.py) applied to the device's own gradients, bit for
bit, on the small VGG-16 Fast R-CNN with its trunk, the integral MultiPathNet across the phase-2 switch, ResNet-18 with
fixed batch norm and in bf16; the hooks move only the rate; determinism, inference after training, the default against
an explicit sgd, resume bit for bit, and a falling loss under adam."""
import dataclasses

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200.batch_provider import integral_thresholds
from multipathnet_b200.train import _train_optim
from test_train_optim_cpu import restate
from test_fit_gpu import NCLS, SCALE, MAX_SIZE, _Setup, _image, _outcome, _run, _script, feed  # noqa: F401

pytestmark = pytest.mark.gpu
f32 = np.float32


def _snapshot(tr):
    return {i: (tr._get(i, 0),) + tr.optim_state(i) for i in tr.trained}


def _check_step(tr, o, before, t, lr, fixed=None, idle=()):
    """every trained tensor after step t against the restatement on the device's gradient (idle: no-gradient rule), and
    the fp64 rule on the same inputs within 1e-5 normwise"""
    wd = tr.cfg.weight_decay
    for i, (w0, *s0) in before.items():
        two = len(s0) == 2
        s1, s2 = s0[0], (s0[1] if two else np.zeros_like(w0))
        g = None if i in idle else tr.gradient(i)
        wdi = 0.0 if np.ndim(w0) == 1 else wd
        a = None
        if fixed is not None and i in fixed:
            a = np.broadcast_to(np.asarray(fixed[i], f32).reshape(-1, *([1] * (np.ndim(w0) - 1))), np.shape(w0)).copy()
        w, r1, r2 = restate(o, w0, g, s1, s2, a, f32(lr), wdi, t)
        got = (tr._get(i, 0),) + tr.optim_state(i)
        assert np.array_equal(got[0], w), (i, t)
        assert np.array_equal(got[1], r1), (i, t)
        if two:
            assert np.array_equal(got[2], r2), (i, t)
        if a is None:
            w64 = _fp64(o, w0, g, s1, s2, lr, wdi, t)
            # 1e-5 of the step, plus the one fp32 rounding of the stored result
            bar = 1e-5 * np.linalg.norm(w64 - w0.astype(np.float64)) + 2.0 ** -24 * np.linalg.norm(w64)
            assert np.linalg.norm(got[0].astype(np.float64) - w64) <= bar, (i, t)


def _fp64(o, w, g, s1, s2, lr, wd, t):
    """optim's rule in fp64 on the same fp32 inputs (the sanity check beside the bit-exact restatement)"""
    w, s1, s2 = (np.asarray(x, np.float64) for x in (w, s1, s2))
    g = np.zeros_like(w) if g is None else np.asarray(g, np.float64)
    g = g + wd * w
    T, clr = t + 1.0, float(lr) / (1.0 + t * o.lr_decay)
    if o.method == 1:
        m, v = o.beta1 * s1 + (1 - o.beta1) * g, o.beta2 * s2 + (1 - o.beta2) * g * g
        return w - clr * np.sqrt(1 - o.beta2 ** T) / (1 - o.beta1 ** T) * m / (np.sqrt(v) + o.epsilon)
    if o.method == 2:
        m, u = o.beta1 * s1 + (1 - o.beta1) * g, np.maximum(o.beta2 * s2, np.abs(g) + o.epsilon)
        return w - float(lr) / (1 - o.beta1 ** T) * m / u
    if o.method == 3:
        return w - clr * g / (np.sqrt(s1 + g * g) + 1e-10)
    if o.method == 4:
        return w - float(lr) * g / (np.sqrt(o.alpha * s1 + (1 - o.alpha) * g * g) + o.epsilon)
    m = g if t == 0 else 0.9 * s1 + g
    return w - clr * m


OPT = {"adam": dict(lr_decay=1e-2), "adamax": {}, "adagrad": dict(lr_decay=1e-2), "rmsprop": {}, "sgd": dict(lr_decay=1e-2)}


@pytest.mark.parametrize("method", list(OPT))
def test_each_method_matches_the_restatement_on_the_vgg_trunk(ctx, feed, method):
    setup = _Setup(ctx, feed, "vgg_trunk")
    setup.kw = dict(setup.kw, method=method, **OPT[method])
    tr = setup.trainer(lr=1e-3)
    o = _train_optim(method, **OPT[method])
    for t in range(3):
        if t == 2:
            tr.decay(0.5)
        before = _snapshot(tr)
        setup.step(tr, t)
        _check_step(tr, o, before, t, tr.cfg.lr)
    assert all(np.isfinite(w).all() for w in tr.weights())
    tr.close(); tr.model.close()


def test_integral_multipathnet_across_the_switch_under_adam(ctx, feed):
    """idle heads take the no-gradient rule; set_phase2(lr), decay and _zero_buffers leave every state untouched; the
    trunk tensors start from zero state with the global t"""
    setup = _Setup(ctx, feed, "mpn_phase2")
    setup.kw = dict(setup.kw, method="adam")
    tr = setup.trainer()
    o = _train_optim("adam")
    heads = setup.spec.cls_heads
    for t in range(3):
        if t == 2:
            held = _snapshot(tr)
            tr.set_phase2(0.004)
            tr.decay(0.5)
            tr._zero_buffers()
            assert tr.cfg.lr == f32(f32(0.004) * f32(0.5))
            for i, ts in held.items():
                assert all(np.array_equal(a, b) for a, b in zip(ts, _snapshot(tr)[i]))
            new = [i for i in tr.trained if i not in held]
            assert new and all(not s.any() for i in new for s in tr.optim_state(i))
        before = _snapshot(tr)
        batch = setup.prov.sample_integral(t)
        tr.step_batch(batch)
        idle = {i for k, h in enumerate(heads) if k != tr.head for i in (h.weight, h.bias) if i >= 0}
        _check_step(tr, o, before, t, tr.cfg.lr, idle=idle)
    tr.close(); tr.model.close()


def test_resnet18_fixed_batch_norm_under_adam(ctx, feed):
    setup = _Setup(ctx, feed, "resnet18")
    setup.kw = dict(setup.kw, method="adam")
    tr = setup.trainer()
    o = _train_optim("adam")
    fixed = {i: a for i, a in setup.spec.fixed_bn.items() if i in tr.trained}
    assert fixed
    for t in range(2):
        before = _snapshot(tr)
        setup.step(tr, t)
        idle = {i for k, h in enumerate(setup.spec.cls_heads) if k != tr.head for i in (h.weight, h.bias) if i >= 0}
        _check_step(tr, o, before, t, tr.cfg.lr, fixed=fixed, idle=idle)
        for i, a in fixed.items():                                  # fp64 on the unfolded W, within 1e-5 normwise
            w0, m0, v0 = before[i]
            ab = np.asarray(a, np.float64).reshape(-1, *([1] * (np.ndim(w0) - 1)))
            W0 = w0 / ab
            W64 = _fp64(o, W0, ab * tr.gradient(i), m0, v0, tr.cfg.lr, tr.cfg.weight_decay, t)
            # W' = fl(a W) is rounded once more than W: two fp32 roundings beside 1e-5 of the step
            assert np.linalg.norm(tr._get(i, 0) / ab - W64) <= 1e-5 * np.linalg.norm(W64 - W0) + 2.0 ** -23 * np.linalg.norm(W64)
    tr.close(); tr.model.close()


def test_bf16_under_adam(ctx, feed):
    setup = _Setup(ctx, feed, "vgg_trunk")
    setup.kw = dict(setup.kw, method="adam", bf16=True)
    tr = setup.trainer(lr=1e-3)
    o = _train_optim("adam")
    for t in range(2):
        before = _snapshot(tr)
        setup.step(tr, t)
        _check_step(tr, o, before, t, tr.cfg.lr)
    tr.close(); tr.model.close()


def test_determinism_inference_and_the_default_method(ctx, feed):
    setup = _Setup(ctx, feed, "vgg_trunk")
    img = wl.transform(wl.raw_image(144, 192, 3), setup.spec.transformer)
    boxes = wl.random_boxes(40, 144, 192, 5)
    runs = []
    for kw in (dict(method="adam"), dict(method="adam"), {}, dict(method="sgd", lr_decay=0.0)):
        setup.kw = dict(train_trunk=True, **kw)
        tr = setup.trainer(lr=1e-3)
        losses = [setup.step(tr, t) for t in range(3)]
        ws = tr.weights()
        states = [s for i in tr.trained for s in tr.optim_state(i)]
        det = tr.model.detect(img, boxes, 1.0)
        runs.append((losses, ws, states, det, tr._fingerprint))
        if len(runs) == 1:                                          # inference after training = a model built from weights()
            fresh = mpn.Model(ctx, dataclasses.replace(setup.spec, weights=ws), max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
            assert all(np.array_equal(a, b) for a, b in zip(det, fresh.detect(img, boxes, 1.0)))
            fresh.close()
        tr.close(); tr.model.close()
    for a, b in ((runs[0], runs[1]), (runs[2], runs[3])):
        assert a[0] == b[0] and a[4] == b[4]
        assert all(np.array_equal(x, y) for x, y in zip(a[1], b[1]))
        assert all(np.array_equal(x, y) for x, y in zip(a[2], b[2]))
        assert all(np.array_equal(x, y) for x, y in zip(a[3], b[3]))
    assert "optim" not in runs[2][4] and runs[0][4]["optim"]["method"] == "adam"
    assert not all(np.array_equal(x, y) for x, y in zip(runs[0][1], runs[2][1]))


@pytest.mark.parametrize("which,method,k,switch", [("vgg_trunk", "adam", 1, None), ("vgg_trunk", "adam", 3, None),
                                                   ("mpn_phase2", "rmsprop", 1, 2), ("mpn_phase2", "rmsprop", 3, 2),
                                                   ("resnet18", "adagrad", 1, None), ("resnet18", "adagrad", 3, None)])
def test_resume_equals_uninterrupted(ctx, feed, tmp_path, which, method, k, switch):
    setup = _Setup(ctx, feed, which)
    setup.kw = dict(setup.kw, method=method)
    n = k + 2
    first, rest = _script(k, n, switch)
    ta = setup.trainer()
    la = _run(setup, ta, first + rest)
    want, want_s = _outcome(setup, ta), _snapshot(ta)
    tb = setup.trainer()
    lb = _run(setup, tb, first)
    path = str(tmp_path / "ck.npz")
    mpn.save_checkpoint(path, tb)
    tb.close(); tb.model.close()
    tc = setup.trainer()
    tc.load_state_dict(mpn.load_checkpoint(path))
    lb += _run(setup, tc, rest)
    got, got_s = _outcome(setup, tc), _snapshot(tc)
    assert la == lb
    assert all(np.array_equal(a, c) for a, c in zip(want[0], got[0]))
    assert want_s.keys() == got_s.keys() and all(np.array_equal(a, c) for i in want_s for a, c in zip(want_s[i], got_s[i]))
    assert all(np.array_equal(a, c) for a, c in zip(want[3], got[3])) and want[4] == got[4]
    for t in (ta, tc):
        t.close(); t.model.close()


def test_adam_lowers_the_loss_over_200_steps(ctx, feed):
    gt, props, sizes = feed
    spec = models.vgg16_fast_rcnn(NCLS + 1, seed=5, width_div=4, fc_dim=256)
    db = mpn.RoiDB(ctx, gt, props, NCLS, integral_thresholds(1), best_number=45)
    prov = mpn.BatchProviderROI(db, _image(sizes), spec.transformer, batch_size=48, scale=SCALE, max_size=MAX_SIZE, seed=31)
    prov.setup_data()
    m = mpn.Model(ctx, spec, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
    tr = mpn.Trainer(m, lr=1e-4, train_trunk=True, method="adam")
    losses = [tr.step_batch(prov.sample(k))[0] for k in range(200)]
    assert np.isfinite(losses).all()
    assert np.mean(losses[-20:]) < np.mean(losses[:20]), (np.mean(losses[:20]), np.mean(losses[-20:]))
    tr.close(); m.close()

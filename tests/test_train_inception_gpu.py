"""GPU: training Inception-v3 Fast R-CNN's per-ROI tower with fixed batch norm (models.inception_v3_fast_rcnn(fixed_bn=True),
inceptionv3.lua's BNtoFixed): Mixed_7a .. 7c and the heads, the trunk frozen, against fp64 torch autograd on the unfolded
tower (_train_inception_ref.py); the backward kernels of its 1 x n / n x 1 / 3 x 3-s2-valid convolutions and its windowed
average pools; three SGD steps, the integral loss, determinism, inference after training, resume, a live trainer over
changing shapes, bf16 training, the refusals, and the COCO recipe's minibatch."""
import dataclasses

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import MPN_LAYER_CONV, _i32p
from conftest import rel_err, record_parity
from _train_bf16_ref import bars, split_planes, three_oracles, unit_scales
from _train_inception_ref import avgpool_win_backward_np, inception_step_oracle, joined
from _train_resnet_ref import fold, sgd_unfolded, unfolded

pytestmark = pytest.mark.gpu
DEV = "cuda" if torch.cuda.is_available() else "cpu"
NAN16 = np.uint16(0x7FC0)


def _spec(seed=21, integral_k=0, C=5):
    return models.inception_v3_fast_rcnn(C, seed=seed, integral_k=integral_k, fixed_bn=True)


def _model(ctx, spec, max_rois=32, max_hw=(192, 224)):
    return mpn.Model(ctx, spec, max_rois=max_rois, max_h=max_hw[0], max_w=max_hw[1])


def _batch(spec, sizes=((160, 192), (128, 176)), per_image=(5, 4), seed=0):
    rng = np.random.default_rng(seed)
    ims = [wl.transform(wl.raw_image(h, w, seed + i), spec.transformer) for i, (h, w) in enumerate(sizes)]
    rois = [wl.random_boxes(n, h, w, seed + i).astype(np.float32) for i, ((h, w), n) in enumerate(zip(sizes, per_image))]
    R, C = sum(per_image), spec.num_classes
    labels = rng.integers(1, C + 1, R).astype(np.int32)
    labels[:2] = 1
    tg = np.zeros((R, 4 * C), np.float32)
    for r in range(R):
        if labels[r] > 1:
            tg[r, 4 * labels[r] - 4:4 * labels[r]] = rng.standard_normal(4) * 0.8
    return ims, rois, labels, tg


def _oracle(m, tr, spec, weights, labels, tg, head=0):
    pooled = joined(m.slot_planes(0, 0))
    gates = {li: tr.relu_gate(0, li) for li, L in enumerate(spec.towers[0].layers) if L.kind == MPN_LAYER_CONV and L.relu}
    return inception_step_oracle(spec, pooled, labels, tg, weights, gates, head=head, dev=DEV)


def _constants(spec):
    """the entries that never train: the trunk and the recorded layers' biases"""
    out = {i for L in spec.trunk_layers for i in (L.weight, L.bias) if i >= 0}
    return out | {L.bias for L in spec.towers[0].layers if L.weight in spec.fixed_bn}


# ---------------------------------------------------------------------------------------------------- the kernels
CONV_CASES = [(1, 7, 1, 0, 3), (7, 1, 1, 3, 0), (1, 3, 1, 0, 1), (3, 1, 1, 1, 0), (3, 3, 2, 0, 0)]


@pytest.mark.parametrize("hw", [17, 8])
@pytest.mark.parametrize("kh,kw,stride,ph,pw", CONV_CASES, ids=lambda v: str(v))
def test_conv_backward_ext_in_a_nan_padded_slice_vs_fp64(ctx, kh, kw, stride, ph, pw, hw):
    rng = np.random.default_rng(kh * 10 + kw + stride + hw)
    R, cin, cout, x_off, ldx, g_off, ldg = 3, 128, 64, 32, 192, 16, 96
    Ho, Wo = (hw + 2 * ph - kh) // stride + 1, (hw + 2 * pw - kw) // stride + 1
    x = rng.standard_normal((R, hw, hw, cin)).astype(np.float32)
    hi, lo = split_planes(x)
    xh = np.full((R, hw, hw, ldx), NAN16, np.uint16); xl = xh.copy()
    xh[..., x_off:x_off + cin], xl[..., x_off:x_off + cin] = hi, lo
    g = rng.standard_normal((R, Ho, Wo, cout)).astype(np.float32)
    gfull = np.full((R, Ho, Wo, ldg), np.nan, np.float32)
    gfull[..., g_off:g_off + cout] = g
    w = (rng.standard_normal((cout, cin, kh, kw)) * np.sqrt(2.0 / (cin * kh * kw))).astype(np.float32)
    dw, dx = np.empty_like(w), np.empty((R, hw, hw, cin), np.float32)
    sizes = np.array([hw, hw] * R, np.int32)
    ctx.check(ctx.lib.mpn_debug_conv_backward_ext(ctx.h, R, sizes.ctypes.data_as(_i32p), cin, cout, kh, kw, stride, ph, pw, xh.ctypes.data,
                                                  xl.ctypes.data, ldx, x_off, gfull.ctypes.data, ldg, g_off, w.ctypes.data, dw.ctypes.data,
                                                  dx.ctypes.data), "mpn_debug_conv_backward_ext")
    xv = joined(dict(hi=hi, lo=lo))
    X = torch.tensor(xv, dtype=torch.float64, device=DEV).permute(0, 3, 1, 2).requires_grad_(True)
    Wt = torch.tensor(w, dtype=torch.float64, device=DEV, requires_grad=True)
    Y = torch.nn.functional.conv2d(X, Wt, stride=stride, padding=(ph, pw))
    Y.backward(torch.tensor(g, dtype=torch.float64, device=DEV).permute(0, 3, 1, 2))
    ew = rel_err(dw, Wt.grad.cpu().numpy())
    ex = rel_err(dx, X.grad.permute(0, 2, 3, 1).cpu().numpy())
    record_parity(f"train_inception_conv_bwd_{kh}x{kw}s{stride}_{hw}", dw=ew, dx=ex)
    assert np.all(np.isfinite(dw)) and np.all(np.isfinite(dx))          # no NaN neighbour was read
    assert ew < 1e-4 and ex < 1e-4, (ew, ex)


@pytest.mark.parametrize("xp", [0, 1])
@pytest.mark.parametrize("n,H,W,C", [(3, 17, 17, 64), (4, 8, 8, 128), (1, 35, 60, 32)])
def test_avgpool_win_backward_bits_vs_numpy_and_fp64(ctx, n, H, W, C, xp):
    rng = np.random.default_rng(H * W + xp)
    ld, off = C + 24, 8
    g = rng.standard_normal((n, H, W, C)).astype(np.float32)          # 3 x 3 / 1 / 1: Ho x Wo = H x W
    gfull = np.full((n, H, W, ld), np.nan, np.float32)
    gfull[..., off:off + C] = g
    out = np.empty((n, H, W, C), np.float32)
    ctx.check(ctx.lib.mpn_debug_avgpool_win_backward(ctx.h, n, H, W, C, 3, 1, 1, xp, gfull.ctypes.data, ld, off, out.ctypes.data),
              "mpn_debug_avgpool_win_backward")
    assert np.array_equal(out.view(np.uint32), avgpool_win_backward_np(g, H, W, 3, 1, 1, xp).view(np.uint32))
    X = torch.zeros((n, C, H, W), dtype=torch.float64, requires_grad=True)
    Y = torch.nn.functional.avg_pool2d(X, 3, 1, 1, count_include_pad=not xp)
    Y.backward(torch.tensor(g, dtype=torch.float64).permute(0, 3, 1, 2))
    e = rel_err(out, X.grad.permute(0, 2, 3, 1).numpy())
    record_parity(f"train_inception_avgpool_bwd_{H}x{W}_xp{xp}", err=e)
    assert e < 1e-6, e


# ------------------------------------------------------------------------------------------------ the step vs fp64
def test_step_losses_and_gradients_vs_fp64(ctx):
    spec = _spec()
    m = _model(ctx, spec)
    tr = mpn.Trainer(m, seed=7)
    assert not (set(tr.trained) & _constants(spec))
    assert set(tr.trained) | _constants(spec) == set(range(len(spec.weights)))
    ims, rois, labels, tg = _batch(spec)
    L = tr.step(ims, rois, labels, tg)
    (rl, rce, rsl), grads = _oracle(m, tr, spec, spec.weights, labels, tg)
    el = [abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl))]
    assert set(grads) == set(tr.trained)
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    record_parity("train_inception_step", loss=el[0], cls=el[1], bbox=el[2], grad_max=max(eg.values()))
    assert max(el) < 1e-4, (L, (rl, rce, rsl))
    assert max(eg.values()) < 1e-3, eg
    tr.close(); m.close()


def test_three_steps_with_momentum_and_decay_vs_fp64_sgd_on_the_unfolded_weights(ctx):
    spec = _spec(seed=5)
    m = _model(ctx, spec)
    lr, mom, wd = 1e-2, 0.9, 5e-4
    tr = mpn.Trainer(m, lr=lr, momentum=mom, weight_decay=wd, seed=3)
    ims, rois, labels, tg = _batch(spec, seed=4)
    w = {i: v for i, v in unfolded(spec, spec.weights).items() if i in tr.trained}
    buf = {}
    biases = {L.bias for L in spec.towers[0].layers} | {h.bias for h in spec.cls_heads} | {spec.bbox_head.bias}
    for k in range(3):
        tr.step(ims, rois, labels, tg)
        cur = fold(spec, w)
        _, grads = _oracle(m, tr, spec, [cur.get(i, spec.weights[i]) for i in range(len(spec.weights))], labels, tg)
        sgd_unfolded(spec, w, buf, grads, lr, mom, wd, k == 0, biases)
        if k == 0:
            tr.decay(0.5); lr *= 0.5
            for i in buf:
                buf[i] = buf[i] * 0.5
    got, want = tr.weights(), fold(spec, w)
    errs = {i: rel_err(got[i] - spec.weights[i], want[i] - spec.weights[i]) for i in w}
    record_parity("train_inception_three_steps", delta_max=max(errs.values()))
    assert max(errs.values()) < 1e-3, errs
    for i in _constants(spec):
        assert np.array_equal(got[i], spec.weights[i])
    tr.close(); m.close()


def test_integral_step_vs_fp64_and_idle_heads_take_the_zero_gradient_update(ctx):
    spec = _spec(seed=8, integral_k=3)
    m = _model(ctx, spec)
    lr, mom, wd = 1e-3, 0.9, 5e-4
    tr = mpn.Trainer(m, lr=lr, momentum=mom, weight_decay=wd, seed=7, integral=True)
    ims, rois, labels, tg = _batch(spec, seed=2)
    heads = [(h.weight, h.bias) for h in spec.cls_heads]
    before = {i: (np.array(spec.weights[i], np.float32), np.zeros(np.shape(spec.weights[i]), np.float32)) for hw in heads for i in hw}
    tr.select_head(2)
    L = tr.step(ims, rois, labels, tg)
    (rl, _, _), grads = _oracle(m, tr, spec, spec.weights, labels, tg, head=2)
    assert abs(L[0] - rl) / abs(rl) < 1e-4
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    assert max(eg.values()) < 1e-3, eg
    lib = mpn.load_library()
    for k in (0, 1):
        for i in heads[k]:
            assert not np.any(tr.gradient(i))
            w, b = (a.copy().reshape(-1) for a in before[i])
            z = np.zeros_like(w)
            assert lib.mpn_debug_sgd(w.ctypes.data, z.ctypes.data, b.ctypes.data, w.size, lr, mom, 0.0,
                                     0.0 if i == heads[k][1] else wd, 1) == 0
            assert np.array_equal(tr.weights()[i].reshape(-1).view(np.uint32), w.view(np.uint32)), (k, i)
            assert np.array_equal(tr.momentum_buffer(i).reshape(-1).view(np.uint32), b.view(np.uint32)), (k, i)
    tr.close(); m.close()


# ------------------------------------------------------------------------------------------------------------ bits
def _run(ctx, spec, batches, **kw):
    m = _model(ctx, spec)
    tr = mpn.Trainer(m, seed=99, **kw)
    ls = [tr.step(*b) for b in batches]
    out = (ls, [tr.gradient(i) for i in tr.trained], tr.weights())
    tr.close(); m.close()
    return out


def _same(a, b):
    assert a[0] == b[0]
    assert all(np.array_equal(x, y) for x, y in zip(a[1], b[1]))
    assert all(np.array_equal(x, y) for x, y in zip(a[2], b[2]))


def test_two_trainers_same_bits(ctx):
    spec = _spec(seed=13)
    b = _batch(spec, seed=6)
    _same(_run(ctx, spec, [b, b]), _run(ctx, spec, [b, b]))


def test_inference_after_a_step_equals_a_model_built_from_the_weights(ctx):
    spec = _spec(seed=17)
    m = _model(ctx, spec)
    tr = mpn.Trainer(m, seed=1)
    ims, rois, labels, tg = _batch(spec, seed=3)
    tr.step(ims, rois, labels, tg)
    s1, b1 = m.detect(ims[0], rois[0], 1.0)
    m2 = _model(ctx, dataclasses.replace(spec, weights=tr.weights()))
    s2, b2 = m2.detect(ims[0], rois[0], 1.0)
    assert np.array_equal(s1, s2) and np.array_equal(b1, b2)
    tr.close(); m.close(); m2.close()


def test_resume_from_a_checkpoint_equals_the_uninterrupted_run(ctx, tmp_path):
    spec = _spec(seed=19)
    batches = [_batch(spec, seed=s) for s in range(4)]
    whole = _run(ctx, spec, batches)
    m = _model(ctx, spec)
    tr = mpn.Trainer(m, seed=99)
    ls = [tr.step(*b) for b in batches[:2]]
    mpn.save_checkpoint(str(tmp_path / "ck.npz"), tr)
    tr.close(); m.close()
    m = _model(ctx, spec)
    tr = mpn.Trainer(m, seed=99)
    tr.load_state_dict(mpn.load_checkpoint(str(tmp_path / "ck.npz")))
    ls += [tr.step(*b) for b in batches[2:]]
    _same(whole, (ls, [tr.gradient(i) for i in tr.trained], tr.weights()))
    tr.close(); m.close()


def test_one_live_trainer_over_changing_shapes_equals_fresh_trainers(ctx):
    spec = _spec(seed=23)
    shapes = [(((160, 192), (128, 176)), (5, 4)), (((192, 224),), (7,)), (((128, 128), (160, 160), (144, 192)), (2, 3, 6)),
              (((160, 192), (128, 176)), (5, 4))]
    m = _model(ctx, spec)
    live = mpn.Trainer(m, seed=4)
    for k, (sizes, per) in enumerate(shapes):
        b = _batch(spec, sizes=sizes, per_image=per, seed=30 + k)
        state = live.state_dict()
        mf = _model(ctx, spec)
        fresh = mpn.Trainer(mf, seed=4)
        fresh.load_state_dict(state)
        la, lb = live.step(*b), fresh.step(*b)
        assert la == lb, k
        assert all(np.array_equal(live.gradient(i), fresh.gradient(i)) for i in live.trained), k
        assert all(np.array_equal(x, y) for x, y in zip(live.weights(), fresh.weights())), k
        fresh.close(); mf.close()
    live.close(); m.close()


# ------------------------------------------------------------------------------------------------------------ bf16
def test_bf16_step_vs_the_oracle_of_bf16_operands_and_deterministic(ctx):
    spec = _spec(seed=29)
    ims, rois, labels, tg = _batch(spec, seed=5)
    runs = []
    for _ in range(2):
        m = _model(ctx, spec)
        tr = mpn.Trainer(m, seed=7, bf16=True)
        L = tr.step(ims, rois, labels, tg)
        runs.append((L, {i: tr.gradient(i) for i in tr.trained}))
        if len(runs) == 1:
            unit = unit_scales(spec)
            plain, b64, b32 = three_oracles(lambda: _oracle(m, tr, unit, spec.weights, labels, tg))
            res = bars(L, runs[0][1], plain, b64, b32)
            worst = max(res.values(), key=lambda v: v[0] / v[1])
            record_parity("train_bf16_step_inception", err_max=max(v[0] for v in res.values()), bar_use=worst[0] / worst[1],
                          plain_max=max(v[2] for v in res.values()))
            bad = {k: v for k, v in res.items() if v[0] > max(5e-3, v[1]) or v[2] > v[3]}
            assert not bad, bad
        tr.close(); m.close()
    assert runs[0][0] == runs[1][0]
    assert all(np.array_equal(runs[0][1][i], runs[1][1][i]) for i in runs[0][1])


# ------------------------------------------------------------------------------------------------------- refusals
def test_refusals(ctx):
    spec = _spec(seed=3)
    m = _model(ctx, spec)
    with pytest.raises(mpn.MpnError, match="K tails"):
        mpn.Trainer(m, train_trunk=True)
    from multipathnet_b200._lib import CTrainConfig
    from multipathnet_b200.train import _train_spec
    s, _keep = _train_spec(spec, 5, False, False)
    assert ctx.lib.mpn_model_train_begin(m.h, CTrainConfig(1e-3, 0.9, 0.0, 5e-4, 0.5, 1.0, 1), s) != 0
    assert "K tails" in ctx.lib.mpn_last_error(ctx.h).decode()
    tr = mpn.Trainer(m)                                       # the refusals left the model as it was
    tr.step(*_batch(spec))
    tr.close(); m.close()


# ---------------------------------------------------------------------------------------------------- recipe size
def test_recipe_minibatch_step_finite_and_deterministic(ctx):
    spec = models.inception_v3_fast_rcnn(81, integral_k=6, fixed_bn=True)
    sizes = [(800, 1000), (800, 1000), (666, 1000), (800, 800)]
    b = _batch(spec, sizes=sizes, per_image=(64, 64, 64, 64))
    outs = []
    for _ in range(2):
        m = mpn.Model(ctx, spec, max_rois=256, max_h=1000, max_w=1000)
        tr = mpn.Trainer(m, seed=5, integral=True)
        L = tr.step(*b)
        g = [tr.gradient(i) for i in tr.trained[:4] + tr.trained[-4:]]
        outs.append((L, g))
        assert all(np.isfinite(L)) and all(np.all(np.isfinite(x)) for x in g)
        tr.close(); m.close()
    assert outs[0][0] == outs[1][0]
    assert all(np.array_equal(a, b) for a, b in zip(outs[0][1], outs[1][1]))

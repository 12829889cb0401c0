"""GPU: training ResNet Fast R-CNN with fixed batch norm (models.resnet{18,50}_fast_rcnn(fixed_bn=True), resnet.lua's
BNtoFixed): layer2 .. layer4 and the heads against fp64 torch autograd on the unfolded graph (_train_resnet_ref.py),
three SGD steps against optim.sgd on the unfolded W, determinism, the frozen forward, inference after training, the
integral loss, step_batch, the refusals, the backward kernels per (k, stride), and the recipe-sized step."""
import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import MPN_LAYER_CONV
from conftest import rel_err, record_parity
from _train_resnet_ref import fold, resnet_step_oracle, sgd_unfolded, unfolded

pytestmark = pytest.mark.gpu
DEV = "cuda" if torch.cuda.is_available() else "cpu"


def _spec(which="r18", seed=21, integral_k=0, C=5):
    if which == "r18":
        return models.resnet18_fast_rcnn(C, seed=seed, integral_k=integral_k, blocks=(1, 1, 1, 1), fixed_bn=True)
    return models.resnet50_fast_rcnn(C, seed=seed, integral_k=integral_k, blocks=(1, 1, 1, 1), fixed_bn=True)


def _model(ctx, spec, max_rois=64, max_hw=(160, 192)):
    return mpn.Model(ctx, spec, max_rois=max_rois, max_h=max_hw[0], max_w=max_hw[1])


def _batch(spec, sizes=((128, 160), (96, 144)), per_image=(12, 16), seed=0):
    rng = np.random.default_rng(seed)
    ims = [wl.transform(wl.raw_image(h, w, seed + i), spec.transformer) for i, (h, w) in enumerate(sizes)]
    rois = [wl.random_boxes(n, h, w, seed + i).astype(np.float32) for i, ((h, w), n) in enumerate(zip(sizes, per_image))]
    R, C = sum(per_image), spec.num_classes
    labels = rng.integers(1, C + 1, R).astype(np.int32)
    labels[:3] = 1
    tg = np.zeros((R, 4 * C), np.float32)
    for r in range(R):
        if labels[r] > 1:
            tg[r, 4 * labels[r] - 4:4 * labels[r]] = rng.standard_normal(4) * 0.8
    return ims, rois, labels, tg


def _oracle(tr, spec, weights, rois, labels, tg, head=0):
    k0 = spec.trunk_train_from
    slots = {spec.trunk_layers[k0].in_slot} | {L.out_slot for L in spec.trunk_layers[k0:]}
    stored = [{s: tr.trunk_slot(i, s) for s in slots} for i in range(len(rois))]
    gates = {li: tr.relu_gate(0, li) for li, L in enumerate(spec.towers[0].layers) if L.kind == MPN_LAYER_CONV and L.relu}
    return resnet_step_oracle(spec, stored, rois, labels, tg, weights, gates, head=head, dev=DEV)


def _constants(spec):
    """the entries that never train: everything below layer2 and the recorded layers' biases"""
    out = set()
    for L in spec.trunk_layers[:spec.trunk_train_from]:
        out |= {i for i in (L.weight, L.bias) if i >= 0}
    for L in spec.trunk_layers + spec.towers[0].layers:
        if L.weight in spec.fixed_bn:
            out.add(L.bias)
    return out


@pytest.mark.parametrize("which", ["r18", "r50"])
def test_step_losses_and_gradients_vs_fp64(ctx, which):
    spec = _spec(which)
    m = _model(ctx, spec)
    tr = mpn.Trainer(m, seed=7, train_trunk=True)
    assert not (set(tr.trained) & _constants(spec))
    assert set(tr.trained) | _constants(spec) == set(range(len(spec.weights)))
    ims, rois, labels, tg = _batch(spec)
    L = tr.step(ims, rois, labels, tg)
    (rl, rce, rsl), grads = _oracle(tr, spec, spec.weights, rois, labels, tg)
    el = [abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl))]
    assert set(grads) == set(tr.trained)
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    record_parity(f"train_resnet_step_{which}", loss=el[0], cls=el[1], bbox=el[2], grad_max=max(eg.values()))
    assert max(el) < 1e-4, (L, (rl, rce, rsl))
    assert max(eg.values()) < 1e-3, eg
    with pytest.raises(mpn.MpnError):                      # a recorded bias is a constant, not a trained tensor
        tr.gradient(next(iter(_constants(spec) & {L.bias for L in spec.towers[0].layers})))
    tr.close(); m.close()


def test_three_steps_with_momentum_and_decay_vs_fp64_sgd_on_the_unfolded_weights(ctx):
    spec = _spec(seed=5)
    m = _model(ctx, spec)
    lr, mom, wd = 1e-2, 0.9, 5e-4
    tr = mpn.Trainer(m, lr=lr, momentum=mom, weight_decay=wd, seed=3, train_trunk=True)
    ims, rois, labels, tg = _batch(spec, seed=4)
    w = {i: v for i, v in unfolded(spec, spec.weights).items() if i in tr.trained}
    buf = {}
    biases = {L.bias for L in spec.towers[0].layers + spec.trunk_layers} | {h.bias for h in spec.cls_heads} | {spec.bbox_head.bias}
    for k in range(3):
        tr.step(ims, rois, labels, tg)
        cur = fold(spec, w)
        _, grads = _oracle(tr, spec, [cur.get(i, spec.weights[i]) for i in range(len(spec.weights))], rois, labels, tg)
        sgd_unfolded(spec, w, buf, grads, lr, mom, wd, k == 0, biases)
        if k == 0:
            tr.decay(0.5); lr *= 0.5
            for i in buf:
                buf[i] = buf[i] * 0.5
    got, want = tr.weights(), fold(spec, w)
    errs = {i: rel_err(got[i] - spec.weights[i], want[i] - spec.weights[i]) for i in w}
    record_parity("train_resnet_three_steps", delta_max=max(errs.values()))
    assert max(errs.values()) < 1e-3, errs
    for i in _constants(spec):
        assert np.array_equal(got[i], spec.weights[i])
    tr.close(); m.close()


def test_two_trainers_same_bits(ctx):
    spec = _spec(seed=13)
    ims, rois, labels, tg = _batch(spec, seed=6)
    outs = []
    for _ in range(2):
        m = _model(ctx, spec)
        tr = mpn.Trainer(m, seed=99, train_trunk=True)
        ls = [tr.step(ims, rois, labels, tg) for _ in range(2)]
        outs.append((ls, [tr.gradient(i) for i in tr.trained], tr.weights()))
        tr.close(); m.close()
    assert outs[0][0] == outs[1][0]
    for k in (1, 2):
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(outs[0][k], outs[1][k]))


def test_frozen_and_trained_trunk_agree_and_inference_after_training(ctx):
    spec = _spec(seed=31)
    ims, rois, labels, tg = _batch(spec, seed=3)
    res = []
    for trunk in (False, True):
        m = _model(ctx, spec)
        tr = mpn.Trainer(m, seed=4, train_trunk=trunk)
        L = tr.step(ims, rois, labels, tg)
        per_roi = [i for i in tr.trained if all(i != x.weight for x in spec.trunk_layers)]
        res.append((L, tr.outputs(), {i: tr.gradient(i) for i in per_roi}))
        if trunk:
            for _ in range(2):
                tr.step(ims, rois, labels, tg)
            img, H, W = ims[0], ims[0].shape[1], ims[0].shape[2]
            boxes = wl.random_boxes(24, H, W, 11)
            got = m.detect(img, boxes, 1.0)
            ws = tr.weights()
            tr.close(); m.close()
            ref = mpn.Model(ctx, models.ModelSpec(**{**spec.__dict__, "weights": ws}), max_rois=64, max_h=160, max_w=192)
            want = ref.detect(img, boxes, 1.0)
            assert all(np.array_equal(a, b) for a, b in zip(got, want))
            ref.close()
        else:
            tr.close(); m.close()
    (l0, o0, g0), (l1, o1, g1) = res
    assert l0 == l1 and all(np.array_equal(a, b) for a, b in zip(o0, o1))
    assert g0.keys() == g1.keys() and all(np.array_equal(g0[i], g1[i]) for i in g0)


def test_integral_head_step_vs_fp64_and_idle_heads(ctx):
    spec = _spec(seed=17, integral_k=3)
    m = _model(ctx, spec)
    lr, wd = 1e-2, 5e-4
    tr = mpn.Trainer(m, lr=lr, weight_decay=wd, seed=2, train_trunk=True, integral=True)
    ims, rois, labels, tg = _batch(spec, seed=9)
    tr.select_head(1)
    L = tr.step(ims, rois, labels, tg)
    (rl, _, _), grads = _oracle(tr, spec, spec.weights, rois, labels, tg, head=1)
    assert abs(L[0] - rl) / abs(rl) < 1e-4
    for i, g in grads.items():
        assert rel_err(tr.gradient(i), g) < 1e-3, i
    got = tr.weights()
    lib = mpn.load_library()
    for k in (0, 2):
        h = spec.cls_heads[k]
        for i in (h.weight, h.bias):
            assert not np.any(tr.gradient(i))
            w = np.array(spec.weights[i], np.float32).reshape(-1)
            b = np.zeros_like(w)
            assert lib.mpn_debug_sgd(w.ctypes.data, np.zeros_like(w).ctypes.data, b.ctypes.data, w.size, lr, 0.9, 0.0,
                                     wd if i == h.weight else 0.0, 1) == 0
            assert np.array_equal(got[i].reshape(-1), w), (k, i)
    tr.close(); m.close()


def test_step_batch_equals_step_with_the_imagenet_transformer(ctx, oracle_built):
    import _batch_provider_ref as ref
    NCLS, THR, SCALE, MAX_SIZE = 6, [(0.5, 0.1, 0.5)], 160, 192
    gt, props, sizes = ref.synthetic_coco(12, NCLS, 11)
    R = ref.restate_roidb(gt, props, NCLS, THR, best_number=45)
    spec = models.resnet18_fast_rcnn(NCLS + 1, seed=4, integral_k=0, blocks=(1, 1, 1, 1), fixed_bn=True)

    def image(i):
        H, W = sizes[i]
        return np.random.default_rng(100 + i).integers(0, 256, (H, W, 3), dtype=np.uint8)
    db = mpn.RoiDB(ctx, gt, props, NCLS, THR, best_number=45)
    prov = mpn.BatchProviderROI(db, image, spec.transformer, scale=SCALE, max_size=MAX_SIZE, seed=31)
    mean, std = prov.setup_data()
    ma, mb = _model(ctx, spec, 256, (MAX_SIZE, MAX_SIZE)), _model(ctx, spec, 256, (MAX_SIZE, MAX_SIZE))
    ta, tb = mpn.Trainer(ma, seed=9, train_trunk=True), mpn.Trainer(mb, seed=9, train_trunk=True)
    for step in range(2):
        la = ta.step_batch(prov.sample(step))
        P, hw, rb, rl, rt, rpi = ref.sample(R, 31, step, 0, 2, 96, 32, sizes, mean, std, NCLS + 1, SCALE, MAX_SIZE)
        ims = [oracle_built.hd_get_images_u8(np.ascontiguousarray(image(img)[:, ::-1] if flip else image(img)), spec.transformer, *hw[k])
               for k, (img, _, _, flip) in enumerate(P)]
        lb = tb.step(ims, np.split(rb, np.cumsum(rpi)[:-1]), rl, rt)
        assert la == lb, (step, la, lb)
    for i in ta.trained:
        assert np.array_equal(ta._get(i, 0), tb._get(i, 0)) and np.array_equal(ta.gradient(i), tb.gradient(i)), i
    ta.close(); tb.close(); ma.close(); mb.close(); db.close()


def test_refusals_on_the_device(ctx):
    spec = _spec()
    for opt in ("bf16", "fp8"):
        ctx.set_option(opt, 1)
        try:
            m = _model(ctx, spec)
            with pytest.raises(mpn.MpnError, match="bf16"):
                mpn.Trainer(m, train_trunk=True)
            m.close()
        finally:
            ctx.set_option(opt, 0)
    m = _model(ctx, models.resnet50_fast_rcnn(5, seed=1, integral_k=0, blocks=(1, 1, 1, 1)))
    with pytest.raises(mpn.MpnError, match="1x1 convolution"):
        mpn.Trainer(m)
    m.close()


@pytest.mark.parametrize("k,stride", [(1, 1), (1, 2), (3, 1), (3, 2)])
def test_conv_backward_kernels_vs_fp64(ctx, k, stride):
    rng = np.random.default_rng(10 * k + stride)
    cin, cout = 64, 128
    sizes = [(7, 7), (14, 14), (63, 63)]
    q = (k - 1) // 2
    xs = [rng.standard_normal((h, w, cin)).astype(np.float32) for h, w in sizes]
    outs = [((h + 2 * q - k) // stride + 1, (w + 2 * q - k) // stride + 1) for h, w in sizes]
    gs = [rng.standard_normal((ho * wo, cout)).astype(np.float32) for ho, wo in outs]
    w = (rng.standard_normal((cout, cin, k, k)) * np.sqrt(2.0 / (cin * k * k))).astype(np.float32)
    x = np.concatenate([a.reshape(-1, cin) for a in xs])
    hi = (x.view(np.uint32) >> 16).astype(np.uint16)
    lo_f = x - (hi.astype(np.uint32) << 16).view(np.float32)
    lo = (lo_f.view(np.uint32) >> 16).astype(np.uint16)
    xq = (hi.astype(np.uint32) << 16).view(np.float32).astype(np.float64) + (lo.astype(np.uint32) << 16).view(np.float32)
    g = np.concatenate(gs)
    hw = np.array(sizes, np.int32).reshape(-1)
    dw = np.empty_like(w); dx = np.empty_like(x)
    ctx.check(ctx.lib.mpn_debug_conv_backward(ctx.h, len(sizes), hw.ctypes.data_as(mpn._lib._i32p), cin, cout, k, stride, hi.ctypes.data,
                                              lo.ctypes.data, g.ctypes.data, w.ctypes.data, dw.ctypes.data, dx.ctypes.data), "conv_backward")
    W = torch.tensor(w, dtype=torch.float64, requires_grad=True)
    rdw = torch.zeros_like(W)
    rdx, off, go = [], 0, 0
    for (h, wd), (ho, wo) in zip(sizes, outs):
        xi = torch.tensor(xq[off:off + h * wd].reshape(h, wd, cin).transpose(2, 0, 1)[None], requires_grad=True)
        y = torch.nn.functional.conv2d(xi, W, stride=stride, padding=q)
        gi = torch.tensor(g[go:go + ho * wo].reshape(ho, wo, cout).transpose(2, 0, 1)[None], dtype=torch.float64)
        (y * gi).sum().backward()
        rdx.append(xi.grad[0].permute(1, 2, 0).reshape(-1, cin).numpy())
        off += h * wd; go += ho * wo
    rdw = W.grad.numpy()
    ew, ex = rel_err(dw, rdw), rel_err(dx, np.concatenate(rdx))
    record_parity("train_resnet_conv_backward", k=k, stride=stride, dw=ew, dx=ex)
    assert ew < 1e-4 and ex < 1e-4, (ew, ex)


def test_resnet18_inference_vs_oracle(ctx):
    from oracle import graphs as G
    spec = models.resnet18_fast_rcnn(21, seed=5, integral_k=3)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=256, max_w=320)
    img = wl.transform(wl.raw_image(160, 224, 1), spec.transformer)
    boxes = wl.random_boxes(48, 160, 224, 8)
    s, b = m.detect(img, boxes, 1.0)
    rs, rb = G.detect(spec, img, boxes, 1.0)
    assert rel_err(s, rs) < 1e-3 and rel_err(b, rb) < 1e-3
    m.close()


def _recipe(spec, seed=0):
    sizes = [(800, 1000), (800, 1000), (666, 1000), (800, 800)]
    return _batch(spec, sizes=sizes, per_image=(64, 64, 64, 64), seed=seed)


@pytest.mark.parametrize("which", ["r18", "r50"])
def test_recipe_step_finite_and_deterministic(ctx, which):
    spec = (models.resnet18_fast_rcnn(81, integral_k=6, fixed_bn=True) if which == "r18"
            else models.resnet50_fast_rcnn(81, integral_k=6, fixed_bn=True))
    ims, rois, labels, tg = _recipe(spec)
    outs = []
    for _ in range(2):
        m = mpn.Model(ctx, spec, max_rois=256, max_h=1000, max_w=1000)
        tr = mpn.Trainer(m, seed=5, train_trunk=True, integral=True)
        L = tr.step(ims, rois, labels, tg)
        g = [tr.gradient(i) for i in tr.trained[:4] + tr.trained[-4:]]
        outs.append((L, g))
        assert all(np.isfinite(L)) and all(np.all(np.isfinite(x)) for x in g)
        tr.close(); m.close()
    assert outs[0][0] == outs[1][0]
    assert all(np.array_equal(a, b) for a, b in zip(outs[0][1], outs[1][1]))


def test_full_size_one_image_vs_fp64(ctx):
    spec = models.resnet18_fast_rcnn(81, integral_k=6, fixed_bn=True)
    ims, rois, labels, tg = _batch(spec, sizes=((800, 1000),), per_image=(16,), seed=2)
    m = mpn.Model(ctx, spec, max_rois=64, max_h=1000, max_w=1000)
    tr = mpn.Trainer(m, seed=5, train_trunk=True, integral=True)
    L = tr.step(ims, rois, labels, tg)
    (rl, _, _), grads = _oracle(tr, spec, spec.weights, rois, labels, tg)
    assert abs(L[0] - rl) / abs(rl) < 1e-4
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    record_parity("train_resnet_full_size", grad_max=max(eg.values()))
    assert max(eg.values()) < 1e-3, eg
    tr.close(); m.close()

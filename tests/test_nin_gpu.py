"""GPU: Network-in-Network Fast R-CNN (models.nin_fast_rcnn, models/nin.lua) and the engine features it needs.

  * the K tail: convolutions and GEMMs whose Cin is a multiple of 8 but not of 64 (the last K block of each tap is the
    TMA's zero fill on A and the zero pad of the [Cout][kh][kw][conv_k_pad(Cin)] weight layout on B), and 5 x 5 kernels,
    against fp64 at the engine tests' bars: BF16X3 1e-4 normwise (test_engine_gpu.py), BF16X1 1e-5 against the fp64
    product of the bf16-rounded operands, + 2^-17 for the split-plane store (test_bf16_gpu.py);
  * a view whose channels between C and ld hold NaN: the output is finite and bit-identical to the dense input's;
  * every layer of the graph against fp64 on its own device inputs (test_layers_gpu.py's walk, tests/_layer_ref.py), in
    the default and the bf16 numerics (fp8 refuses the tailed layers);
  * detect at 600 x 1000 with 1000 ROIs against the CPU oracle, NMS keep lists bit-exact against nms.c, Tester.testOne;
  * per-ROI training with fixed batch norm (block 4 and the heads) against fp64 autograd on the unfolded graph, three
    SGD steps, determinism, inference after training, integral / bf16."""
import types

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import MPN_LAYER_CONV
from oracle import graphs as G
from conftest import rel_err, record_parity
from test_model_gpu import _inputs, assert_nms_every_class
import _bf16_oracle as B
import test_layers_gpu as TL
from _train_resnet_ref import fold, resnet_step_oracle, sgd_unfolded, unfolded

pytestmark = pytest.mark.gpu
TOL = 1e-4
TOL_BF16 = 1e-5
SPLIT = 2.0 ** -17
DEV = "cuda" if torch.cuda.is_available() else "cpu"
TAILS = (8, 24, 96, 136, 200)


def _bf16(ctx, on):
    ctx.set_option("bf16", 1 if on else -1)


def _rn(a):
    return B.rn_bf16(torch.from_numpy(np.ascontiguousarray(a, np.float32))).double()


# ---------------------------------------------------------------- 1. engine: K tail and 5 x 5
@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("k", [1, 3, 5])
@pytest.mark.parametrize("cin", TAILS)
def test_conv_tail(ctx, cin, k, stride):
    rng = np.random.default_rng(cin * 10 + k + stride)
    N, H, W, Cout, pad = 2, 19, 23, 72, (k - 1) // 2
    x = rng.standard_normal((N, cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, cin, k, k)) / np.sqrt(cin * k * k)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    ref = F.relu(F.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(), stride=stride,
                          padding=pad)).numpy()
    got0 = ctx.conv_check(x, w, b, stride=stride, pad=pad, relu=True, impl=0)
    got1 = ctx.conv_check(x, w, b, stride=stride, pad=pad, relu=True, impl=1)
    e0, e1 = rel_err(got0, ref), rel_err(got1, ref)
    try:
        _bf16(ctx, True)
        h0 = ctx.conv_check(x, w, b, stride=stride, pad=pad, relu=True, impl=0)
    finally:
        _bf16(ctx, False)
    refb = F.relu(F.conv2d(_rn(x), _rn(w), torch.from_numpy(b).double(), stride=stride, padding=pad)).numpy()
    eb = rel_err(h0, refb)
    record_parity("nin_conv_tail", cin=cin, k=k, stride=stride, bf16x3=e0, check=e1, bf16x1=eb)
    assert e0 < TOL and e1 < TOL and eb <= TOL_BF16 + SPLIT, (e0, e1, eb)


@pytest.mark.parametrize("cin", TAILS)
def test_gemm_tail(ctx, cin):
    rng = np.random.default_rng(cin)
    M, N = 300, 84
    A = rng.standard_normal((M, cin)).astype(np.float32)
    Bm = (rng.standard_normal((N, cin)) / np.sqrt(cin)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    got = ctx.gemm_check(A, Bm, bias, relu=True, impl=0)
    ref = torch.relu(torch.from_numpy(A).double() @ torch.from_numpy(Bm).double().t() + torch.from_numpy(bias).double()).numpy()
    try:
        _bf16(ctx, True)
        gb = ctx.gemm_check(A, Bm, bias, relu=True, impl=0)
    finally:
        _bf16(ctx, False)
    refb = torch.relu(_rn(A) @ _rn(Bm).t() + torch.from_numpy(bias).double()).numpy()
    e, eb = rel_err(got, ref), rel_err(gb, refb)
    record_parity("nin_gemm_tail", cin=cin, bf16x3=e, bf16x1=eb)
    assert e < TOL and eb <= TOL_BF16, (e, eb)


@pytest.mark.parametrize("cin,ld,k,stride", [(24, 32, 3, 1), (96, 128, 1, 1), (96, 104, 5, 1), (200, 256, 3, 2), (8, 64, 5, 2)])
def test_nan_beyond_the_view_is_never_read(ctx, cin, ld, k, stride):
    rng = np.random.default_rng(ld + k)
    x = rng.standard_normal((1, cin, 17, 21)).astype(np.float32)
    w = (rng.standard_normal((64, cin, k, k)) / np.sqrt(cin * k * k)).astype(np.float32)
    b = rng.standard_normal(64).astype(np.float32)
    pad = (k - 1) // 2
    for impl in (0, 1):
        dense = ctx.conv_check(x, w, b, stride=stride, pad=pad, relu=False, impl=impl)
        view = ctx.conv_check_view(x, w, ld, b, stride=stride, pad=pad, relu=False, impl=impl)
        assert np.isfinite(view).all() and np.array_equal(view.view(np.uint32), dense.view(np.uint32)), impl


def test_fp8_refuses_a_tail(ctx):
    x = np.ones((1, 96, 8, 8), np.float32)
    w = np.ones((64, 96, 1, 1), np.float32)
    try:
        ctx.set_option("fp8", 1)
        with pytest.raises(mpn.MpnError, match="fp8"):
            ctx.conv_check(x, w)
        spec = models.nin_fast_rcnn(21, seed=1)
        m = mpn.Model(ctx, spec, max_rois=64, max_h=160, max_w=192)
        img, boxes = _inputs(spec, 160, 192, 16, 1)
        with pytest.raises(mpn.MpnError, match="96 input channels, not a multiple of 64"):
            m.detect(img, boxes, 1.0)
        m.close()
    finally:
        ctx.set_option("fp8", -1)


# ---------------------------------------------------------------- 2. every layer against fp64 on its own inputs
@pytest.mark.parametrize("numerics", ["default", "bf16"])
def test_every_layer_of_nin(ctx, numerics):
    spec = models.nin_fast_rcnn(21, seed=5)
    H, W, R, seed = 224, 288, 200, 3
    img, boxes = _inputs(spec, H, W, R, seed, sharp=True)
    rng = np.random.default_rng(seed)
    walk = TL.Walk("nin", numerics)
    with TL.options(ctx, TL.NUMERICS[numerics]):
        m = mpn.Model(ctx, spec, max_rois=256, max_h=224, max_w=288)
        try:
            m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3, want_raw=False)
            TL.walk_trunk(walk, m, spec, img, numerics, False, rng)
            rows, outs, _, _ = TL.walk_towers(walk, m, spec, numerics, R, False, rng)
            TL.walk_heads(walk, m, spec, numerics, rows, outs)
        finally:
            m.close()
    assert len(walk.worst) >= 11 + 4, sorted(walk.worst)           # 11 trunk layers, 4 tower layers, the heads
    worst = max(((v[0], k) for k, v in walk.worst.items() if isinstance(v, tuple)), default=(0.0, ""))
    record_parity("layer_worst", graph="nin", numerics=numerics, layer=worst[1], error=worst[0])
    assert not walk.fails, "\n".join(walk.fails)


# ---------------------------------------------------------------- 3. detect at full size
def test_detect_full_size_vs_oracle_and_nms(ctx):
    spec = models.nin_fast_rcnn(21, seed=1234)
    m = mpn.Model(ctx, spec, max_rois=1048, max_h=608, max_w=1000)
    img, boxes = _inputs(spec, 600, 1000, 1000, 5, sharp=True)
    scores, bboxes, keeps = m.detect_nms(img, boxes, 1.0, 1000, 600, -1.5, 0.3)
    rs, rb, _ = G.test_one(spec, img, boxes, 1.0, 1000, 600, nms_fn=lambda sb, thr: np.zeros(0, np.int64))
    es, eb = rel_err(scores, rs), rel_err(bboxes, rb)
    record_parity("nin_full_size", scores=es, boxes=eb)
    assert es < 1e-3 and eb < 1e-3, (es, eb)
    assert_nms_every_class(scores, bboxes, keeps)
    tf, hf = m.last_flops()
    assert abs(tf - models.trunk_flops(spec, 600, 1000)) < 1e-6 * tf
    assert abs(hf / 1000 - models.head_flops_per_roi(spec)) < 1e-6 * hf
    m.close()


def test_tester_test_one(ctx):
    spec = models.nin_fast_rcnn(21, seed=9)
    m = mpn.Model(ctx, spec, max_rois=256, max_h=320, max_w=400)
    raw = wl.raw_image(180, 240, 4)
    boxes = wl.random_boxes(120, 180, 240, 4)
    t = mpn.Tester(m, mpn.modules.ImageTransformer(spec.transformer), scale=[180], max_size=400)
    img_boxes = t.testOne(raw, boxes)
    assert len(img_boxes) == spec.num_classes - 1 and all(b.shape[1] == 5 for b in img_boxes)
    det = mpn.ImageDetect(m, mpn.modules.ImageTransformer(spec.transformer), [180], 400)
    s, b = det.detect(raw, boxes)
    rs, rb = G.detect(spec, wl.transform(raw, spec.transformer), boxes, 1.0)
    assert rel_err(s, rs) < 1e-3 and rel_err(b, rb) < 1e-3
    m.close()


# ---------------------------------------------------------------- 4. per-ROI training with fixed batch norm
def _spec(seed=21, integral_k=0, C=5):
    return models.nin_fast_rcnn(C, seed=seed, fixed_bn=True, integral_k=integral_k)


def _model(ctx, spec):
    return mpn.Model(ctx, spec, max_rois=64, max_h=160, max_w=192)


def _batch(spec, seed=0, sizes=((128, 160), (96, 144)), per_image=(12, 16)):
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


def _stored(ctx, spec, ims):
    """per image the device's trunk slots around the last trunk layer (its input and the pooled map), read after an
    inference trunk pass: the frozen trunk's forward is the same in a training step"""
    last = spec.trunk_layers[-1]
    m = _model(ctx, spec)
    out = []
    for im in ims:
        m.trunk(im)
        out.append({s: m.trunk_slot(s)[0] for s in (last.in_slot, last.out_slot)})
    m.close()
    return out


def _oracle(ctx, tr, spec, weights, ims, rois, labels, tg, head=0):
    """resnet_step_oracle with the trunk's last layer recomputed in fp64 from its stored input (the pooled map's
    gradient is not needed: the trunk is frozen); its parameters' gradients are dropped"""
    view = types.SimpleNamespace(**{**spec.__dict__, "trunk_train_from": len(spec.trunk_layers) - 1})
    gates = {li: tr.relu_gate(0, li) for li, L in enumerate(spec.towers[0].layers) if L.kind == MPN_LAYER_CONV and L.relu}
    losses, grads = resnet_step_oracle(view, _stored(ctx, spec, ims), rois, labels, tg, weights, gates, head=head, dev=DEV)
    return losses, {i: g for i, g in grads.items() if i in tr.trained}


def test_step_losses_and_gradients_vs_fp64(ctx):
    spec = _spec()
    m = _model(ctx, spec)
    tr = mpn.Trainer(m, seed=7)
    tower = {i for L in spec.towers[0].layers for i in (L.weight, L.bias) if i >= 0 and L.weight >= 0}
    heads = {i for h in spec.cls_heads + [spec.bbox_head] for i in (h.weight, h.bias)}
    recorded_biases = {L.bias for L in spec.towers[0].layers if L.weight in spec.fixed_bn}
    assert set(tr.trained) == (tower | heads) - recorded_biases
    ims, rois, labels, tg = _batch(spec)
    L = tr.step(ims, rois, labels, tg)
    (rl, rce, rsl), grads = _oracle(ctx, tr, spec, spec.weights, ims, rois, labels, tg)
    el = [abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl))]
    assert set(grads) == set(tr.trained)
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    record_parity("nin_train_step", loss=el[0], cls=el[1], bbox=el[2], grad_max=max(eg.values()))
    assert max(el) < 1e-4, (L, (rl, rce, rsl))
    assert max(eg.values()) < 1e-3, eg
    tr.close(); m.close()


def test_three_steps_with_momentum_and_decay(ctx):
    spec = _spec(seed=5)
    m = _model(ctx, spec)
    lr, mom, wd = 1e-2, 0.9, 5e-4
    tr = mpn.Trainer(m, lr=lr, momentum=mom, weight_decay=wd, seed=3)
    ims, rois, labels, tg = _batch(spec, seed=4)
    w = {i: v for i, v in unfolded(spec, spec.weights).items() if i in tr.trained}
    buf = {}
    biases = {L.bias for L in spec.towers[0].layers + spec.trunk_layers} | {h.bias for h in spec.cls_heads} | {spec.bbox_head.bias}
    for k in range(3):
        tr.step(ims, rois, labels, tg)
        cur = fold(spec, w)
        _, grads = _oracle(ctx, tr, spec, [cur.get(i, spec.weights[i]) for i in range(len(spec.weights))], ims, rois, labels, tg)
        sgd_unfolded(spec, w, buf, grads, lr, mom, wd, k == 0, biases)
        if k == 0:
            tr.decay(0.5); lr *= 0.5
            for i in buf:
                buf[i] = buf[i] * 0.5
    got, want = tr.weights(), fold(spec, w)
    errs = {i: rel_err(got[i] - spec.weights[i], want[i] - spec.weights[i]) for i in w}
    record_parity("nin_train_three_steps", delta_max=max(errs.values()))
    assert max(errs.values()) < 1e-3, errs
    for i in set(range(len(spec.weights))) - set(tr.trained):
        assert np.array_equal(got[i], spec.weights[i])
    tr.close(); m.close()


@pytest.mark.parametrize("mode", ["default", "bf16", "integral"])
def test_deterministic_and_inference_after_training(ctx, mode):
    spec = _spec(seed=13, integral_k=2 if mode == "integral" else 0)
    ims, rois, labels, tg = _batch(spec, seed=6)
    outs = []
    for rep in range(2):
        m = _model(ctx, spec)
        tr = mpn.Trainer(m, seed=99, bf16=mode == "bf16", integral=mode == "integral")
        ls = [tr.step(ims, rois, labels, tg) for _ in range(2)]
        assert all(np.isfinite(x).all() for x in ls)
        outs.append((ls, [tr.gradient(i) for i in tr.trained], tr.weights()))
        if rep == 1:
            img = ims[0]
            boxes = wl.random_boxes(24, img.shape[1], img.shape[2], 11)
            got = m.detect(img, boxes, 1.0)
            ws = tr.weights()
            tr.close(); m.close()
            ref = _model(ctx, models.ModelSpec(**{**spec.__dict__, "weights": ws}))
            want = ref.detect(img, boxes, 1.0)
            assert all(np.array_equal(a, b) for a, b in zip(got, want))
            ref.close()
        else:
            tr.close(); m.close()
    assert outs[0][0] == outs[1][0]
    for k in (1, 2):
        assert all(np.array_equal(a.view(np.uint32), b.view(np.uint32)) for a, b in zip(outs[0][k], outs[1][k]))


def test_training_refusals(ctx):
    spec = _spec()
    m = _model(ctx, spec)
    with pytest.raises(mpn.MpnError, match="fixed-batch-norm layer"):      # block 2's 5x5: trunk training is out of scope
        mpn.Trainer(m, train_trunk=True)
    m.close()
    # a trained layer with a K tail: the nin.lua graph at tiny widths, whose block 4 reads 48 channels
    from multipathnet_b200 import t7
    from test_nin_cpu import _tiny_nin
    tiny = t7.model_from_t7(_tiny_nin(np.random.default_rng(17)), transformer="imagenet")
    m = mpn.Model(ctx, tiny, max_rois=64, max_h=160, max_w=192)
    with pytest.raises(mpn.MpnError, match="multiple of 64 input channels"):
        mpn.Trainer(m)
    img, boxes = _inputs(tiny, 96, 128, 8, 2)
    assert np.isfinite(m.detect(img, boxes, 1.0)[0]).all()             # the refused model still runs inference
    m.close()


# ---------------------------------------------------------------- 5. a Linear over a FLATTENed map off the 64 grid
def _flat_spec(c, P, seed=3, C=5, trunk_tail=True):
    """trunk 3 -> 64 (direct), 1x1 64 -> c, 1x1 c -> c (a K tail when c % 64 != 0; left out without trunk_tail), 2x2 / 2
    pool; one tower
    ROIPooling(P, P, 1/2) -> FLATTEN -> Linear(c * P * P -> 256) -> Linear(256 -> 256), heads: the ROIPooling -> View ->
    Linear graph of an imported Fast R-CNN. The Linear's K = c * P * P is the flat (h, w, c) vector, padded at its end."""
    from multipathnet_b200._lib import Head, Layer, ModelSpec, Tower, MPN_LAYER_FLATTEN, MPN_LAYER_MAXPOOL
    W = models._W(seed)
    w0, b0 = W.conv(64, 3, 3, 3, gain=1.0 / 64)
    w1, b1 = W.conv(c, 64, 1, 1)
    w2, b2 = W.conv(c, c, 1, 1)
    trunk = [Layer(MPN_LAYER_CONV, 0, 1, cin=3, cout=64, kh=3, kw=3, pad=1, relu=1, weight=w0, bias=b0),
             Layer(MPN_LAYER_CONV, 1, 2, cin=64, cout=c, relu=1, weight=w1, bias=b1),
             Layer(MPN_LAYER_CONV, 2, 3, cin=c, cout=c, relu=1, weight=w2, bias=b2),
             Layer(MPN_LAYER_MAXPOOL, 3, 4, kh=2, kw=2, stride=2, ceil_mode=1)]
    if not trunk_tail:
        trunk = trunk[:2] + [Layer(MPN_LAYER_MAXPOOL, 2, 4, kh=2, kw=2, stride=2, ceil_mode=1)]
    w6, b6 = W.linear(256, c * P * P)
    w7, b7 = W.linear(256, 256)
    tl = [Layer(MPN_LAYER_FLATTEN, 0, 1), Layer(MPN_LAYER_CONV, 1, 2, cin=c * P * P, cout=256, relu=1, weight=w6, bias=b6),
          Layer(MPN_LAYER_CONV, 2, 3, cin=256, cout=256, relu=1, weight=w7, bias=b7)]
    wc, bc = W.linear(C, 256, std=0.01, zero_bias=True)
    wb, bb = W.linear(4 * C, 256, std=0.001, zero_bias=True)
    return ModelSpec(name=f"flat_{c}_{P}", trunk_layers=trunk, towers=[Tower(region=0, levels=[(4, 0.5)], pooled_w=P, pooled_h=P,
                     normalize=0, layers=tl, out_slot=3)], cls_heads=[Head(0, 256, C, wc, bc)], bbox_head=Head(0, 256, 4 * C, wb, bb),
                     num_classes=C, weights=W.arrays, transformer="ross", taps={"top": 4})


@pytest.mark.parametrize("c,P", [(32, 7), (24, 7), (32, 8), (64, 7)])
def test_linear_after_flatten_off_the_64_grid(ctx, c, P):
    """K = c * P * P: 1568 and 1176 end in a tail, 2048 and 3136 do not (the dense layout as before). Imported through
    the .t7 writer and reader, as a graph of ROIPooling -> View -> Linear arrives."""
    from multipathnet_b200 import t7
    spec = t7.model_from_t7(t7.model_to_t7(_flat_spec(c, P)), transformer="ross")
    assert any(L.kind == 4 for L in spec.towers[0].layers)
    img, boxes = _inputs(spec, 96, 128, 40, 7)
    m = mpn.Model(ctx, spec, max_rois=64, max_h=96, max_w=128)
    s, b = m.detect(img, boxes, 1.0)
    rs, rb = G.detect(spec, img, boxes, 1.0)
    es, eb = rel_err(s, rs), rel_err(b, rb)
    record_parity("flat_linear", c=c, P=P, scores=es, boxes=eb)
    assert es < 1e-3 and eb < 1e-3, (es, eb)
    m.close()
    if c * P * P % 64:                                          # the backward GEMMs take no K tail
        m = mpn.Model(ctx, spec, max_rois=64, max_h=96, max_w=128)
        with pytest.raises(mpn.MpnError, match="multiple of 64 input channels"):
            mpn.Trainer(m)
        m.close()


def test_fp8_linear_after_flatten_with_a_dense_k(ctx):
    """fp8 on a flat Linear whose 32 channels are off the 64 grid but whose K = 32 * 8 * 8 is not: its e4m3 plane is
    quantised from the dense rows, checked against the fp8-operand oracle as test_fp8_gpu.py checks its graphs. A K off
    the grid (32 * 7 * 7) is refused by name."""
    from test_fp8_gpu import _graph_check
    spec = _flat_spec(32, 8, trunk_tail=False)
    img, boxes = _inputs(spec, 96, 128, 40, 7)
    try:
        ctx.set_option("fp8", 1)
        m = mpn.Model(ctx, spec, max_rois=64, max_h=96, max_w=128)
        scores, bboxes, _ = m.detect_nms(img, boxes, 1.0, 128, 96, -1.5, 0.3)
        m.close()
        m = mpn.Model(ctx, _flat_spec(32, 7, trunk_tail=False), max_rois=64, max_h=96, max_w=128)
        with pytest.raises(mpn.MpnError, match="1568 input channels, not a multiple of 64"):
            m.detect(img, boxes, 1.0)
        m.close()
    finally:
        ctx.set_option("fp8", -1)
    _graph_check("flat_linear_fp8", (scores, bboxes), spec, img, boxes, 128, 96)

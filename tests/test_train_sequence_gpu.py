"""GPU: one live Model + Trainer through a run of minibatches that differ in every step, as train.lua draws them: the
image count (1, 2, 3), each image's size (largest first, smallest first, a portrait image), the ROIs per image and the
total R, which goes below 64, to exactly 64, to max_rois and to a value off the 64 grid right after a step with a larger
ceil64(R), the row stride of the dW operands; one trunk-training step has an image without ROIs. Per step k:
  1. a fresh Model + Trainer of the same arguments, loaded with the state_dict from before step k and run on step k's
     batch, equals the long-lived trainer bit for bit: losses, gradients, masters, optim state, dropout masks, ReLU
     gates and the trainer state;
  2. the losses within 1e-4 relative and every gradient within 1e-3 normwise of the setup's fp64 oracle at the device's
     weights before step k (bf16: the bars of DESIGN 4 against the bf16-operand oracle; adam: every master and state bit
     for bit against the numpy restatement of csrc/train_rule.cuh);
after the last step, detect_nms on the live model at a size training never used equals a model built from weights()."""
import dataclasses
import types

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import MPN_LAYER_CONV
from multipathnet_b200.train import _train_optim
from conftest import rel_err, record_parity
from _train_bf16_ref import three_oracles
from _train_phase2_ref import phase2_step_oracle
from _train_resnet_ref import resnet_step_oracle
from _train_trunk_ref import trunk_step_oracle
from test_shape_sequence_gpu import _assert_same
from test_train_bf16_gpu import _check as bf16_check
from test_train_optim_gpu import _check_step as optim_check, _snapshot

pytestmark = pytest.mark.gpu
DEV = "cuda" if torch.cuda.is_available() else "cpu"
LIMITS = dict(max_rois=160, max_h=192, max_w=256)

# per step: [(H, W, ROIs) per image]
BATCHES = [
    [(176, 240, 100), (128, 160, 60)],                   # R = 160 = max_rois, largest image first
    [(96, 128, 20), (160, 208, 0), (128, 176, 10)],       # R = 30 < 64, smallest first, an image without ROIs
    [(192, 144, 64)],                                     # R = 64, one portrait image
    [(144, 192, 70), (112, 160, 59)],                     # R = 129: ceil64 = 192
    [(128, 176, 40), (160, 224, 43)],                     # R = 83 after a larger ceil64(R)
]


def _spec_vgg(seed=21):
    return models.vgg16_fast_rcnn(21, seed=seed, width_div=4, fc_dim=256)


def _spec_mpn(seed=21):
    return models.vgg16_multipathnet(21, seed=seed, width_div=4, fc_dim=256, integral_k=2)


def _spec_r18(seed=21):
    return models.resnet18_fast_rcnn(5, seed=seed, integral_k=2, blocks=(1, 1, 1, 1), fixed_bn=True)


def _spec_nin(seed=21):
    return models.nin_fast_rcnn(5, seed=seed, fixed_bn=True)


SGD = dict(lr=1e-2, momentum=0.9, weight_decay=5e-4)
# name -> (spec, Trainer arguments, per step (head, phase-2 switch before it, decay before it), trains the trunk)
SETUPS = {
    "a_vgg_trunk": (_spec_vgg, dict(SGD, seed=3, train_trunk=True), [(0, False, k == 2) for k in range(5)]),
    "b_mpn_phase2_integral": (_spec_mpn, dict(SGD, seed=5, phase2=True, integral=True),
                              [(k % 2, k == 2, False) for k in range(5)]),
    "c_r18_integral": (_spec_r18, dict(SGD, seed=7, train_trunk=True, integral=True), [(k % 2, False, False) for k in range(5)]),
    "d_nin": (_spec_nin, dict(SGD, seed=9), [(0, False, False) for k in range(5)]),
    "e_vgg_trunk_bf16": (_spec_vgg, dict(SGD, seed=3, train_trunk=True, bf16=True), [(0, False, k == 2) for k in range(5)]),
    "f_r18_adam": (_spec_r18, dict(lr=1e-3, seed=7, train_trunk=True, integral=True, method="adam"),
                   [(k % 2, False, False) for k in range(5)]),
}


def batch(spec, k, script=BATCHES, seed=100):
    sizes = script[k]
    rng = np.random.default_rng(seed + k)
    ims = [wl.transform(wl.raw_image(h, w, seed + 10 * k + i), spec.transformer) for i, (h, w, _) in enumerate(sizes)]
    rois = []
    for i, (h, w, n) in enumerate(sizes):
        r = wl.random_boxes(n, h, w, seed + 10 * k + i).astype(np.float32).reshape(n, 4)
        if len(spec.towers) > 1 and n >= 2:
            r[0] = (1, 1, w, h)                                  # MultiPathNet's x4 region leaves the image
            r[1] = (w / 4, h / 4, 3 * w / 4, 3 * h / 4)
        rois.append(r)
    R, C = sum(n for _, _, n in sizes), spec.num_classes
    labels = rng.integers(1, C + 1, R).astype(np.int32)
    labels[:3] = 1
    tg = np.zeros((R, 4 * C), np.float32)
    for r in range(R):
        if labels[r] > 1:
            tg[r, 4 * labels[r] - 4:4 * labels[r]] = rng.standard_normal(4) * 0.8
    return ims, rois, labels, tg


def _gates(tr, spec, per_tower=False):
    return {((t, li) if per_tower else li): tr.relu_gate(t, li) for t, T in enumerate(spec.towers)
            for li, L in enumerate(T.layers) if L.kind == MPN_LAYER_CONV and L.relu}


def _stored(tr, spec, k0, n):
    slots = {spec.trunk_layers[k0].in_slot} | {L.out_slot for L in spec.trunk_layers[k0:]}
    return [{s: tr.trunk_slot(i, s) for s in slots} for i in range(n)]


def _frozen_stored(ctx, spec, weights, ims, k0):
    """the slots from layer k0's input up, from an inference trunk call at `weights` (a frozen trunk's forward is a
    training step's)"""
    m = mpn.Model(ctx, dataclasses.replace(spec, weights=list(weights)), **LIMITS)
    slots = {spec.trunk_layers[k0].in_slot} | {L.out_slot for L in spec.trunk_layers[k0:]}
    out = []
    for im in ims:
        m.trunk(im)
        out.append({s: m.trunk_slot(s)[0] for s in slots})
    m.close()
    return out


def oracle(name, ctx, tr, spec, w, ims, rois, labels, tg):
    """fp64 (losses, {weight index: gradient}) of the step just made, at the weights w it started from"""
    head = tr.head
    if name.startswith(("a_", "e_")):
        return trunk_step_oracle(spec, spec.trunk_train_from, _stored(tr, spec, spec.trunk_train_from, len(ims)), rois, labels, tg,
                                 w, {(0, li): g for li, g in _gates(tr, spec).items()}, 0.5, dev=DEV)
    if name.startswith("b_"):
        k0 = spec.phase2_from
        stored = _stored(tr, spec, k0, len(ims)) if tr.phase == 2 else _frozen_stored(ctx, spec, w, ims, k0)
        losses, grads = phase2_step_oracle(spec, k0, stored, rois, labels, tg, w, _gates(tr, spec, True), 0.5, head=head, dev=DEV)
        return losses, {i: g for i, g in grads.items() if i in tr.trained}
    if name.startswith(("c_", "f_")):
        return resnet_step_oracle(spec, _stored(tr, spec, spec.trunk_train_from, len(ims)), rois, labels, tg, w, _gates(tr, spec),
                                  head=head, dev=DEV)
    # NIN: per-ROI training; the oracle recomputes the trunk's last layer in fp64 from its stored input
    last = len(spec.trunk_layers) - 1
    view = types.SimpleNamespace(**{**spec.__dict__, "trunk_train_from": last})
    losses, grads = resnet_step_oracle(view, _frozen_stored(ctx, spec, w, ims, last), rois, labels, tg, w, _gates(tr, spec),
                                       head=head, dev=DEV)
    return losses, {i: g for i, g in grads.items() if i in tr.trained}


def _everything(tr, spec):
    """what a step leaves behind, in a comparable form"""
    out = {"state": tr.state_dict()["state"]}
    for i in tr.trained:
        out[f"grad {i}"] = tr.gradient(i)
        out[f"master {i}"] = tr._get(i, 0)
        out[f"optim {i}"] = tr.optim_state(i)
    for t, T in enumerate(spec.towers):
        for li, L in enumerate(T.layers):
            if L.kind == MPN_LAYER_CONV:
                out[f"dropout {t}.{li}"] = tr.dropout_mask(t, li)
                if L.relu:
                    out[f"gate {t}.{li}"] = tr.relu_gate(t, li)
    out["outputs"] = tr.outputs()
    return out


def _compare(a, b, what):
    assert a.keys() == b.keys(), what
    assert a["state"] == b["state"], (what, a["state"], b["state"])
    for k in a:
        if k != "state":
            _assert_same(a[k], b[k], f"{what}: {k}")


def _fp64_check(name, k, L, ref, tr, spec, worst):
    (rl, rce, rsl), grads = ref
    el = [abs(a - b) / abs(b) for a, b in zip(L, (rl, rce, rsl))]
    assert set(grads) <= set(tr.trained), name
    for i in set(tr.trained) - set(grads):                 # the idle class heads
        assert not np.any(tr.gradient(i)), (name, k, i)
    eg = {i: rel_err(tr.gradient(i), g) for i, g in grads.items()}
    record_parity("train_sequence", setup=name, step=k, loss=max(el), grad_max=max(eg.values()))
    worst[0] = max(worst[0], max(el)); worst[1] = max(worst[1], max(eg.values()))
    assert max(el) < 1e-4, (name, k, L, (rl, rce, rsl))
    assert max(eg.values()) < 1e-3, (name, k, {i: e for i, e in eg.items() if e >= 1e-3})


@pytest.mark.parametrize("name", list(SETUPS))
def test_one_trainer_through_changing_batches(ctx, name):
    make, kw, plan = SETUPS[name]
    spec = make()
    m = mpn.Model(ctx, spec, **LIMITS)
    tr = mpn.Trainer(m, **kw)
    worst = [0.0, 0.0]
    try:
        for k, (head, switch, decay) in enumerate(plan):
            if switch:
                tr.set_phase2(4e-3)
            if decay:
                tr.decay(0.5)
            if len(spec.cls_heads) > 1:
                tr.select_head(head)
            ims, rois, labels, tg = batch(spec, k)
            sd, w = tr.state_dict(), tr.weights()
            before = _snapshot(tr)
            L = tr.step(ims, rois, labels, tg)
            # 1. a fresh trainer from the state before step k
            f = mpn.Model(ctx, spec, **LIMITS)
            ft = mpn.Trainer(f, **kw)
            try:
                ft.load_state_dict(sd)
                assert ft.step(ims, rois, labels, tg) == L, (name, k)
                _compare(_everything(tr, spec), _everything(ft, spec), f"{name} step {k}")
            finally:
                ft.close(); f.close()
            # 2. fp64
            if name.startswith("e_"):
                plain, b64, b32 = three_oracles(lambda: oracle(name, ctx, tr, spec, w, ims, rois, labels, tg))
                bf16_check(f"train_sequence_{name}", L, {i: tr.gradient(i) for i in b64[1]}, plain, b64, b32)
            else:
                _fp64_check(name, k, L, oracle(name, ctx, tr, spec, w, ims, rois, labels, tg), tr, spec, worst)
            if name.startswith("f_"):
                idle = {i for j, h in enumerate(spec.cls_heads) if j != tr.head for i in (h.weight, h.bias) if i >= 0}
                fixed = {i: a for i, a in spec.fixed_bn.items() if i in tr.trained}
                optim_check(tr, _train_optim("adam"), before, k, tr.cfg.lr, fixed=fixed, idle=idle)
        # 3. inference on the live model at a size training never used
        H, W = 150, 203
        img = wl.transform(wl.raw_image(H, W, 77), spec.transformer)
        boxes = wl.random_boxes(100, H, W, 77)
        got = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        ref = mpn.Model(ctx, models.ModelSpec(**{**spec.__dict__, "weights": tr.weights()}), **LIMITS)
        _assert_same(got, ref.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3), f"{name}: inference after training")
        ref.close()
        record_parity("train_sequence_worst", setup=name, loss=worst[0], grad_max=worst[1])
    finally:
        tr.close(); m.close()


FULL_BATCHES = [[(600, 1000, 128), (600, 800, 128)], [(1000, 600, 64)], [(600, 667, 128), (600, 1000, 128)]]


def test_full_size_vgg_trunk_over_coco_shaped_pairs(ctx):
    """setup (a) on the full VGG-16 Fast R-CNN over COCO-shaped pairs: each step bit for bit against a fresh trainer"""
    spec = models.vgg16_fast_rcnn(21, seed=1234)
    lim = dict(max_rois=256, max_h=1000, max_w=1000)
    kw = dict(SGD, seed=3, train_trunk=True)
    m = mpn.Model(ctx, spec, **lim)
    tr = mpn.Trainer(m, **kw)
    try:
        for k in range(len(FULL_BATCHES)):
            ims, rois, labels, tg = batch(spec, k, FULL_BATCHES, seed=200)
            sd = tr.state_dict()
            L = tr.step(ims, rois, labels, tg)
            f = mpn.Model(ctx, spec, **lim)
            ft = mpn.Trainer(f, **kw)
            try:
                ft.load_state_dict(sd)
                assert ft.step(ims, rois, labels, tg) == L, k
                _compare(_everything(tr, spec), _everything(ft, spec), f"full size step {k}")
            finally:
                ft.close(); f.close()
    finally:
        tr.close(); m.close()

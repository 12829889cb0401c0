"""GPU: data-parallel training over K model replicas (Trainer(replicas=...), train.lua's train_nGPU). Unless a test says
otherwise the replicas share device 0, each on a context with a stream of its own, so the whole path (the shards, the
peer copies of the reduction, the scatter of a sampled batch) runs on one GPU.
  - K = 1 through the replica entry is the single trainer bit for bit;
  - two and four replicas against one trainer loaded with the same state before every step, on five setups: every row's
    logits, deltas and dropout masks bit for bit, losses within 1e-6, the summed gradients within the fp32-reordering bar
    of DESIGN 4, and within the fp64 bars (losses 1e-4, gradients 1e-3) except in bf16; the three-step weight delta
    against the sum of the single trainer's steps within its bar; after every step every replica's masters and states
    bit for bit, and a detect on every replica at the end;
  - replicas on devices 0 and 1 give the bits of replicas on device 0 (skipped with one GPU);
  - step_batch on sampled batches equals step on the same rows; fit with snapshots; a resumed run equals the
    uninterrupted one bit for bit;
  - the refusals."""
import ctypes as C
import os

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import workloads as wl
from multipathnet_b200._lib import MPN_LAYER_CONV, _ptr, _vp
from multipathnet_b200.batch_provider import integral_thresholds
from conftest import rel_err, record_parity
from test_train_sequence_gpu import LIMITS, SETUPS, batch, oracle
import _batch_provider_ref as bref

pytestmark = pytest.mark.gpu

# per step: [(H, W, ROIs) per image]; four images, so two and four replicas split every step
DP_BATCHES = [
    [(176, 240, 40), (128, 160, 30), (96, 128, 20), (160, 208, 25)],
    [(128, 176, 10), (160, 224, 50), (144, 192, 33), (112, 160, 9)],
    [(192, 144, 21), (128, 160, 19), (176, 240, 64), (96, 128, 16)],
]
# the fp32-reordering bars (DESIGN 4): the summed gradients (max-norm relative) and the three-step weight deltas (L2
# relative), each step against one trainer started from the same state
REORDER_BAR = 1e-4
DELTA_BAR = 1e-4
DP_SETUPS = ["a_vgg_trunk", "b_mpn_phase2_integral", "c_r18_integral", "e_vgg_trunk_bf16", "f_r18_adam"]


def _contexts(devices):
    """replica 0 on a context of devices[0]'s, the others on contexts with streams of their own"""
    return [mpn.Context(d, own_stream=True) for d in devices]


def _trainer(spec, kw, ctxs):
    ms = [mpn.Model(c, spec, **LIMITS) for c in ctxs]
    return mpn.Trainer(ms[0], replicas=ms[1:], **kw)


def _close(*trainers):
    for t in trainers:
        t.close()
        for m in t.models:
            m.close()


def _plan(name, k):
    """(head, switch to phase 2 before the step) of step k"""
    _, _, script = SETUPS[name]
    head, switch, _ = script[k]
    return head, switch


def _prepare(tr, name, k):
    head, switch = _plan(name, k)
    if switch:
        tr.set_phase2(0.005)
    if len(tr.model.spec.cls_heads) > 1:
        tr.select_head(head)


def _replica_get(tr, j, i, what):
    m = tr.models[j]
    out = np.empty(m.spec.weights[i].shape, np.float32)
    m.ctx.check(m.ctx.lib.mpn_model_train_get(m.h, int(i), int(what), _ptr(out), out.size), "mpn_model_train_get")
    return out


def _assert_replicas_identical(tr):
    for i in tr.trained:
        for what in range(0, 2 + tr._n_states):
            if what == 1:
                continue
            a = _replica_get(tr, 0, i, what)
            for j in range(1, len(tr.models)):
                assert np.array_equal(a, _replica_get(tr, j, i, what)), (i, what, j)


def _masks(tr, spec):
    return {(t, li): tr.dropout_mask(t, li) for t, T in enumerate(spec.towers) for li, L in enumerate(T.layers)
            if L.kind == MPN_LAYER_CONV and L.relu}


def _detect(m, spec):
    img = wl.transform(wl.raw_image(144, 192, 3), spec.transformer)
    return m.detect(img, wl.random_boxes(40, 144, 192, 5), 1.0)


def test_one_replica_through_the_replica_entry_is_the_trainer(ctx):
    name = "a_vgg_trunk"
    spec_fn, kw, _ = SETUPS[name]
    spec = spec_fn()
    ta = mpn.Trainer(mpn.Model(ctx, spec, **LIMITS), **kw)
    tb = mpn.Trainer(mpn.Model(ctx, spec, **LIMITS), **kw)
    lib = ctx.lib
    for k in range(3):
        ims, rois, labels, tg = batch(spec, k, DP_BATCHES)
        la = ta.step(ims, rois, labels, tg)
        keep = [np.ascontiguousarray(im, np.float32) for im in ims]
        ptrs = (_vp * len(keep))(*[im.ctypes.data for im in keep])
        hw = np.array([[im.shape[1], im.shape[2]] for im in keep], np.int32).reshape(-1)
        counts = np.array([r.shape[0] for r in rois], np.int32)
        boxes = np.ascontiguousarray(np.concatenate(rois), np.float32)
        losses = np.zeros(3, np.float32)
        ctx.check(lib.mpn_model_train_step_replicas((_vp * 1)(tb.model.h.value), 1, len(keep), ptrs, hw.ctypes.data_as(C.POINTER(C.c_int32)),
                                                    counts.ctypes.data_as(C.POINTER(C.c_int32)), _ptr(boxes), _ptr(labels), _ptr(tg),
                                                    _ptr(losses)), "step_replicas")
        tb.steps += 1
        assert la == tuple(float(v) for v in losses)
    assert all(np.array_equal(a, b) for a, b in zip(ta.weights(), tb.weights()))
    assert all(np.array_equal(ta.momentum_buffer(i), tb.momentum_buffer(i)) for i in ta.trained)
    assert all(np.array_equal(ta.gradient(i), tb.gradient(i)) for i in ta.trained)
    da, db = _detect(ta.model, spec), _detect(tb.model, spec)
    assert all(np.array_equal(a, b) for a, b in zip(da, db))
    _close(ta, tb)


@pytest.mark.parametrize("K", [2, 4])
@pytest.mark.parametrize("name", DP_SETUPS)
def test_replicas_equal_one_trainer(ctx, name, K):
    spec_fn, kw, _ = SETUPS[name]
    spec = spec_fn()
    ctxs = _contexts([0] * K)
    dp = _trainer(spec, kw, ctxs)
    one = mpn.Trainer(mpn.Model(ctx, spec, **LIMITS), **kw)       # loaded with dp's state before every step
    w0 = dp.weights()
    moved = [np.zeros(np.shape(a)) for a in w0]                   # the sum of one's steps from dp's weights
    worst = {"loss": 0.0, "grad": 0.0, "delta": 0.0, "fp64_loss": 0.0, "fp64_grad": 0.0}
    for k in range(len(DP_BATCHES)):
        ims, rois, labels, tg = batch(spec, k, DP_BATCHES)
        _prepare(dp, name, k)
        one.load_state_dict(dp.state_dict())
        if _plan(name, k)[1] and one.phase == 1:
            one.set_phase2(0.005)
        w = dp.weights()
        ld = dp.step(ims, rois, labels, tg)
        lo = one.step(ims, rois, labels, tg)
        for acc, a, b in zip(moved, one.weights(), w):
            acc += a.astype(np.float64) - b
        # every row as one trainer computes it
        for a, b in zip(dp.outputs(), one.outputs()):
            assert np.array_equal(a, b)
        ma, mb = _masks(dp, spec), _masks(one, spec)
        assert ma.keys() == mb.keys() and all(np.array_equal(ma[q], mb[q]) for q in ma)
        worst["loss"] = max(worst["loss"], max(abs(x - y) / max(abs(y), 1e-30) for x, y in zip(ld, lo)))
        assert worst["loss"] <= 1e-6, (k, ld, lo)
        for i in dp.trained:
            worst["grad"] = max(worst["grad"], rel_err(dp.gradient(i), one.gradient(i)) if np.any(one.gradient(i)) else 0.0)
        assert worst["grad"] <= REORDER_BAR, (k, worst)
        if not kw.get("bf16"):
            ol, og = oracle(name, ctx, dp, spec, w, ims, rois, labels, tg)
            worst["fp64_loss"] = max(worst["fp64_loss"], max(abs(a - b) / abs(b) for a, b in zip(ld, ol)))
            worst["fp64_grad"] = max(worst["fp64_grad"], max(rel_err(dp.gradient(i), g) for i, g in og.items() if np.any(g)))
            assert worst["fp64_loss"] <= 1e-4 and worst["fp64_grad"] <= 1e-3, (k, worst)
        _assert_replicas_identical(dp)
    for i, (a, b, c) in enumerate(zip(dp.weights(), moved, w0)):
        if i in dp.trained and np.any(b):
            worst["delta"] = max(worst["delta"], float(np.linalg.norm(a.astype(np.float64) - c - b) / np.linalg.norm(b)))
    assert worst["delta"] <= DELTA_BAR, worst
    dets = [_detect(m, spec) for m in dp.models]
    for d in dets[1:]:
        assert all(np.array_equal(a, b) for a, b in zip(dets[0], d))
    record_parity(f"train_dp::{name}::K{K}", **worst)
    _close(dp, one)
    for c in ctxs:
        c.close()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs two GPUs")
def test_placement_does_not_change_the_bits():
    name = "b_mpn_phase2_integral"
    spec_fn, kw, _ = SETUPS[name]
    spec = spec_fn()
    runs = []
    for devices in ([0, 0], [0, 1]):
        ctxs = _contexts(devices)
        tr = _trainer(spec, kw, ctxs)
        losses = []
        for k in range(len(DP_BATCHES)):
            _prepare(tr, name, k)
            losses.append(tr.step(*batch(spec, k, DP_BATCHES)))
            _assert_replicas_identical(tr)
        runs.append((losses, tr.weights(), [tr.optim_state(i) for i in tr.trained], tr.outputs()))
        _close(tr)
        for c in ctxs:
            c.close()
    (la, wa, sa, oa), (lb, wb, sb, ob) = runs
    assert la == lb
    assert all(np.array_equal(a, b) for a, b in zip(wa, wb))
    assert all(np.array_equal(x, y) for a, b in zip(sa, sb) for x, y in zip(a, b))
    assert all(np.array_equal(a, b) for a, b in zip(oa, ob))


NCLS, SCALE, MAX_SIZE = 6, 160, 256


@pytest.fixture(scope="module")
def feed():
    return bref.synthetic_coco(24, NCLS, 11)


def _image(sizes):
    def get(i):
        H, W = sizes[i]
        return np.random.default_rng(100 + i).integers(0, 256, (H, W, 3), dtype=np.uint8)
    return get


def _mpn_feed(ctx, feed, imgs_per_batch=2):
    gt, props, sizes = feed
    spec = mpn.models.vgg16_multipathnet(NCLS + 1, seed=6, width_div=4, fc_dim=256, integral_k=3)
    db = mpn.RoiDB(ctx, gt, props, NCLS, integral_thresholds(3), best_number=45)
    prov = mpn.BatchProviderROI(db, _image(sizes), spec.transformer, imgs_per_batch=imgs_per_batch, batch_size=48, scale=SCALE,
                                max_size=MAX_SIZE, seed=31)
    prov.setup_data()
    return spec, db, prov


def _dp(spec, ctxs, lr=0.01):
    ms = [mpn.Model(c, spec, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE) for c in ctxs]
    return mpn.Trainer(ms[0], replicas=ms[1:], lr=lr, seed=77, phase2=True, integral=True)


def test_step_batch_equals_step_on_the_same_rows(feed):
    ctxs = _contexts([0, 0])
    spec, db, prov = _mpn_feed(ctxs[0], feed, imgs_per_batch=4)
    ctxs_b = _contexts([0, 0])
    ta, tb = _dp(spec, ctxs), _dp(spec, ctxs_b)
    for k in range(3):
        if k == 2:
            ta.set_phase2(0.005)
            tb.set_phase2(0.005)
        b = prov.sample_integral(k)
        ims, boxes, labels, targets = b.to_host()
        tb.select_head(b.set)
        rois = np.split(boxes, np.cumsum(b.rois_per_image)[:-1])
        lb = tb.step(ims, rois, labels, targets)
        la = ta.step_batch(b)
        assert la == lb and ta.head == tb.head == b.set
        for x, y in zip(ta.outputs(), tb.outputs()):
            assert np.array_equal(x, y)
        _assert_replicas_identical(ta)
    assert all(np.array_equal(a, b) for a, b in zip(ta.weights(), tb.weights()))
    assert all(np.array_equal(ta.momentum_buffer(i), tb.momentum_buffer(i)) for i in ta.trained)
    _close(ta, tb)
    db.close()
    for c in ctxs + ctxs_b:
        c.close()


OPT = dict(nEpochs=4, epochSize=2, step=2, decay=0.1, snapshot=2, phase2_epoch=3, phase2_learningRate=0.001, integral=True)


def test_fit_and_resume_on_two_replicas(feed, tmp_path):
    ctxs = _contexts([0, 0])
    spec, db, prov = _mpn_feed(ctxs[0], feed)
    ta = _dp(spec, ctxs, 1e-3)
    recs = mpn.fit(ta, prov, dict(OPT, save_folder=str(tmp_path / "a")), log=lambda s: None)
    assert [r["epoch"] for r in recs] == [1, 2, 3, 4] and all(np.isfinite(r["train_loss"]) for r in recs)
    assert sorted(os.listdir(tmp_path / "a")) == sorted(["checkpoint_2.npz", "checkpoint_4.npz", "checkpoint_final.npz", "model_2.t7",
                                                         "model_4.t7", "model_final.t7"])
    _assert_replicas_identical(ta)
    # the two-replica run resumed from epoch 2's snapshot ends where the uninterrupted one ended
    ctxs_c, ctxs_d = [ctxs[0]] + _contexts([0]), _contexts([0, 0])     # replica 0 samples on the RoiDB's context
    tc = _dp(spec, ctxs_c, 1e-3)
    rc = mpn.fit(tc, prov, dict(OPT, save_folder=str(tmp_path / "c"), resume=str(tmp_path / "a" / "checkpoint_2.npz")), log=lambda s: None)
    assert [r["train_loss"] for r in rc] == [r["train_loss"] for r in recs[2:]]
    assert all(np.array_equal(a, b) for a, b in zip(ta.weights(), tc.weights()))
    assert all(np.array_equal(ta.momentum_buffer(i), tc.momentum_buffer(i)) for i in ta.trained)
    _assert_replicas_identical(tc)
    # the same checkpoint loads into a one-replica trainer, and a one-replica checkpoint into two replicas
    one = mpn.Trainer(mpn.Model(ctxs[0], spec, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE), lr=1e-3, seed=77, phase2=True, integral=True)
    one.load_state_dict(mpn.load_checkpoint(str(tmp_path / "a" / "checkpoint_final.npz")))
    assert all(np.array_equal(a, b) for a, b in zip(ta.weights(), one.weights()))
    td = _dp(spec, ctxs_d, 1e-3)
    td.load_state_dict(one.state_dict())
    _assert_replicas_identical(td)
    assert all(np.array_equal(a, b) for a, b in zip(one.weights(), td.weights()))
    _close(ta, tc, one, td)
    db.close()
    for c in ctxs + ctxs_c[1:] + ctxs_d:
        c.close()


def test_refusals(ctx):
    spec_fn, kw, _ = SETUPS["a_vgg_trunk"]
    spec = spec_fn()
    ctxs = _contexts([0, 0])
    m0 = mpn.Model(ctxs[0], spec, **LIMITS)
    with pytest.raises(mpn.MpnError, match="replica 1 is the same Model as replica 0"):
        mpn.Trainer(m0, replicas=[m0], **kw)
    other = mpn.Model(ctxs[1], SETUPS["a_vgg_trunk"][0](seed=22), **LIMITS)
    with pytest.raises(mpn.MpnError, match="replica 1 has another spec"):
        mpn.Trainer(m0, replicas=[other], **kw)
    used = mpn.Model(ctxs[1], spec, **LIMITS)
    used.detect(wl.transform(wl.raw_image(96, 128, 1), spec.transformer), wl.random_boxes(8, 96, 128, 1), 1.0)
    with pytest.raises(mpn.MpnError, match="replica 1 already ran inference"):
        mpn.Trainer(m0, replicas=[used], **kw)
    m1 = mpn.Model(ctxs[1], spec, **LIMITS)
    tr = mpn.Trainer(m0, replicas=[m1], **kw)
    ims, rois, labels, tg = batch(spec, 0, DP_BATCHES)
    with pytest.raises(mpn.MpnError, match="images_per_batch must be a multiple of train_nGPU"):
        tr.step(ims[:3], rois[:3], labels[:90], tg[:90])
    empty = [rois[0], rois[1], rois[2][:0], rois[3][:0]]
    with pytest.raises(mpn.MpnError, match="replica 1's images 2..3 have no ROIs"):
        tr.step(ims, empty, labels[:70], tg[:70])
    # the library refuses the same, and a refused step leaves nothing pending: the next step runs
    lib = ctx.lib
    h = (_vp * 2)(m0.h.value, m0.h.value)
    assert lib.mpn_model_train_allreduce(h, 2) != 0 and b"same model" in lib.mpn_last_error(m0.ctx.h)
    tr.step(ims, rois, labels, tg)
    _assert_replicas_identical(tr)
    _close(tr)
    for m in (other, used):
        m.close()
    for c in ctxs:
        c.close()

"""GPU: resuming a training bit for bit (Trainer.state_dict / load_state_dict, save_checkpoint / load_checkpoint over
mpn_model_train_set / _get_state / _set_state) on three setups and at the resume points where optim.sgd's first-step
rule applies; the refusals; fit's schedule against the same calls made by hand, its snapshots and a resume from one;
validate against Tester.testOne + coco_evaluate on a fresh model, and training unchanged by validation."""
import ctypes as C
import dataclasses
import json
import os

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import coco_eval, models, utils, workloads as wl
from multipathnet_b200._lib import CTrainState, MPN_LAYER_CONV, _ptr
from multipathnet_b200.batch_provider import integral_thresholds
from multipathnet_b200.modules import ImageTransformer
import _batch_provider_ref as bref

pytestmark = pytest.mark.gpu

NCLS, SCALE, MAX_SIZE = 6, 160, 256


@pytest.fixture(scope="module")
def feed():
    return bref.synthetic_coco(24, NCLS, 11)


def _image(sizes):
    def get(i):
        H, W = sizes[i]
        return np.random.default_rng(100 + i).integers(0, 256, (H, W, 3), dtype=np.uint8)
    return get


def _batch(spec, seed, sizes=((128, 176), (160, 208)), per_image=(24, 24)):
    rng = np.random.default_rng(seed)
    ims = [wl.transform(wl.raw_image(h, w, seed + i), spec.transformer) for i, (h, w) in enumerate(sizes)]
    rois = [wl.random_boxes(n, h, w, seed + i).astype(np.float32) for i, ((h, w), n) in enumerate(zip(sizes, per_image))]
    R, C_ = sum(per_image), spec.num_classes
    labels = rng.integers(1, C_ + 1, R).astype(np.int32)
    labels[:4] = 1
    tg = np.zeros((R, 4 * C_), np.float32)
    for r in range(R):
        if labels[r] > 1:
            tg[r, 4 * labels[r] - 4:4 * labels[r]] = rng.standard_normal(4) * 0.8
    return ims, rois, labels, tg


class _Setup:
    """one training setup: how to build the model and trainer, and how to run step number k"""

    def __init__(self, ctx, feed, which):
        self.ctx, self.which = ctx, which
        gt, props, sizes = feed
        self.image = _image(sizes)
        if which == "vgg_trunk":
            self.spec = models.vgg16_fast_rcnn(NCLS + 1, seed=5, width_div=4, fc_dim=256)
            self.kw = dict(train_trunk=True)
            self.prov = None
        else:
            if which == "mpn_phase2":
                self.spec = models.vgg16_multipathnet(NCLS + 1, seed=6, width_div=4, fc_dim=256, integral_k=3)
                self.kw = dict(phase2=True, integral=True)
            else:
                self.spec = models.resnet18_fast_rcnn(NCLS + 1, seed=7, blocks=(1, 1, 1, 1), fixed_bn=True, integral_k=3)
                self.kw = dict(train_trunk=True, integral=True)
            self.db = mpn.RoiDB(ctx, gt, props, NCLS, integral_thresholds(3), best_number=45)
            self.prov = mpn.BatchProviderROI(self.db, self.image, self.spec.transformer, batch_size=48, scale=SCALE, max_size=MAX_SIZE, seed=31)
            self.prov.setup_data()

    def trainer(self, lr=0.01):
        m = mpn.Model(self.ctx, self.spec, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
        return mpn.Trainer(m, lr=lr, seed=77, **self.kw)

    def step(self, tr, k):
        if self.prov is not None:
            return tr.step_batch(self.prov.sample_integral(k))
        return tr.step(*_batch(self.spec, 40 + k))


def _script(k, n, switch=None):
    """the calls of a run of n steps whose first k steps include a set_lr and a decay (both before any step when k = 0)
    and, at step `switch`, MultiPathNet's switch to phase 2: a list of ("step", index) / ("set_lr", lr) / ... up to the
    resume point k, then the rest"""
    first = [("set_lr", 0.005)] + [("step", j) for j in range((k + 1) // 2)] + [("decay", 0.5)] + [("step", j) for j in range((k + 1) // 2, k)]
    rest = [("step", j) for j in range(k, n)]
    if switch is not None:
        for part in (first, rest):
            for p, c in enumerate(part):
                if c == ("step", switch):
                    part.insert(p, ("phase2", 0.001))
                    break
    return first, rest


def _run(setup, tr, calls):
    losses = []
    for c in calls:
        if c[0] == "step":
            losses.append(setup.step(tr, c[1]))
        elif c[0] == "set_lr":
            tr.set_lr(c[1])
        elif c[0] == "decay":
            tr.decay(c[1])
        else:
            tr.set_phase2(c[1])
    return losses


def _outcome(setup, tr):
    spec = setup.spec
    masks = {}
    for t, T in enumerate(spec.towers):
        for li, L in enumerate(T.layers):
            if L.kind == MPN_LAYER_CONV and L.relu:
                masks[(t, li)] = tr.dropout_mask(t, li)
    bufs = {i: tr.momentum_buffer(i) for i in tr.trained}
    st = CTrainState()
    tr.ctx.check(tr.ctx.lib.mpn_model_train_get_state(tr.model.h, C.byref(st)), "state")
    ws = tr.weights()
    img = wl.transform(wl.raw_image(144, 192, 3), spec.transformer)
    det = tr.model.detect(img, wl.random_boxes(40, 144, 192, 5), 1.0)
    return ws, bufs, masks, det, (st.step, st.lr, st.head, st.last_head, st.phase2), tr.steps, tr.trained


CASES = [("vgg_trunk", k, None) for k in (0, 1, 3)] + [("mpn_phase2", k, 2) for k in (0, 1, 3)] + [("resnet18", k, None) for k in (0, 1)]


@pytest.mark.parametrize("which,k,switch", CASES)
def test_resume_equals_uninterrupted(ctx, feed, tmp_path, which, k, switch):
    setup = _Setup(ctx, feed, which)
    n = k + max(k, 2)
    first, rest = _script(k, n, switch)
    ta = setup.trainer()
    la = _run(setup, ta, first + rest)
    want = _outcome(setup, ta)
    tb = setup.trainer()
    lb = _run(setup, tb, first)
    path = str(tmp_path / "ck.npz")
    mpn.save_checkpoint(path, tb, epoch=1)
    tb.close(); tb.model.close()
    tc = setup.trainer()                                         # a fresh Model from the original spec, a fresh Trainer
    d = mpn.load_checkpoint(path)
    assert d["extra"] == {"epoch": 1}
    tc.load_state_dict(d)
    lb += _run(setup, tc, rest)
    got = _outcome(setup, tc)
    assert la == lb, (la, lb)
    ws_a, bufs_a, masks_a, det_a, st_a, steps_a, trained_a = want
    ws_c, bufs_c, masks_c, det_c, st_c, steps_c, trained_c = got
    assert st_a == st_c and steps_a == steps_c == n and trained_a == trained_c
    assert all(np.isfinite(a).all() for a in ws_a)
    assert all(np.array_equal(a, c) for a, c in zip(ws_a, ws_c))
    assert bufs_a.keys() == bufs_c.keys() and all(np.array_equal(bufs_a[i], bufs_c[i]) for i in bufs_a)
    assert masks_a.keys() == masks_c.keys() and all(np.array_equal(masks_a[key], masks_c[key]) for key in masks_a)
    assert all(np.array_equal(a, c) for a, c in zip(det_a, det_c))
    assert st_a[4] == int(("phase2", 0.001) in first + rest)
    for t in (ta, tc):
        t.close(); t.model.close()


def test_set_rewrites_the_planes_a_step_would_leave(ctx, feed):
    """setting every master of a trainer to another trainer's trained values makes the two step identically, also after
    an inference call in between (the inference plan's planes are re-derived)"""
    setup = _Setup(ctx, feed, "vgg_trunk")
    ta, tb = setup.trainer(), setup.trainer()
    for j in range(2):
        setup.step(ta, j)
    img = wl.transform(wl.raw_image(144, 192, 3), setup.spec.transformer)
    boxes = wl.random_boxes(40, 144, 192, 5)
    tb.model.detect(img, boxes, 1.0)                           # tb holds an inference plan from the initial weights
    tb.load_state_dict(ta.state_dict())
    assert all(np.array_equal(a, b) for a, b in zip(ta.model.detect(img, boxes, 1.0), tb.model.detect(img, boxes, 1.0)))
    assert setup.step(ta, 2) == setup.step(tb, 2)
    assert all(np.array_equal(a, b) for a, b in zip(ta.weights(), tb.weights()))
    for t in (ta, tb):
        t.close(); t.model.close()


def _err(ctx, rc):
    assert rc != 0
    return ctx.lib.mpn_last_error(ctx.h).decode()


def test_checkpoint_and_train_state_refusals(ctx, feed):
    setup = _Setup(ctx, feed, "mpn_phase2")
    tr = setup.trainer()
    setup.step(tr, 0)
    d = tr.state_dict()
    # another spec, another K, another config
    other = dataclasses.replace(setup.spec, name="other")
    for spec, kw, what in ((other, dict(phase2=True, integral=True), "name"),
                           (models.vgg16_multipathnet(NCLS + 1, seed=6, width_div=4, fc_dim=256, integral_k=2), dict(phase2=True, integral=True),
                            "shapes"),
                           (setup.spec, dict(phase2=True, integral=True, seed=78), "seed"),
                           (setup.spec, dict(phase2=True, integral=True, momentum=0.8), "momentum"),
                           (setup.spec, dict(integral=True), "phase2_from")):
        m = mpn.Model(ctx, spec, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
        t = mpn.Trainer(m, lr=0.01, **dict(dict(seed=77), **kw))
        with pytest.raises(mpn.MpnError, match=what):
            t.load_state_dict(d)
        t.close(); m.close()
    bad = dict(d, tensors={i: (np.zeros(3, np.float32), b) for i, (w, b) in d["tensors"].items()})
    with pytest.raises(mpn.MpnError, match="tensor"):
        tr.load_state_dict(bad)
    # the entry points' own refusals
    lib, h = ctx.lib, tr.model.h
    frozen = setup.spec.trunk_layers[1].weight
    w = np.zeros(setup.spec.weights[frozen].size, np.float32)
    assert "not a trained tensor" in _err(ctx, lib.mpn_model_train_set(h, frozen, 0, _ptr(w), w.size))
    i = tr.trained[0]
    w = np.zeros(setup.spec.weights[i].size + 1, np.float32)
    assert "elements" in _err(ctx, lib.mpn_model_train_set(h, i, 0, _ptr(w), w.size))
    assert "what" in _err(ctx, lib.mpn_model_train_set(h, i, 1, _ptr(w), w.size - 1))
    st = CTrainState()
    ctx.check(lib.mpn_model_train_get_state(h, C.byref(st)), "state")
    for field, v, msg in (("head", 3, "class head out of range"), ("last_head", -1, "class head out of range"), ("lr", float("nan"), "lr"),
                          ("step", -1, "step out of range"), ("phase2", 2, "phase2 is 0 or 1")):
        s2 = CTrainState(st.step, st.lr, st.head, st.last_head, st.phase2)
        setattr(s2, field, v)
        assert msg in _err(ctx, lib.mpn_model_train_set_state(h, C.byref(s2)))
    tr.set_phase2(None)
    s2 = CTrainState(st.step, st.lr, st.head, st.last_head, 0)
    assert "cannot be undone" in _err(ctx, lib.mpn_model_train_set_state(h, C.byref(s2)))
    ph1 = dict(d, state=dict(d["state"], phase2=0))
    with pytest.raises(mpn.MpnError, match="phase 1"):
        tr.load_state_dict(ph1)
    tr.close()
    assert "no training begun" in _err(ctx, lib.mpn_model_train_set(h, i, 0, _ptr(w), w.size))
    assert "no training begun" in _err(ctx, lib.mpn_model_train_set_state(h, C.byref(st)))
    tr.model.close()
    plain = _Setup(ctx, feed, "vgg_trunk").trainer()
    s3 = CTrainState()
    ctx.check(lib.mpn_model_train_get_state(plain.model.h, C.byref(s3)), "state")
    s3.phase2 = 1
    assert "did not begin with mpn_train_spec.phase2 = 1" in _err(ctx, lib.mpn_model_train_set_state(plain.model.h, C.byref(s3)))
    plain.close(); plain.model.close()


OPT = dict(nEpochs=6, epochSize=2, step=2, decay=0.1, snapshot=3, phase2_epoch=4, phase2_learningRate=0.001, phase2_step=1,
           phase2_decay=0.5, integral=True)


def test_fit_equals_the_calls_by_hand_and_resumes_from_a_snapshot(ctx, feed, tmp_path):
    setup = _Setup(ctx, feed, "mpn_phase2")
    ta = setup.trainer(1e-3)
    logs = []
    recs = mpn.fit(ta, setup.prov, dict(OPT, save_folder=str(tmp_path / "a")), log=logs.append)
    # by hand: train.lua's hooks for this schedule
    tb = setup.trainer(1e-3)
    lr = np.float32(1e-3)
    want_lr, losses = [], []
    for epoch in range(1, 7):
        if epoch == 4:
            tb.set_phase2(0.001)
            lr = np.float32(0.001)
        el = [setup.step(tb, (epoch - 1) * 2 + n) for n in range(2)]
        losses.append((0.0 + el[0][0] + el[1][0]) / 2)
        if epoch % (2 if epoch < 4 else 1) == 0:
            d = 0.1 if epoch < 4 else 0.5
            tb.decay(d)
            lr = np.float32(lr * np.float32(d))
        want_lr.append(float(lr))
    assert [r["epoch"] for r in recs] == [1, 2, 3, 4, 5, 6]
    assert [r["learningRate"] for r in recs] == want_lr
    assert [r["decay"] for r in recs] == [0.1, 0.1, 0.1, 0.5, 0.5, 0.5]
    assert [r["train_loss"] for r in recs] == losses
    assert all(line.startswith("json_stats: ") and json.loads(line[12:]) == r for line, r in zip(logs, recs))
    assert all(np.isfinite(a).all() for a in ta.weights())
    assert all(np.array_equal(a, b) for a, b in zip(ta.weights(), tb.weights()))
    assert all(np.array_equal(ta.momentum_buffer(i), tb.momentum_buffer(i)) for i in ta.trained)
    files = sorted(os.listdir(tmp_path / "a"))
    assert files == sorted(["checkpoint_3.npz", "checkpoint_6.npz", "checkpoint_final.npz", "model_3.t7", "model_6.t7", "model_final.t7"])
    # resuming from epoch 3's snapshot ends where the uninterrupted run ended
    tc = setup.trainer(1e-3)
    rc = mpn.fit(tc, setup.prov, dict(OPT, save_folder=str(tmp_path / "c"), resume=str(tmp_path / "a" / "checkpoint_3.npz")))
    assert [r["epoch"] for r in rc] == [4, 5, 6] and [r["learningRate"] for r in rc] == want_lr[3:]
    assert [r["train_loss"] for r in rc] == [r["train_loss"] for r in recs[3:]]
    assert all(np.array_equal(a, b) for a, b in zip(ta.weights(), tc.weights()))
    assert all(np.array_equal(ta.momentum_buffer(i), tc.momentum_buffer(i)) for i in ta.trained)
    assert tc.phase == 2 and tc.steps == 12
    for t in (ta, tb, tc):
        t.close(); t.model.close()


def _test_set(feed, n=6):
    gt, props, sizes = feed
    get = _image(sizes)
    idx = [i for i in range(len(sizes)) if len(props["boxes"][i])][:n]
    images = [np.ascontiguousarray(get(i).transpose(2, 0, 1), np.float32) / np.float32(255) for i in idx]
    ids = sorted(int(im["id"]) for im in gt["images"])
    sub = dict(gt, images=[im for im in gt["images"] if int(im["id"]) in {ids[i] for i in idx}],
               annotations=[a for a in gt["annotations"] if int(a["image_id"]) in {ids[i] for i in idx}])
    return images, [np.asarray(props["boxes"][i], np.float32) for i in idx], [ids[i] for i in idx], sub


def test_validate_equals_tester_on_a_fresh_model(ctx, feed):
    setup = _Setup(ctx, feed, "vgg_trunk")
    tr = setup.trainer()
    for j in range(3):
        setup.step(tr, j)
    images, props, ids, gt = _test_set(feed)
    stats = mpn.validate(tr.model, setup.spec.transformer, images, props, ids, gt, scale=SCALE, max_size=MAX_SIZE)
    fresh = mpn.Model(ctx, dataclasses.replace(setup.spec, weights=tr.weights()), max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
    tester = mpn.Tester(fresh, ImageTransformer(setup.spec.transformer), [SCALE], MAX_SIZE)
    aboxes_t = [tester.testOne(im, b) for im, b in zip(images, props)]
    aboxes = tester.transposeBoxes(tester.keepTopKPerImage(aboxes_t, 100))
    g = coco_eval.CocoGroundTruth.from_dict(gt)
    want = coco_eval.coco_evaluate(ctx, g, utils.coco_results(aboxes, ids, list(g.cat_ids)))["stats"]
    assert stats.shape == (12,) and np.array_equal(stats, want)
    assert setup.step(tr, 3)                                     # training goes on after validating on its own handle
    tr.close(); tr.model.close(); fresh.close()


def test_validating_every_epoch_trains_as_never_validating(ctx, feed):
    setup = _Setup(ctx, feed, "mpn_phase2")
    images, props, ids, gt = _test_set(feed, 3)
    seen = []

    def val(model):
        s = mpn.validate(model, setup.spec.transformer, images, props, ids, gt, scale=SCALE, max_size=MAX_SIZE)
        seen.append(s)
        return s
    opt = dict(OPT, nEpochs=4, snapshot=1)
    ta, tb = setup.trainer(1e-3), setup.trainer(1e-3)
    ra = mpn.fit(ta, setup.prov, opt, validate_fn=val, log=lambda s: None)
    rb = mpn.fit(tb, setup.prov, opt, log=lambda s: None)
    assert len(seen) == 5 and len(ra) == 9                       # per epoch a line, then one with the metrics; and final
    assert [(r["coco_metric"], r["voc_metric"]) for r in ra[1::2]] + [(ra[-1]["coco_metric"], ra[-1]["voc_metric"])] == \
        [(float(s[0]), float(s[1])) for s in seen]
    assert [r["train_loss"] for r in ra[0:8:2]] == [r["train_loss"] for r in rb]
    assert all(np.array_equal(a, b) for a, b in zip(ta.weights(), tb.weights()))
    assert all(np.array_equal(ta.momentum_buffer(i), tb.momentum_buffer(i)) for i in ta.trained)
    for t in (ta, tb):
        t.close(); t.model.close()

"""GPU: the training feed (RoiDB's matching pass, setupData, BatchProviderROI.sample, the flipped getImages,
Trainer.step_batch) against the numpy restatement in _batch_provider_ref.py and the host getImages oracle."""
import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from conftest import record_parity
import _batch_provider_ref as ref

pytestmark = pytest.mark.gpu
NCLS = 6
THR = [(0.5, 0.1, 0.5), (0.6, 0.1, 0.6), (0.7, 0.0, 0.7)]
SCALE, MAX_SIZE = 160, 256


@pytest.fixture(scope="module")
def data():
    gt, props, sizes = ref.synthetic_coco(40, NCLS, 11)
    return gt, props, sizes, ref.restate_roidb(gt, props, NCLS, THR, best_number=45)


def _image(sizes):
    def get(i):
        H, W = sizes[i]
        return np.random.default_rng(100 + i).integers(0, 256, (H, W, 3), dtype=np.uint8)
    return get


def test_matching_pass_matches_the_restatement_bit_for_bit(ctx, data):
    gt, props, sizes, R = data
    db = mpn.RoiDB(ctx, gt, props, NCLS, THR, best_number=45)
    db2 = mpn.RoiDB(ctx, gt, props, NCLS, THR, best_number=45)
    assert db.n_images == len(R)
    kinds = {"empty": 0, "crowd_masked": 0, "no_props": 0}
    for i, (allb, corr, lab, lists, ov) in enumerate(R):
        b, o, c, l, g = db.image_rows(i)
        assert np.array_equal(b, allb) and np.array_equal(o.view(np.uint32), ov.view(np.uint32)), i
        assert np.array_equal(c, corr) and np.array_equal(l, lab), i
        b2, o2, c2, l2, _ = db2.image_rows(i)
        assert np.array_equal(o2.view(np.uint32), o.view(np.uint32)) and np.array_equal(c2, c) and np.array_equal(l2, l)
        for s in range(len(THR)):
            for kind in (0, 1):
                rows = db.rows(s, kind, i)
                assert np.array_equal(rows, lists[s][kind]), (i, s, kind)
                assert np.array_equal(db2.rows(s, kind, i), rows)
                assert db.counts[s, kind, i] == len(rows)
        kinds["empty"] += g == 0
        kinds["crowd_masked"] += int((o == -1).sum())
        kinds["no_props"] += len(o) == g
    assert kinds["empty"] > 0 and kinds["crowd_masked"] > 0 and kinds["no_props"] > 0
    db.close(); db2.close()


def test_regression_stats_within_1e6_of_the_double_restatement(ctx, data):
    gt, props, sizes, R = data
    db = mpn.RoiDB(ctx, gt, props, NCLS, THR, best_number=45)
    prov = mpn.BatchProviderROI(db, _image(sizes), "ross", scale=SCALE, max_size=MAX_SIZE)
    mean, std = prov.setup_data()
    rm, rs = ref.regression_stats([(a, c, L[0][1]) for a, c, _, L, _ in R[:1000]])
    err = max(float(np.max(np.abs(mean - rm) / np.abs(rm))), float(np.max(np.abs(std - rs) / np.abs(rs))))
    record_parity("batch_provider_stats", rel_err=err)
    assert err < 1e-6, (mean, rm, std, rs)
    db.close()


def _ulps(a, b):
    ia, ib = a.view(np.int32).astype(np.int64), b.view(np.int32).astype(np.int64)
    return np.abs(ia - ib)


@pytest.mark.parametrize("seed", [555, 7])
def test_sampled_batches_match_the_restatement(ctx, data, oracle_built, seed):
    gt, props, sizes, R = data
    db = mpn.RoiDB(ctx, gt, props, NCLS, THR, best_number=45)
    prov = mpn.BatchProviderROI(db, _image(sizes), "ross", scale=SCALE, max_size=MAX_SIZE, seed=seed)
    mean, std = prov.setup_data()
    off_ulp = 0
    for set_ in (0, 2):
        for step in range(3):
            batch = prov.sample(step, set_)
            ims, boxes, labels, targets = batch.to_host()
            P, hw, rb, rl, rt, rpi = ref.sample(R, seed, step, set_, 2, 96, 32, sizes, mean, std, NCLS + 1, SCALE, MAX_SIZE)
            assert np.array_equal(batch.plan, P) and np.array_equal(batch.image_hw, hw) and np.array_equal(batch.rois_per_image, rpi)
            assert np.array_equal(boxes.view(np.uint32), rb.view(np.uint32)) and np.array_equal(labels, rl)
            u = _ulps(targets, rt)
            off_ulp += int((u > 0).sum())
            assert u.max() <= 2
            for k, (img, _, _, flip) in enumerate(P):
                raw = _image(sizes)(img)
                want = oracle_built.hd_get_images_u8(np.ascontiguousarray(raw[:, ::-1] if flip else raw), "ross", *hw[k])
                assert np.array_equal(ims[k], want), (step, k)
    record_parity("batch_provider_targets", seed=seed, targets_off_by_ulp=off_ulp)
    again = prov.sample(1, 0).to_host()
    first = prov.sample(1, 0).to_host()
    assert all(np.array_equal(a, b) for a, b in zip(again[1:], first[1:]))
    db.close()


def test_flipped_get_images_equals_np_flip_of_the_raw_image(ctx, oracle_built):
    rng = np.random.default_rng(5)
    im = rng.integers(0, 256, (97, 133, 3), dtype=np.uint8)
    for kind, (h, w) in (("ross", (150, 205)), ("imagenet", (61, 80))):
        tf = mpn._lib.CImageTransform.of(kind)
        for flip in (0, 1):
            out = np.empty((3, h, w), np.float32)
            ctx.check(ctx.lib.mpn_get_images_u8_flip(ctx.h, im.ctypes.data, 97, 133, mpn._lib.C.byref(tf), h, w, flip, out.ctypes.data), "flip")
            src = np.ascontiguousarray(np.flip(im, 1)) if flip else im
            assert np.array_equal(out, oracle_built.hd_get_images_u8(src, kind, h, w))
            if flip == 0:
                plain = np.empty_like(out)
                ctx.check(ctx.lib.mpn_get_images_u8(ctx.h, im.ctypes.data, 97, 133, mpn._lib.C.byref(tf), h, w, plain.ctypes.data), "u8")
                assert np.array_equal(out, plain)


def test_step_batch_equals_step_on_the_restated_rows(ctx, data, oracle_built):
    gt, props, sizes, R = data
    spec = models.vgg16_fast_rcnn(NCLS + 1, seed=4, width_div=4, fc_dim=256)
    db = mpn.RoiDB(ctx, gt, props, NCLS, THR, best_number=45)
    prov = mpn.BatchProviderROI(db, _image(sizes), spec.transformer, scale=SCALE, max_size=MAX_SIZE, seed=31)
    mean, std = prov.setup_data()
    ma = mpn.Model(ctx, spec, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
    mb = mpn.Model(ctx, spec, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
    ta, tb = mpn.Trainer(ma, seed=9), mpn.Trainer(mb, seed=9)
    for step in range(3):
        la = ta.step_batch(prov.sample(step))
        P, hw, rb, rl, rt, rpi = ref.sample(R, 31, step, 0, 2, 96, 32, sizes, mean, std, NCLS + 1, SCALE, MAX_SIZE)
        ims = []
        for k, (img, _, _, flip) in enumerate(P):
            raw = _image(sizes)(img)
            ims.append(oracle_built.hd_get_images_u8(np.ascontiguousarray(raw[:, ::-1] if flip else raw), spec.transformer, *hw[k]))
        rois = np.split(rb, np.cumsum(rpi)[:-1])
        lb = tb.step(ims, rois, rl, rt)
        assert la == lb, (step, la, lb)
    for i in ta.trained:
        assert np.array_equal(ta._get(i, 0), tb._get(i, 0)) and np.array_equal(ta.gradient(i), tb.gradient(i)), i
    ta.close(); tb.close(); ma.close(); mb.close(); db.close()


def test_refusals(ctx, data):
    gt, props, sizes, R = data
    missing = dict(props, images=list(props["images"]), boxes=list(props["boxes"]), scores=list(props["scores"]))
    name = missing["images"].pop(3); missing["boxes"].pop(3); missing["scores"].pop(3)
    with pytest.raises(mpn.MpnError, match=name):
        mpn.RoiDB(ctx, gt, missing, NCLS)
    with pytest.raises(mpn.MpnError):
        mpn.RoiDB(ctx, gt, props, NCLS, [(0.5, 0.6, 0.5)])                     # bg_lo > bg_hi
    with pytest.raises(mpn.MpnError):
        mpn.RoiDB(ctx, gt, props, NCLS - 3)                                   # class ids out of range
    db = mpn.RoiDB(ctx, gt, props, NCLS, [(0.5, 0.1, 0.5), (1.5, 0.1, 0.5)])   # set 1: no fg row anywhere
    prov = mpn.BatchProviderROI(db, _image(sizes), "ross", scale=SCALE, max_size=MAX_SIZE)
    prov.setup_data()
    with pytest.raises(mpn.MpnError, match="no image"):
        prov.sample(0, 1)
    stale = prov.sample(0)
    prov.sample(1)
    with pytest.raises(mpn.MpnError, match="overwritten"):
        stale.to_host()
    spec = models.vgg16_fast_rcnn(NCLS + 1, seed=4, width_div=4, fc_dim=256)
    m = mpn.Model(ctx, spec, max_rois=8, max_h=MAX_SIZE, max_w=MAX_SIZE)         # a batch has more rows
    tr = mpn.Trainer(m)
    with pytest.raises(mpn.MpnError, match="max_rois"):
        tr.step_batch(prov.sample(0))
    tr.close(); m.close()
    spec2 = models.vgg16_fast_rcnn(NCLS + 3, seed=4, width_div=4, fc_dim=256)
    m2 = mpn.Model(ctx, spec2, max_rois=256, max_h=MAX_SIZE, max_w=MAX_SIZE)
    tr2 = mpn.Trainer(m2)
    with pytest.raises(mpn.MpnError, match="classes"):
        tr2.step_batch(prov.sample(0))
    tr2.close(); m2.close(); db.close()

"""GPU: detect + NMS over several images in one model call (mpn_model_detect_nms_batch / _dev) against per-image
mpn_model_detect_nms calls, bit for bit: scores, clamped boxes, keep lists in emission order, keep counts, im_scale and
the detection sink's records, for every model family in every numerics it runs, with ragged ROI counts (0 and 1
included); the full-size COCO case against the literal nms.c; one live model alternating batched, per-image and heads
calls; the device form and determinism; Tester.testMany and validate(images_per_batch=4); the refusals."""
import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, t7, workloads as wl
from multipathnet_b200._lib import split_detect_batch
from multipathnet_b200.image_detect import ImageDetect
from multipathnet_b200.modules import ImageTransformer
from test_layers_gpu import NUMERICS, options
from test_model_gpu import assert_nms_every_class

pytestmark = pytest.mark.gpu
LIMITS = dict(max_rois=512, max_h=256, max_w=256)
SCALE, MAX_SIZE = 160, 240
THRESH, NMS = -1.5, 0.3

BUILDERS = {
    "vgg": lambda: models.vgg16_fast_rcnn(21, seed=7, width_div=4, fc_dim=256),
    "mpn": lambda: models.vgg16_multipathnet(21, seed=11, width_div=4, fc_dim=256),
    "mpn_integral": lambda: models.vgg16_multipathnet(21, seed=13, width_div=4, fc_dim=256, integral_k=3),
    "resnet18": lambda: models.resnet18_fast_rcnn(21, seed=3, integral_k=0, blocks=(1, 1, 1, 1)),
    "resnet50": lambda: models.resnet50_fast_rcnn(21, seed=5, integral_k=3, blocks=(1, 1, 1, 1)),
    "nin": lambda: models.nin_fast_rcnn(21, seed=9),
    "inception": lambda: models.inception_v3_fast_rcnn(21, seed=4),
    "svd": lambda: models.svd_compress(models.vgg16_fast_rcnn(21, seed=17, width_div=4, fc_dim=256), (128, 64)),
    "t7": lambda: t7.model_from_t7(t7.model_to_t7(models.vgg16_fast_rcnn(21, seed=19, width_div=4, fc_dim=256)), transformer="ross"),
}
# Inception-v3 and NIN (96-channel 1x1 layers) do not run in fp8
CASES = [(b, n) for b in BUILDERS for n in ("default", "bf16", "fp8") if not (b in ("inception", "nin") and n == "fp8")]
# (raw H0, W0) per image and ragged ROI counts: empty images, one-ROI images, the 64-row tile edge
SIZES = [(120, 160), (200, 150), (96, 200), (180, 180), (130, 170)]
BATCHES = [[77], [50, 1], [37, 0, 1, 65, 129]]


def _images(spec, n, seed):
    return [wl.raw_image(h, w, seed + i) for i, (h, w) in enumerate(SIZES[:n])]


def _boxes(rois, seed):
    return [wl.random_boxes(r, h, w, seed + i).astype(np.float32).reshape(-1, 4) for i, (r, (h, w)) in enumerate(zip(rois, SIZES))]


def _sink(model, n):
    rec = torch.zeros((n, mpn.MPN_REC_FLOATS), dtype=torch.float32, device="cuda")
    model.set_detection_sink(rec, n, 100)
    return rec


def per_image(model, spec, ims, boxes_list, scale=SCALE, max_size=MAX_SIZE):
    """what the batched call must give: one detect_nms per image (on the host-scaled image) -> [(scores, bboxes, keeps)],
    im_scales"""
    det = ImageDetect(model, ImageTransformer(spec.transformer), [scale], max_size)
    out, scales = [], []
    for im, b in zip(ims, boxes_list):
        img, s = det.getImages(im)
        scales.append(s)
        if b.shape[0] == 0:
            out.append((np.zeros((0, spec.num_classes), np.float32), np.zeros((0, 4 * spec.num_classes), np.float32),
                        [np.zeros(0, np.int32) for _ in range(spec.num_classes - 1)]))
            continue
        out.append(model.detect_nms(img, b, s, im.shape[2], im.shape[1], THRESH, NMS))
    return out, np.array(scales, np.float64)


def assert_same(got, want):
    assert len(got) == len(want)
    for i, ((gs, gb, gk), (ws, wb, wk)) in enumerate(zip(got, want)):
        assert np.array_equal(gs, ws), f"image {i}: scores differ"
        assert np.array_equal(gb, wb), f"image {i}: boxes differ"
        assert len(gk) == len(wk) and all(np.array_equal(a, b) for a, b in zip(gk, wk)), f"image {i}: keep lists differ"


def _empty_record(rec):
    return rec[0] == 0 and not rec[1:].any()


@pytest.mark.parametrize("builder,numerics", CASES)
def test_batch_equals_per_image_calls(ctx, builder, numerics):
    spec = BUILDERS[builder]()
    with options(ctx, NUMERICS[numerics]):
        mb, mr = mpn.Model(ctx, spec, **LIMITS), mpn.Model(ctx, spec, **LIMITS)
        try:
            for k, rois in enumerate(BATCHES):
                n = len(rois)
                ims, bl = _images(spec, n, 100 * k), _boxes(rois, 100 * k)
                rb, rr = _sink(mb, n), _sink(mr, n)
                want, want_scale = per_image(mr, spec, ims, bl)
                got, got_scale = mb.detect_nms_batch(ims, bl, spec.transformer, SCALE, MAX_SIZE, THRESH, NMS, return_im_scale=True)
                assert_same(got, want)
                assert np.array_equal(got_scale, want_scale)
                assert mb.detection_sink_count() == n
                rb, rr = rb.cpu().numpy(), rr.cpu().numpy()
                for i, r in enumerate(rois):
                    if r:                      # the per-image calls skip images without ROIs: their records are packed
                        j = sum(1 for q in rois[:i] if q)
                        assert np.array_equal(rb[i], rr[j]), f"batch {k}, image {i}: records differ"
                    else:
                        assert _empty_record(rb[i]), f"batch {k}, image {i}: an image without ROIs has an empty record"
                mb.set_detection_sink(None, 0); mr.set_detection_sink(None, 0)
        finally:
            mb.close(); mr.close()


@pytest.mark.parametrize("cfg", ["vgg", "mpn"])
def test_full_size_coco_batch(ctx, cfg):
    spec = models.vgg16_fast_rcnn(81, seed=21) if cfg == "vgg" else models.vgg16_multipathnet(81, seed=23)
    sizes = [(800, 1000), (800, 1000), (666, 1000), (800, 800)]
    ims = [wl.raw_image(h, w, 40 + i) for i, (h, w) in enumerate(sizes)]
    bl = [wl.sharpmask_boxes(1000, h, w, 50 + i).astype(np.float32) for i, (h, w) in enumerate(sizes)]
    mb = mpn.Model(ctx, spec, max_rois=4000, max_h=1000, max_w=1000)
    mr = mpn.Model(ctx, spec, max_rois=1000, max_h=1000, max_w=1000)
    try:
        want, want_scale = per_image(mr, spec, ims, bl, 600, 1000)
        got, got_scale = mb.detect_nms_batch(ims, bl, spec.transformer, 600, 1000, THRESH, NMS, return_im_scale=True)
        assert_same(got, want)
        assert np.array_equal(got_scale, want_scale)
        for s, b, k in got:
            assert_nms_every_class(s, b, k, NMS)
    finally:
        mb.close(); mr.close()


def test_live_model_alternating_entries(ctx):
    """one live model: batched calls, per-image calls and trunk + heads over changing N, sizes and R, each equal to a
    fresh model's; after a batched call there are no cached trunk features"""
    spec = BUILDERS["mpn"]()
    live = mpn.Model(ctx, spec, **LIMITS)
    det = ImageDetect(live, ImageTransformer(spec.transformer), [SCALE], MAX_SIZE)
    script = [("batch", [129, 3, 0]), ("single", [64]), ("batch", [1]), ("heads", [200]), ("batch", [12, 300, 7, 1, 0]),
              ("single", [1]), ("batch", [65, 64])]
    try:
        for k, (kind, rois) in enumerate(script):
            ims, bl = _images(spec, len(rois), 7 * k), _boxes(rois, 7 * k)
            fresh = mpn.Model(ctx, spec, **LIMITS)
            try:
                if kind == "batch":
                    assert_same(live.detect_nms_batch(ims, bl, spec.transformer, SCALE, MAX_SIZE, THRESH, NMS),
                                fresh.detect_nms_batch(ims, bl, spec.transformer, SCALE, MAX_SIZE, THRESH, NMS))
                    assert_same(live.detect_nms_batch(ims, bl, spec.transformer, SCALE, MAX_SIZE, THRESH, NMS),
                                per_image(fresh, spec, ims, bl)[0])
                    # the documented rule: no cached trunk features after a batched call
                    with pytest.raises(mpn.MpnError, match="heads called before a trunk forward"):
                        live.heads(np.array([[1, 2, 2, 30, 30]], np.float32))
                    with pytest.raises(mpn.MpnError, match="recompute_features=false needs cached trunk features"):
                        live.detect(None, bl[0][:1] if rois[0] else np.array([[1, 1, 9, 9]], np.float32), 1.0, False)
                elif kind == "single":
                    img, s = det.getImages(ims[0])
                    assert_same([live.detect_nms(img, bl[0], s, ims[0].shape[2], ims[0].shape[1], THRESH, NMS)],
                                per_image(fresh, spec, ims, bl)[0])
                else:
                    img, s = det.getImages(ims[0])
                    rois5 = np.concatenate([np.ones((rois[0], 1), np.float32), (bl[0] - 1) * np.float32(s) + 1], 1)
                    a = live.forward(img, rois5)
                    b = fresh.forward(img, rois5)
                    assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1])
            finally:
                fresh.close()
    finally:
        live.close()


def test_device_form_equals_host_form_and_repeats(ctx):
    spec = BUILDERS["resnet50"]()
    rois = [37, 0, 1, 65, 129]
    ims, bl = _images(spec, 5, 3), _boxes(rois, 3)
    m = mpn.Model(ctx, spec, **LIMITS)
    try:
        host, host_scale = m.detect_nms_batch(ims, bl, spec.transformer, SCALE, MAX_SIZE, THRESH, NMS, return_im_scale=True)
        R, C = sum(rois), spec.num_classes
        runs = []
        for _ in range(2):
            ims_d = [torch.from_numpy(np.ascontiguousarray(im, np.float32)).cuda() for im in ims]
            boxes_d = torch.from_numpy(np.concatenate(bl, 0)).cuda()
            sc = torch.empty((R, C), device="cuda"); bb = torch.empty((R, 4 * C), device="cuda")
            kp = torch.empty((C - 1) * R, dtype=torch.int32, device="cuda"); kc = torch.empty((5, C - 1), dtype=torch.int32, device="cuda")
            s = m.detect_nms_batch_dev(ims_d, [im.shape[1:] for im in ims], spec.transformer, SCALE, MAX_SIZE, rois, boxes_d, THRESH, NMS,
                                       sc, bb, kp, kc)
            ctx.synchronize()
            runs.append((sc.cpu().numpy(), bb.cpu().numpy(), kp.cpu().numpy(), kc.cpu().numpy()))
            assert np.array_equal(s, host_scale)
        assert all(np.array_equal(a, b) for a, b in zip(*runs)), "two runs differ"
        assert_same(split_detect_batch(*runs[0], rois), host)
    finally:
        m.close()


def test_testMany_equals_testOne(ctx):
    spec = BUILDERS["vgg"]()
    rois = [37, 2, 1, 65, 129]                  # testOne takes no image without proposals (validate skips those)
    ims, bl = _images(spec, 5, 11), _boxes(rois, 11)
    m = mpn.Model(ctx, spec, max_rois=160, max_h=256, max_w=256)          # the five images take two batched calls
    try:
        t = mpn.Tester(m, ImageTransformer(spec.transformer), [SCALE], MAX_SIZE)
        got = t.testMany(ims, bl)
        want = [t.testOne(im, b) for im, b in zip(ims, bl)]
        assert len(got) == len(want)
        for g, w in zip(got, want):
            assert len(g) == len(w) and all(np.array_equal(a, b) for a, b in zip(g, w))
    finally:
        m.close()


def test_validate_images_per_batch_equals_image_by_image(ctx):
    spec = BUILDERS["vgg"]()
    gt, _ = wl.coco_eval_set(10, spec.num_classes - 1, 4, 10, seed=5)
    ids = [im["id"] for im in gt["images"]]
    rng = np.random.default_rng(6)
    ims = [wl.raw_image(480, 640, 60 + i) for i in range(len(ids))]
    props = []
    for i, iid in enumerate(ids):
        n = 0 if i in (2, 7) else int(rng.integers(20, 120))
        gtb = np.array([a["bbox"] for a in gt["annotations"] if a["image_id"] == iid], np.float32).reshape(-1, 4)
        gtb = np.concatenate([gtb[:, :2] + 1, gtb[:, :2] + gtb[:, 2:] + 1], 1)
        props.append(np.concatenate([gtb, wl.random_boxes(n, 480, 640, 70 + i)], 0).astype(np.float32) if n else np.zeros((0, 4), np.float32))
    m = mpn.Model(ctx, spec, max_rois=512, max_h=256, max_w=256)
    try:
        a = mpn.validate(m, spec.transformer, ims, props, ids, gt, scale=SCALE, max_size=MAX_SIZE)
        b = mpn.validate(m, spec.transformer, ims, props, ids, gt, scale=SCALE, max_size=MAX_SIZE, images_per_batch=4)
        assert a.shape == (12,) and np.array_equal(a, b)
    finally:
        m.close()


def test_refusals_leave_the_model_usable(ctx):
    spec = BUILDERS["vgg"]()
    m = mpn.Model(ctx, spec, max_rois=128, max_h=256, max_w=256)
    ims, bl = _images(spec, 2, 1), _boxes([40, 30], 1)
    lib = ctx.lib
    try:
        with pytest.raises(mpn.MpnError, match="at least one image"):
            ctx.check(lib.mpn_model_detect_nms_batch(m.h, 0, None, None, None, 600.0, 1000.0, None, None, 0.0, 0.3, None, None, None, None, None),
                      "batch")
        with pytest.raises(mpn.MpnError, match="more ROIs than max_rois"):
            m.detect_nms_batch(ims, [wl.random_boxes(100, 120, 160, 0), wl.random_boxes(29, 200, 150, 1)], spec.transformer, SCALE, MAX_SIZE)
        with pytest.raises(mpn.MpnError, match="larger than max_h x max_w"):
            m.detect_nms_batch(ims, bl, spec.transformer, 600, 1000)
        with pytest.raises(mpn.MpnError, match="transformer or ROI counts missing"):
            ctx.check(lib.mpn_model_detect_nms_batch(m.h, 1, (mpn._lib._vp * 1)(ims[0].ctypes.data), None, None, 600.0, 1000.0, None, None,
                                                     0.0, 0.3, None, None, None, None, None), "batch")
        rec = _sink(m, 1)
        with pytest.raises(mpn.MpnError, match="detection sink is full"):
            m.detect_nms_batch(ims, bl, spec.transformer, SCALE, MAX_SIZE)
        m.set_detection_sink(None, 0)
        del rec
        r = mpn.Model(ctx, spec, max_rois=128, max_h=256, max_w=256)
        assert_same(m.detect_nms_batch(ims, bl, spec.transformer, SCALE, MAX_SIZE, THRESH, NMS), per_image(r, spec, ims, bl)[0])
        r.close()
    finally:
        m.close()


def test_model_with_a_training_begun_detects_as_per_image(ctx):
    """a model with a training begun runs the batched call as it runs mpn_model_detect_nms (validation on the training
    model's own handle)"""
    spec = models.vgg16_fast_rcnn(21, seed=29, width_div=4, fc_dim=256)
    rois = [40, 0, 20]
    ims, bl = _images(spec, 3, 21), _boxes(rois, 21)
    ta, tb = mpn.Trainer(mpn.Model(ctx, spec, **LIMITS)), mpn.Trainer(mpn.Model(ctx, spec, **LIMITS))
    try:
        got = ta.model.detect_nms_batch(ims, bl, spec.transformer, SCALE, MAX_SIZE, THRESH, NMS)
        assert_same(got, per_image(tb.model, spec, ims, bl)[0])
    finally:
        for t in (ta, tb):
            t.close(); t.model.close()

"""SVD-compressed models (models.svd_compress, utils.SVDlinear) on the device.

  * cfg 2 and cfg 3 at full size, ranks (1024, 256): scores / boxes within 1e-3 normwise of the CPU oracle run on the same
    factored graph; keep lists bit-exact against nms.c for every class. fc6's first factor runs on the fp16-weight scheme
    with split-K in cfg 2;
  * full-rank factoring, and a model whose fc6 / fc7 weights have rank <= L, detect within 1e-3 of the uncompressed model;
  * heads in chunks == one call, bit for bit; a live factored model taken through a sequence of image sizes and ROI counts
    == a fresh model at each point, bit for bit;
  * the bf16 and fp8 numerics run factored models, with the bars of tests/test_bf16_gpu.py and tests/test_fp8_gpu.py;
  * Trainer refuses a factored model."""
import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from oracle import graphs as G
from conftest import rel_err, record_parity
from test_model_gpu import _inputs, assert_nms_every_class
import test_bf16_gpu as BF
import test_fp8_gpu as F8

pytestmark = pytest.mark.gpu
TOL = 1e-3


def _small_vgg(seed=7):
    return models.vgg16_fast_rcnn(21, seed=seed, width_div=4, fc_dim=256)


def _small_mpn(seed=11):
    return models.vgg16_multipathnet(21, seed=seed, width_div=4, fc_dim=256)


@pytest.mark.parametrize("cfg", [2, 3])
def test_full_size_factored_vs_oracle(ctx, cfg):
    if cfg == 2:
        spec, H, W, R, seed, sharp = models.vgg16_fast_rcnn(21, seed=1234), 600, 800, 1000, 2, False
    else:
        spec, H, W, R, seed, sharp = models.vgg16_multipathnet(81, seed=1234), 600, 800, 1000, 3, True
    svd = models.svd_compress(spec, (1024, 256))
    img, boxes = _inputs(svd, H, W, R, seed, sharp=sharp)
    rs, rb, _ = G.test_one(svd, img, boxes, 1.0, W, H, nms_fn=lambda sb, thr: np.zeros(0, np.int64))
    m = mpn.Model(ctx, svd, max_rois=R + 24, max_h=H + 8, max_w=W)
    try:
        scores, bboxes, keeps = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        hf = m.last_flops()[1]
    finally:
        m.close()
    es, eb = rel_err(scores, rs), rel_err(bboxes, rb)
    record_parity(f"svd_full_size_cfg{cfg}", scores=es, boxes=eb)
    assert es < TOL and eb < TOL, (es, eb)
    assert_nms_every_class(scores, bboxes, keeps)
    assert abs(hf / R / models.head_flops_per_roi(svd) - 1) < 1e-9


def _low_rank(spec, ranks, seed):
    """spec with each tower's fc6 / fc7 weight replaced by a rank-L matrix of the same scale"""
    rng = np.random.default_rng(seed)
    w = list(spec.weights)
    for t in spec.towers:
        fl = [i for i, L in enumerate(t.layers) if L.kind == models.MPN_LAYER_FLATTEN][0]
        for k, r in enumerate(ranks):
            L = t.layers[fl + 1 + k]
            a = rng.standard_normal((L.cout, r)) / np.sqrt(r)
            b = rng.standard_normal((r, L.cin)) * np.sqrt(2.0 / L.cin)
            w[L.weight] = (a @ b).astype(np.float32)
    spec.weights = w
    return spec


@pytest.mark.parametrize("case", ["vgg_full_rank", "vgg_low_rank", "mpn_full_rank", "mpn_low_rank"])
def test_lossless_factoring_matches_the_uncompressed_model(ctx, case):
    spec = _small_vgg() if case.startswith("vgg") else _small_mpn()
    if case.endswith("full_rank"):
        ranks = (256, 256)                     # min(N, K) of fc6 (6272 -> 256) and fc7 (256 -> 256)
    else:
        ranks = (128, 64)
        spec = _low_rank(spec, ranks, 5)
    svd = models.svd_compress(spec, ranks)
    H, W, R = (150, 203, 200) if case.startswith("vgg") else (160, 208, 128)
    img, boxes = _inputs(spec, H, W, R, 4, sharp=not case.startswith("vgg"))
    out = []
    for s in (spec, svd):
        m = mpn.Model(ctx, s, max_rois=256, max_h=256, max_w=320)
        try:
            out.append(m.detect(img, boxes, 1.0))
        finally:
            m.close()
    es, eb = rel_err(out[1][0], out[0][0]), rel_err(out[1][1], out[0][1])
    record_parity(f"svd_lossless_{case}", scores=es, boxes=eb)
    assert es < TOL and eb < TOL, (es, eb)


def test_factored_heads_chunk_invariance(ctx):
    """(192, 128): fc6's first factor 6272 -> 192 takes the fill split (11 splits), fc7's 256 -> 128 the heads' rule"""
    spec = models.svd_compress(_small_vgg(), (192, 128))
    m = mpn.Model(ctx, spec, max_rois=512, max_h=256, max_w=320)
    try:
        img, boxes = _inputs(spec, 150, 203, 300, 3)
        from oracle import ref as O
        rois = O.project_rois(boxes, 1.0)
        m.trunk(img)
        cf, bf = m.heads(rois)
        c1, b1 = m.heads(rois[:130]); c2, b2 = m.heads(rois[130:])
        c3, b3 = m.heads(rois[:1])
    finally:
        m.close()
    assert np.array_equal(np.concatenate([c1, c2]), cf) and np.array_equal(np.concatenate([b1, b2]), bf)
    assert np.array_equal(c3, cf[:1]) and np.array_equal(b3, bf[:1])


SEQUENCE = [(160, 208, 250), (128, 160, 1), (150, 203, 65), (200, 256, 129), (160, 208, 64)]


@pytest.mark.parametrize("graph", ["vgg", "mpn"])
def test_live_factored_model_through_shapes_matches_fresh(ctx, graph):
    spec = models.svd_compress(_small_vgg() if graph == "vgg" else _small_mpn(), (192, 128))
    live = mpn.Model(ctx, spec, max_rois=256, max_h=256, max_w=320)
    try:
        for i, (H, W, R) in enumerate(SEQUENCE):
            img, boxes = _inputs(spec, H, W, R, 10 + i, sharp=graph == "mpn")
            got = live.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
            fresh = mpn.Model(ctx, spec, max_rois=256, max_h=256, max_w=320)
            try:
                want = fresh.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
            finally:
                fresh.close()
            assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1]), (H, W, R)
            assert all(np.array_equal(a, b) for a, b in zip(got[2], want[2])), (H, W, R)
    finally:
        live.close()


@pytest.mark.parametrize("graph", ["vgg", "mpn"])
def test_bf16_numerics_on_a_factored_model(ctx, graph):
    if graph == "vgg":
        spec, (H, W, R, seed, sharp) = _small_vgg(), (150, 203, 200, 2, False)
    else:
        spec, (H, W, R, seed, sharp) = _small_mpn(), (160, 208, 128, 6, True)
    spec = models.svd_compress(spec, (192, 128))
    img, boxes = _inputs(spec, H, W, R, seed, sharp=sharp)
    with BF.option(ctx, "bf16", 1):
        m = mpn.Model(ctx, spec, max_rois=256, max_h=256, max_w=320)
        try:
            scores, bboxes, keeps = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        finally:
            m.close()
    BF._graph_check(f"svd_bf16_small_{graph}", (scores, bboxes), spec, img, boxes, W, H)
    assert_nms_every_class(scores, bboxes, keeps)


@pytest.mark.parametrize("graph", ["vgg", "mpn"])
def test_fp8_numerics_on_a_factored_model(ctx, graph):
    if graph == "vgg":
        spec, (H, W, R, seed, sharp) = _small_vgg(), (150, 203, 200, 2, False)
    else:
        spec, (H, W, R, seed, sharp) = _small_mpn(), (160, 208, 128, 6, True)
    spec = models.svd_compress(spec, (192, 128))
    img, boxes = _inputs(spec, H, W, R, seed, sharp=sharp)
    with F8.option(ctx, "fp8", 1):
        m = mpn.Model(ctx, spec, max_rois=256, max_h=256, max_w=320)
        try:
            scores, bboxes, keeps = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        finally:
            m.close()
    F8._graph_check(f"svd_fp8_small_{graph}", (scores, bboxes), spec, img, boxes, W, H)
    assert_nms_every_class(scores, bboxes, keeps)


def test_trainer_refuses_a_factored_model(ctx):
    spec = models.svd_compress(_small_vgg(), (128, 0))
    m = mpn.Model(ctx, spec, max_rois=128, max_h=256, max_w=320)
    try:
        with pytest.raises(mpn.MpnError, match="SVD-compressed"):
            mpn.Trainer(m)
    finally:
        m.close()

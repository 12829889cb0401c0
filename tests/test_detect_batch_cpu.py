"""CPU side of the batched detect (mpn_model_detect_nms_batch): the header's prototypes, the Python wrappers' argument
checks, the split of the image-major outputs by rois_per_image, and Tester.testMany's fallback to testOne."""
import os
import re

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import _lib
from multipathnet_b200._lib import Model, split_detect_batch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _cdef_body():
    h = open(os.path.join(ROOT, "include", "mpn_abi.h")).read()
    return re.sub(r"/\*.*?\*/", "", re.search(r"MPN_CDEF_BEGIN \*/(.*?)/\* MPN_CDEF_END", h, re.S).group(1), flags=re.S)


@pytest.mark.parametrize("name", ["mpn_model_detect_nms_batch", "mpn_model_detect_nms_batch_dev"])
def test_prototypes_in_the_cdef_block(name):
    m = re.search(rf"int {name}\(([^;]*?)\)\s*;", _cdef_body(), re.S)
    assert m, f"{name} is not declared in the MPN_CDEF block"
    args = [a.strip() for a in m.group(1).split(",")]
    assert len(args) == 16 == len(_lib.SIGNATURES[name][1])
    assert args[0] == "mpn_model *m" and args[1] == "int32_t n_images" and args[-1] == "double *im_scale"


def _split_case(rois, C=4, seed=0):
    """image-major outputs of a batch as the library lays them out, and the per-image results they stand for"""
    rng = np.random.default_rng(seed)
    R = sum(rois)
    scores = rng.random((R, C), dtype=np.float32)
    bboxes = rng.random((R, 4 * C), dtype=np.float32)
    keep = np.full((C - 1) * R, -1, np.int32)
    counts = np.zeros((len(rois), C - 1), np.int32)
    want, r0 = [], 0
    for i, r in enumerate(rois):
        lists = []
        for j in range(C - 1):
            n = int(rng.integers(0, r + 1))
            lst = rng.permutation(r)[:n].astype(np.int32)
            keep[(C - 1) * r0 + j * r:(C - 1) * r0 + j * r + n] = lst
            counts[i, j] = n
            lists.append(lst)
        want.append((scores[r0:r0 + r], bboxes[r0:r0 + r], lists))
        r0 += r
    return scores, bboxes, keep, counts, want


@pytest.mark.parametrize("rois", [[7], [3, 0, 1, 5], [0, 0], [1, 64, 0, 2]])
def test_split_by_rois_per_image(rois):
    scores, bboxes, keep, counts, want = _split_case(rois, seed=len(rois))
    got = split_detect_batch(scores, bboxes, keep, counts, rois)
    assert len(got) == len(rois)
    for (gs, gb, gk), (ws, wb, wk) in zip(got, want):
        assert np.array_equal(gs, ws) and np.array_equal(gb, wb)
        assert len(gk) == len(wk) and all(np.array_equal(a, b) for a, b in zip(gk, wk))
        assert all(k.dtype == np.int32 for k in gk)
    none = split_detect_batch(None, None, keep, counts, rois)
    assert all(s is None and b is None for s, b, _ in none)


def test_split_rejects_inconsistent_outputs():
    scores, bboxes, keep, counts, _ = _split_case([3, 2])
    with pytest.raises(ValueError, match="keep_counts must be 3 x"):
        split_detect_batch(scores, bboxes, keep, counts, [3, 2, 0])
    with pytest.raises(ValueError, match="keep_idx does not hold"):
        split_detect_batch(scores, bboxes, keep[:-1], counts, [3, 2])
    with pytest.raises(ValueError, match="negative ROI count"):
        split_detect_batch(scores, bboxes, keep, counts, [6, -1])


def _unbound_model(C=5):
    m = Model.__new__(Model)                   # the argument checks run before any library call
    m.C, m.limits, m.h = C, (64, 128, 128), None
    return m


def test_wrapper_argument_checks():
    m = _unbound_model()
    im = np.zeros((3, 8, 8), np.float32)
    with pytest.raises(ValueError, match="one or more images"):
        m.detect_nms_batch([], [], "ross")
    with pytest.raises(ValueError, match="one box array per image"):
        m.detect_nms_batch([im, im], [np.zeros((0, 4), np.float32)], "ross")
    with pytest.raises(ValueError, match="3 x H x W"):
        m.detect_nms_batch([np.zeros((8, 8), np.float32)], [np.zeros((1, 4), np.float32)], "ross")
    with pytest.raises(ValueError, match="one size and one ROI count each"):
        m.detect_nms_batch_dev([0, 0], [(8, 8)], "ross", 600, 1000, [1, 1], 0, -1.5, 0.3)
    with pytest.raises(ValueError, match="one or more images"):
        m.detect_nms_batch_dev([], [], "ross", 600, 1000, [], 0, -1.5, 0.3)


class _PerImageOnly:
    """a backend with testOne's single detect + NMS call only (no batched call): testMany must loop over testOne"""

    def __init__(self, C):
        self.C, self.calls = C, []

    def detect_nms(self, img, boxes, im_scale, W0, H0, thresh, nms_thresh):
        self.calls.append(boxes.shape[0])
        R = boxes.shape[0]
        scores = np.tile(np.linspace(0, 1, self.C, dtype=np.float32), (R, 1))
        bboxes = np.tile(boxes, (1, self.C)).astype(np.float32)
        return scores, bboxes, [np.arange(min(R, j), dtype=np.int32) for j in range(1, self.C)]


def test_testMany_without_a_batched_backend_is_testOne():
    be = _PerImageOnly(4)
    t = mpn.Tester(object(), mpn.modules.ImageTransformer("ross"), [32], 48, backend=be)
    rng = np.random.default_rng(3)
    ims = [rng.random((3, 20 + 4 * i, 30), dtype=np.float32) for i in range(3)]
    boxes = [np.array([[1, 1, 9, 9], [2, 3, 12, 14]], np.float32)[: 2 - (i % 2)] for i in range(3)]
    got = t.testMany(ims, boxes)
    assert be.calls == [2, 1, 2]
    want = [t.testOne(im, b) for im, b in zip(ims, boxes)]
    assert all(len(g) == len(w) and all(np.array_equal(a, b) for a, b in zip(g, w)) for g, w in zip(got, want))
    with pytest.raises(ValueError, match="one box array per image"):
        t.testMany(ims, boxes[:2])


def test_validate_refuses_a_batch_size_below_one():
    with pytest.raises(mpn.MpnError, match="images_per_batch must be >= 1"):
        mpn.validate(None, "ross", [], [], [], {"images": [], "annotations": [], "categories": []}, images_per_batch=0)

"""GPU suite: mpn_coco_eval (csrc/coco_eval.cu) against the numpy restatement of pycocotools' COCOeval
(tests/_coco_eval_ref.py): precision / recall bit for bit (-1 entries included), stats within 1e-12 of numpy's means."""
import numpy as np
import pytest

import _coco_eval_ref as R
import multipathnet_b200 as mpn
from multipathnet_b200 import coco_eval as CE, workloads as wl

pytestmark = pytest.mark.gpu


def _check(ctx, gt_json, rows):
    gt = CE.CocoGroundTruth.from_dict(gt_json)
    out = CE.coco_evaluate(ctx, gt, rows)
    p, r, s = R.cocoeval(gt_json, rows)
    assert out["precision"].shape == p.shape and out["recall"].shape == r.shape
    bad = np.argwhere(out["precision"] != p)
    assert bad.size == 0, (len(bad), bad[:5].tolist(), [(out["precision"][tuple(b)], p[tuple(b)]) for b in bad[:5]])
    assert np.array_equal(out["recall"], r)
    assert np.max(np.abs(out["stats"] - s)) <= 1e-12, (out["stats"], s)
    return gt, out


@pytest.mark.parametrize("name", sorted(R.hand_cases()))
def test_hand_cases(ctx, name):
    gt_json, rows = R.hand_cases()[name]
    _check(ctx, gt_json, rows)


@pytest.mark.parametrize("n_images,n_cats,anns,dets,seed", [
    (40, 3, 6, 30, 1),        # small pairs, ties, crowds, unknown categories
    (25, 2, 12, 260, 2),      # pairs beyond 100 detections, many annotations per pair
    (6, 1, 120, 100, 3),      # pairs with nd * ng past the shared-memory IoU block
    (300, 12, 7, 60, 4),
])
def test_seeded_sets(ctx, n_images, n_cats, anns, dets, seed):
    gt_json, rows = wl.coco_eval_set(n_images, n_cats, anns, dets, seed)
    _check(ctx, gt_json, rows)


def test_large_set_and_determinism(ctx):
    """>= 64 k rows with a category of > 10 k detections; two calls give the same bits"""
    gt_json, rows = wl.coco_eval_set(700, 6, 7, 100, 11)
    assert rows.shape[0] >= 64000
    cats, counts = np.unique(rows[:, 6].astype(np.int64), return_counts=True)
    assert counts.max() > 10000
    gt, out = _check(ctx, gt_json, rows)
    again = CE.coco_evaluate(ctx, gt, rows)
    for k in ("precision", "recall", "stats"):
        assert np.array_equal(out[k].view(np.int64), again[k].view(np.int64)), k


def test_bad_input_fails_with_a_message(ctx):
    gt_json, rows = R.hand_cases()["perfect"]
    gt = CE.CocoGroundTruth.from_dict(gt_json)
    bad = rows.copy(); bad[0, 0] = 99                                 # image id not in the ground truth
    with pytest.raises(mpn.MpnError, match="not a ground-truth image"):
        CE.coco_evaluate(ctx, gt, bad)
    bad = rows.copy(); bad[0, 5] = np.nan
    with pytest.raises(mpn.MpnError, match="NaN"):
        CE.coco_evaluate(ctx, gt, bad)
    with pytest.raises(mpn.MpnError, match="no detection rows"):
        CE.coco_evaluate(ctx, gt, np.zeros((0, 7), np.float32))
    # the call stays usable after a refusal
    out = CE.coco_evaluate(ctx, gt, rows)
    assert abs(out["stats"][0] - 0.9999999999999998) <= 1e-12


def test_evaluate_mirrors_testcoco(ctx, capsys):
    """testCoco.evaluate's path: per-class, per-image N x 5 boxes (1-based x1 y1 x2 y2 score) -> rows -> stats + 12 lines"""
    gt_json = {"images": [{"id": 10}, {"id": 20}], "categories": [{"id": 1}, {"id": 5}],
               "annotations": [{"id": 1, "image_id": 10, "category_id": 1, "bbox": [0, 0, 10, 10], "area": 100.0, "iscrowd": 0},
                               {"id": 2, "image_id": 20, "category_id": 5, "bbox": [5, 5, 50, 40], "area": 2000.0, "iscrowd": 0}]}
    gt = CE.CocoGroundTruth.from_dict(gt_json)
    aboxes = [[np.array([[1, 1, 11, 11, 0.9]], np.float32), np.zeros((0, 5), np.float32)],
              [np.zeros((0, 5), np.float32), np.array([[6, 6, 56, 46, 0.8], [100, 100, 120, 130, 0.7]], np.float32)]]
    stats = CE.evaluate(ctx, gt, aboxes, [10, 20], [1, 5])
    rows = mpn.utils.coco_results(aboxes, [10, 20], [1, 5])
    _, _, s = R.cocoeval(gt_json, rows)
    assert np.max(np.abs(stats - s)) <= 1e-12
    assert "Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ]" in capsys.readouterr().out

"""CPU suite: the COCOeval restatement (tests/_coco_eval_ref.py) against hand-computed answers, the thresholds, the json
loader and the summary format of multipathnet_b200.coco_eval. The device evaluator is compared with the restatement in
tests/test_coco_eval_gpu.py."""
import json

import numpy as np
import pytest

import _coco_eval_ref as R
from multipathnet_b200 import coco_eval as CE

ONE = 1.0 / (1.0 + np.spacing(1))          # a lone true positive's precision: 0.9999999999999998
A_ALL, A_S, A_M, A_L = 0, 1, 2, 3


def _run(name):
    gt, rows = R.hand_cases()[name]
    return R.cocoeval(gt, rows)


def test_lone_true_positive_precision():
    assert ONE == 0.9999999999999998
    p, r, _ = _run("perfect")
    defined = p[p > -1]
    assert defined.size == 10 * 101 * 2 * 3 and np.all(defined == ONE)
    assert np.all(p[:, :, 0, A_M] == -1) and np.all(p[:, :, 0, A_L] == -1)
    assert np.all(r[:, 0, A_ALL] == 1.0)


def test_iou_062_matches_only_up_to_060():
    p, r, _ = _run("iou_062")
    assert np.array_equal(R.IOU_THRS[:3], [0.5, 0.55, 0.6])
    assert np.all(p[:3, :, 0, A_ALL] == ONE) and np.all(p[3:, :, 0, A_ALL] == 0.0)
    assert np.all(r[:3, 0, A_ALL] == 1.0) and np.all(r[3:, 0, A_ALL] == 0.0)


def test_crowd_absorbs_detections_and_ignores_them():
    p, r, _ = _run("crowd")
    # two higher-scored detections inside the crowd region are ignored: the true positive keeps precision 1
    assert np.all(p[:, :, 0, A_ALL, 2] == ONE) and np.all(r[:, 0, A_ALL, 2] == 1.0)
    assert np.all(r[:, 0, A_ALL, 0] == 0.0)          # maxDets 1 keeps only the (ignored) top detection


def test_area_buckets_and_inclusive_edges():
    p, r, _ = _run("areas")
    assert np.all(r[0, 0, :, 2] == 1.0)               # the 1024 annotation is in small AND medium
    assert r[0, 0, A_ALL, 0] == 0.25 and r[0, 0, A_S, 0] == 0.0 and r[0, 0, A_L, 0] == 1.0


def test_float32_detection_area_at_the_small_edge():
    """w * h rounds to 1024 in float32 (the exact product is above): the unmatched detection is a false positive in
    'small', not ignored, so the true positive after it has precision 1/2"""
    p, _, _ = _run("area_edge_f32")
    assert np.all(p[0, 1:, 0, A_S, 2] == 0.5) and p[0, 0, 0, A_S, 2] == 0.5


def test_score_ties_go_by_image_id():
    p, _, _ = _run("tie_fp_first")
    assert np.all(p[:, :, 0, A_ALL, 2] == 0.5)
    p, _, _ = _run("tie_tp_first")
    assert np.all(p[:, :, 0, A_ALL, 2] == ONE)


def test_equal_iou_goes_to_the_later_annotation():
    p, r, _ = _run("iou_tie_later")
    assert r[0, 0, A_ALL, 2] == 1.0 and np.all(p[0, :, 0, A_ALL, 2] == 1.0)      # 2 / (2 + eps) rounds to 1


def test_annotations_of_images_without_detections_are_not_counted():
    _, r, _ = _run("no_det_image")
    assert np.all(r[:, 0, A_ALL, 2] == 1.0)
    _, r, _ = _run("unknown_cat")                     # a row of an unknown category still brings its image in
    assert np.all(r[:, 0, A_ALL, 2] == 0.5)


def test_more_than_100_detections_and_max_dets():
    p, r, _ = _run("max_dets")
    assert np.all(r[:, 0, :2] == 0.0) and np.all(p[:, :, 0, :2] == 0.0)    # the true positive ranks 120th in its pair
    assert np.all(r[:, 1, A_ALL] == [0.0, 1.0, 1.0])
    assert np.all(p[:, 1:, 1, A_ALL, 1:] == 1.0 / (6.0 + np.spacing(1))) and np.all(p[:, :, 1, A_ALL, 0] == 0.0)


def test_crowd_only_category_stays_minus_one():
    p, r, s = _run("crowd_only")
    assert np.all(p[:, :, 1] == -1) and np.all(r[:, 1] == -1)
    assert s[0] == np.mean(p[:, :, 0, A_ALL, 2][p[:, :, 0, A_ALL, 2] > -1])


def test_zero_rows_and_unknown_images_fail():
    gt, _ = R.hand_cases()["perfect"]
    with pytest.raises(IndexError):
        R.cocoeval(gt, np.zeros((0, 7), np.float32))
    with pytest.raises(AssertionError):
        R.cocoeval(gt, np.array([[5, 0, 0, 1, 1, 0.5, 3]], np.float32))


def test_thresholds_are_numpy_linspace_bitwise():
    assert np.array_equal(CE.IOU_THRS.view(np.int64), np.linspace(.5, .95, 10).view(np.int64))
    assert np.array_equal(CE.REC_THRS.view(np.int64), np.linspace(0, 1, 101).view(np.int64))
    assert CE.IOU_THRS[8] == 0.8999999999999999 and CE.REC_THRS[57] == 0.5700000000000001
    assert np.array_equal(R.IOU_THRS, CE.IOU_THRS) and np.array_equal(R.REC_THRS, CE.REC_THRS)


def test_json_loader(tmp_path):
    d = {"images": [{"id": 42}, {"id": 7}], "categories": [{"id": 90}, {"id": 3}],
         "annotations": [{"id": 5, "image_id": 42, "category_id": 3, "bbox": [1, 2, 3, 4], "area": 11.5, "iscrowd": 0},
                         {"id": 9, "image_id": 7, "category_id": 90, "bbox": [0.5, 0, 10, 10], "area": 80, "iscrowd": 1}]}
    f = tmp_path / "ann.json"
    f.write_text(json.dumps(d))
    g = CE.CocoGroundTruth.from_json(str(f))
    assert g.image_ids.tolist() == [7, 42] and g.cat_ids.tolist() == [3, 90]
    assert g.gt_img.tolist() == [1, 0] and g.gt_cat.tolist() == [0, 1] and g.gt_crowd.tolist() == [0, 1]
    assert g.gt_area.tolist() == [11.5, 80.0] and g.gt_box[1].tolist() == [0.5, 0, 10, 10]
    d["annotations"][1]["id"] = 0
    with pytest.raises(ValueError, match="id 0"):
        CE.CocoGroundTruth.from_dict(d)
    d["annotations"][1]["id"] = 5
    with pytest.raises(ValueError, match="duplicate"):
        CE.CocoGroundTruth.from_dict(d)
    d["annotations"][1]["id"] = 9; d["annotations"][1]["image_id"] = 8
    with pytest.raises(ValueError, match="unknown"):
        CE.CocoGroundTruth.from_dict(d)


def test_summarize_format():
    lines = CE.summarize([0.244, 0.402, 0.268, -1, 0.5, 0.25, 0.1, 0.2, 0.3, 0.4, 0.5, 0.6])
    assert len(lines) == 12
    assert lines[0] == " Average Precision  (AP) @[ IoU=0.50:0.95 | area=   all | maxDets=100 ] = 0.244"
    assert lines[1] == " Average Precision  (AP) @[ IoU=0.50      | area=   all | maxDets=100 ] = 0.402"
    assert lines[3] == " Average Precision  (AP) @[ IoU=0.50:0.95 | area= small | maxDets=100 ] = -1.000"
    assert lines[6] == " Average Recall     (AR) @[ IoU=0.50:0.95 | area=   all | maxDets=  1 ] = 0.100"
    assert lines[10] == " Average Recall     (AR) @[ IoU=0.50:0.95 | area=medium | maxDets=100 ] = 0.500"

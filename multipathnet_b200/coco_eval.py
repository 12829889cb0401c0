"""testCoco on the device: the COCOeval score of testCoco.evaluate (testCoco/init.lua:30-88, testCoco/coco.lua:24-38).

pycocotools' COCOeval (iouType 'bbox', default Params, params.imgIds = the sorted distinct image ids of the result rows)
runs as one library call, `mpn_coco_eval` (csrc/coco_eval.cu). The rules it keeps are listed in DESIGN section 4. There is
no CPU fallback: without the library or a GPU the call fails, like the rest of the product path.
"""
from __future__ import annotations

import json
from dataclasses import dataclass
from typing import Dict, List

import numpy as np

from ._lib import Context, _ptr
from .utils import coco_results

N_IOU, N_REC, N_AREA, N_MAXDET = 10, 101, 4, 3
MAX_DETS = (1, 10, 100)
AREA_LABELS = ("all", "small", "medium", "large")


def _linspace(start: float, stop: float, num: int) -> np.ndarray:
    """np.linspace as the device computes it: i * ((stop - start) / (num - 1)) + start, the last element set to stop"""
    step = (stop - start) / (num - 1)
    out = np.array([i * step + start for i in range(num)], np.float64)
    out[-1] = stop
    return out


IOU_THRS = _linspace(0.5, 0.95, N_IOU)
REC_THRS = _linspace(0.0, 1.0, N_REC)


@dataclass
class CocoGroundTruth:
    """The annotation json as the arrays mpn_coco_eval takes: images and categories ascending by id, annotations in the
    json's order with 0-based indices into those tables."""
    image_ids: np.ndarray      # int64, ascending
    cat_ids: np.ndarray        # int64, ascending (the K axis of precision / recall)
    ann_ids: np.ndarray        # int64 (not used by the score; kept for callers)
    gt_img: np.ndarray         # int32 index into image_ids
    gt_cat: np.ndarray         # int32 index into cat_ids
    gt_box: np.ndarray         # float64 G x 4, x y w h
    gt_area: np.ndarray        # float64, the json "area" field (not w * h)
    gt_crowd: np.ndarray       # int32 0 / 1

    @staticmethod
    def from_dict(d: Dict) -> "CocoGroundTruth":
        """A COCO annotation json already parsed. Annotation id 0 is rejected: COCO ids start at 1, and pycocotools records a
        match by the annotation's id, so a match to id 0 would count as no match."""
        image_ids = np.array(sorted({int(im["id"]) for im in d["images"]}), np.int64)
        cat_ids = np.array(sorted({int(c["id"]) for c in d["categories"]}), np.int64)
        if len(image_ids) != len(d["images"]) or len(cat_ids) != len(d["categories"]):
            raise ValueError("duplicate image or category id in the annotation file")
        anns = d.get("annotations", [])
        ids = np.array([int(a["id"]) for a in anns], np.int64)
        if (ids == 0).any():
            raise ValueError("annotation id 0: COCO annotation ids start at 1 (pycocotools would count a match to it as no match)")
        if len(np.unique(ids)) != len(ids):
            raise ValueError("duplicate annotation id in the annotation file")
        img_of = {int(v): i for i, v in enumerate(image_ids)}
        cat_of = {int(v): i for i, v in enumerate(cat_ids)}
        try:
            gt_img = np.array([img_of[int(a["image_id"])] for a in anns], np.int32)
            gt_cat = np.array([cat_of[int(a["category_id"])] for a in anns], np.int32)
        except KeyError as e:
            raise ValueError(f"annotation refers to an unknown image or category id {e}") from None
        box = np.array([[float(v) for v in a["bbox"]] for a in anns], np.float64).reshape(-1, 4)
        area = np.array([float(a["area"]) for a in anns], np.float64)
        crowd = np.array([int(a.get("iscrowd", 0)) for a in anns], np.int32)
        return CocoGroundTruth(image_ids, cat_ids, ids, gt_img, gt_cat, box, area, crowd)

    @staticmethod
    def from_json(path: str) -> "CocoGroundTruth":
        with open(path) as f:
            return CocoGroundTruth.from_dict(json.load(f))


def coco_evaluate(ctx: Context, gt: CocoGroundTruth, rows) -> Dict[str, np.ndarray]:
    """COCOeval(cocoGt, cocoGt.loadRes(rows)).evaluate / accumulate / summarize on the device. rows: D x 7
    [image_id, x, y, w, h, score, category_id] (float32, as testCoco/init.lua builds them). Returns precision
    [10, 101, K, 4, 3], recall [10, K, 4, 3] and stats [12], as pycocotools' eval['precision'], eval['recall'], stats."""
    d = np.ascontiguousarray(rows, np.float32).reshape(-1, 7)
    K = len(gt.cat_ids)
    prec = np.empty((N_IOU, N_REC, K, N_AREA, N_MAXDET), np.float64)
    rec = np.empty((N_IOU, K, N_AREA, N_MAXDET), np.float64)
    stats = np.empty(12, np.float64)
    arrs = [np.ascontiguousarray(gt.image_ids, np.int64), np.ascontiguousarray(gt.cat_ids, np.int64),
            np.ascontiguousarray(gt.gt_img, np.int32), np.ascontiguousarray(gt.gt_cat, np.int32),
            np.ascontiguousarray(gt.gt_box, np.float64).reshape(-1, 4), np.ascontiguousarray(gt.gt_area, np.float64),
            np.ascontiguousarray(gt.gt_crowd, np.int32)]
    img, cat, gi, gc, gb, ga, gcr = arrs
    G = len(gi)
    if not (len(gc) == len(gb) == len(ga) == len(gcr) == G):
        raise ValueError("ground-truth arrays differ in length")
    ctx.check(ctx.lib.mpn_coco_eval(ctx.h, len(img), _ptr(img), len(cat), _ptr(cat), G, _ptr(gi), _ptr(gc), _ptr(gb), _ptr(ga), _ptr(gcr),
                                    d.shape[0], _ptr(d), _ptr(prec), _ptr(rec), _ptr(stats)), "mpn_coco_eval")
    return {"precision": prec, "recall": rec, "stats": stats}


_SUMMARY = [  # (ap, iouThr, area, maxDets) of COCOeval.summarize's _summarizeDets
    (1, None, "all", 100), (1, 0.5, "all", 100), (1, 0.75, "all", 100), (1, None, "small", 100), (1, None, "medium", 100),
    (1, None, "large", 100), (0, None, "all", 1), (0, None, "all", 10), (0, None, "all", 100), (0, None, "small", 100),
    (0, None, "medium", 100), (0, None, "large", 100)]


def summarize(stats) -> List[str]:
    """The 12 lines COCOeval.summarize prints, in its format."""
    lines = []
    for (ap, thr, area, md), v in zip(_SUMMARY, stats):
        title, kind = ("Average Precision", "(AP)") if ap else ("Average Recall", "(AR)")
        iou = f"{IOU_THRS[0]:0.2f}:{IOU_THRS[-1]:0.2f}" if thr is None else f"{thr:0.2f}"
        lines.append(f" {title:<18} {kind} @[ IoU={iou:<9} | area={area:>6s} | maxDets={md:>3d} ] = {float(v):0.3f}")
    return lines


def evaluate(ctx: Context, gt: CocoGroundTruth, aboxes, image_ids, category_ids, verbose: bool = True) -> np.ndarray:
    """testCoco.evaluate (testCoco/init.lua:30-88): aboxes[class][image] = N x 5 [x1, y1, x2, y2, score] (1-based pixels),
    image_ids[image], category_ids[class] -> the rows of utils.coco_results -> the 12 stats (printed like summarize)."""
    out = coco_evaluate(ctx, gt, coco_results(aboxes, image_ids, category_ids))
    if verbose:
        print("\n".join(summarize(out["stats"])))
    return out["stats"]

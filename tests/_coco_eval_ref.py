"""Test infrastructure: a literal numpy restatement of what pycocotools computes for testCoco's call
(COCO.loadRes of an N x 7 array, COCOeval with iouType 'bbox' and default Params, params.imgIds = the sorted image ids of the
result rows), written the way pycocotools' loops are written: coco.py loadNumpyAnnotations / loadRes, cocoeval.py _prepare /
computeIoU / evaluateImg / accumulate / _summarize, maskApi.c bbIou. pycocotools itself is not available here: the rules are
restated from its published code (DESIGN section 4, parity unpinned)."""
from collections import defaultdict

import numpy as np

IOU_THRS = np.linspace(.5, 0.95, int(np.round((0.95 - .5) / .05)) + 1, endpoint=True)
REC_THRS = np.linspace(.0, 1.00, int(np.round((1.00 - .0) / .01)) + 1, endpoint=True)
MAX_DETS = [1, 10, 100]
AREA_RNG = [[0 ** 2, 1e5 ** 2], [0 ** 2, 32 ** 2], [32 ** 2, 96 ** 2], [96 ** 2, 1e5 ** 2]]
AREA_LBL = ["all", "small", "medium", "large"]


def bb_iou(dt, gt, iscrowd):
    """maskApi.c bbIou: dt m x 4, gt n x 4 (x, y, w, h) doubles -> m x n"""
    m, n = len(dt), len(gt)
    o = np.zeros((m, n))
    for g in range(n):
        G = gt[g]; ga = G[2] * G[3]; crowd = iscrowd[g]
        for d in range(m):
            D = dt[d]; da = D[2] * D[3]
            w = min(D[2] + D[0], G[2] + G[0]) - max(D[0], G[0])
            if w <= 0:
                continue
            h = min(D[3] + D[1], G[3] + G[1]) - max(D[1], G[1])
            if h <= 0:
                continue
            i = w * h
            u = da if crowd else da + ga - i
            o[d, g] = i / u
    return o


def load_res(gt_images, rows):
    """COCO.loadRes(np.ndarray) for boxes: float32 bbox / score scalars, area = w * h in float32, id = row + 1"""
    data = np.asarray(rows, np.float32).reshape(-1, 7)
    anns = []
    for i in range(data.shape[0]):
        anns.append({"image_id": int(data[i, 0]), "bbox": [data[i, 1], data[i, 2], data[i, 3], data[i, 4]], "score": data[i, 5],
                     "category_id": int(data[i, 6])})
    assert isinstance(anns, list)
    anns_img_ids = [a["image_id"] for a in anns]
    assert set(anns_img_ids) == (set(anns_img_ids) & set(gt_images)), "Results do not correspond to current coco set"
    if "bbox" in anns[0] and not anns[0]["bbox"] == []:            # IndexError on zero rows, as pycocotools
        for id, ann in enumerate(anns):
            bb = ann["bbox"]
            ann["area"] = bb[2] * bb[3]
            ann["id"] = id + 1
            ann["iscrowd"] = 0
    return anns


def cocoeval(gt, rows):
    """gt: a parsed annotation json (images, categories, annotations with id, image_id, category_id, bbox, area,
    iscrowd). Returns precision, recall, stats."""
    dts_all = load_res([im["id"] for im in gt["images"]], rows)
    img_ids = sorted(set(a["image_id"] for a in dts_all))
    cat_ids = sorted(c["id"] for c in gt["categories"])
    img_set, cat_set = set(img_ids), set(cat_ids)
    # _prepare: getAnnIds(imgIds, catIds) goes image by image through imgToAnns (json order inside an image)
    img_to_anns = defaultdict(list)
    for a in gt["annotations"]:
        img_to_anns[a["image_id"]].append(a)
    gts = [dict(a) for i in img_ids for a in img_to_anns.get(i, []) if a["category_id"] in cat_set]
    dts = [a for a in dts_all if a["image_id"] in img_set and a["category_id"] in cat_set]
    for g in gts:
        g["ignore"] = g["ignore"] if "ignore" in g else 0
        g["ignore"] = "iscrowd" in g and g["iscrowd"]
    _gts, _dts = defaultdict(list), defaultdict(list)
    for g in gts:
        _gts[g["image_id"], g["category_id"]].append(g)
    for d in dts:
        _dts[d["image_id"], d["category_id"]].append(d)

    def compute_iou(imgId, catId):
        g, d = _gts[imgId, catId], _dts[imgId, catId]
        if len(g) == 0 and len(d) == 0:
            return []
        inds = np.argsort([-x["score"] for x in d], kind="mergesort")
        d = [d[i] for i in inds]
        if len(d) > MAX_DETS[-1]:
            d = d[0:MAX_DETS[-1]]
        if len(g) == 0 or len(d) == 0:
            return []
        gb = [[float(v) for v in x["bbox"]] for x in g]
        db = [[float(v) for v in x["bbox"]] for x in d]
        return bb_iou(db, gb, [int(o["iscrowd"]) for o in g])

    ious = {(i, c): compute_iou(i, c) for i in img_ids for c in cat_ids}

    def evaluate_img(imgId, catId, aRng, maxDet):
        gt_ = _gts[imgId, catId]
        dt = _dts[imgId, catId]
        if len(gt_) == 0 and len(dt) == 0:
            return None
        for g in gt_:
            if g["ignore"] or (g["area"] < aRng[0] or g["area"] > aRng[1]):
                g["_ignore"] = 1
            else:
                g["_ignore"] = 0
        gtind = np.argsort([g["_ignore"] for g in gt_], kind="mergesort")
        gt_ = [gt_[i] for i in gtind]
        dtind = np.argsort([-d["score"] for d in dt], kind="mergesort")
        dt = [dt[i] for i in dtind[0:maxDet]]
        iscrowd = [int(o["iscrowd"]) for o in gt_]
        iou_ = ious[imgId, catId][:, gtind] if len(ious[imgId, catId]) > 0 else ious[imgId, catId]
        T, G, D = len(IOU_THRS), len(gt_), len(dt)
        gtm = np.zeros((T, G)); dtm = np.zeros((T, D))
        gtIg = np.array([g["_ignore"] for g in gt_])
        dtIg = np.zeros((T, D))
        if not len(iou_) == 0:
            for tind, t in enumerate(IOU_THRS):
                for dind, d in enumerate(dt):
                    iou = min([t, 1 - 1e-10])
                    m = -1
                    for gind, g in enumerate(gt_):
                        if gtm[tind, gind] > 0 and not iscrowd[gind]:
                            continue
                        if m > -1 and gtIg[m] == 0 and gtIg[gind] == 1:
                            break
                        if iou_[dind, gind] < iou:
                            continue
                        iou = iou_[dind, gind]
                        m = gind
                    if m == -1:
                        continue
                    dtIg[tind, dind] = gtIg[m]
                    dtm[tind, dind] = gt_[m]["id"]
                    gtm[tind, m] = d["id"]
        a = np.array([d["area"] < aRng[0] or d["area"] > aRng[1] for d in dt]).reshape((1, len(dt)))
        dtIg = np.logical_or(dtIg, np.logical_and(dtm == 0, np.repeat(a, T, 0)))
        return {"dtMatches": dtm, "dtScores": [d["score"] for d in dt], "gtIgnore": gtIg, "dtIgnore": dtIg}

    eval_imgs = [evaluate_img(i, c, a, MAX_DETS[-1]) for c in cat_ids for a in AREA_RNG for i in img_ids]

    # accumulate
    T, R, K, A, M = len(IOU_THRS), len(REC_THRS), len(cat_ids), len(AREA_RNG), len(MAX_DETS)
    precision = -np.ones((T, R, K, A, M))
    recall = -np.ones((T, K, A, M))
    I0, A0 = len(img_ids), len(AREA_RNG)
    for k in range(K):
        Nk = k * A0 * I0
        for a in range(A):
            Na = a * I0
            for m, maxDet in enumerate(MAX_DETS):
                E = [eval_imgs[Nk + Na + i] for i in range(I0)]
                E = [e for e in E if e is not None]
                if len(E) == 0:
                    continue
                dtScores = np.concatenate([e["dtScores"][0:maxDet] for e in E])
                inds = np.argsort(-dtScores, kind="mergesort")
                dtm = np.concatenate([e["dtMatches"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                dtIg = np.concatenate([e["dtIgnore"][:, 0:maxDet] for e in E], axis=1)[:, inds]
                gtIg = np.concatenate([e["gtIgnore"] for e in E])
                npig = np.count_nonzero(gtIg == 0)
                if npig == 0:
                    continue
                tps = np.logical_and(dtm, np.logical_not(dtIg))
                fps = np.logical_and(np.logical_not(dtm), np.logical_not(dtIg))
                tp_sum = np.cumsum(tps, axis=1).astype(dtype=float)
                fp_sum = np.cumsum(fps, axis=1).astype(dtype=float)
                for t, (tp, fp) in enumerate(zip(tp_sum, fp_sum)):
                    tp = np.array(tp); fp = np.array(fp)
                    nd = len(tp)
                    rc = tp / npig
                    pr = tp / (fp + tp + np.spacing(1))
                    q = np.zeros((R,))
                    recall[t, k, a, m] = rc[-1] if nd else 0
                    pr = pr.tolist(); q = q.tolist()
                    for i in range(nd - 1, 0, -1):
                        if pr[i] > pr[i - 1]:
                            pr[i - 1] = pr[i]
                    inds_r = np.searchsorted(rc, REC_THRS, side="left")
                    try:
                        for ri, pi in enumerate(inds_r):
                            q[ri] = pr[pi]
                    except IndexError:
                        pass
                    precision[t, :, k, a, m] = np.array(q)
    return precision, recall, summarize_stats(precision, recall)


def summarize_stats(precision, recall):
    def _s(ap, iouThr=None, areaRng="all", maxDets=100):
        aind = [i for i, l in enumerate(AREA_LBL) if l == areaRng]
        mind = [i for i, d in enumerate(MAX_DETS) if d == maxDets]
        if ap == 1:
            s = precision
            if iouThr is not None:
                s = s[np.where(iouThr == IOU_THRS)[0]]
            s = s[:, :, :, aind, mind]
        else:
            s = recall
            if iouThr is not None:
                s = s[np.where(iouThr == IOU_THRS)[0]]
            s = s[:, :, aind, mind]
        return -1 if len(s[s > -1]) == 0 else np.mean(s[s > -1])
    return np.array([_s(1), _s(1, iouThr=.5), _s(1, iouThr=.75), _s(1, areaRng="small"), _s(1, areaRng="medium"),
                     _s(1, areaRng="large"), _s(0, maxDets=1), _s(0, maxDets=10), _s(0), _s(0, areaRng="small"),
                     _s(0, areaRng="medium"), _s(0, areaRng="large")], np.float64)


# ---- hand-computed cases: name -> (annotation json, result rows). The expected values are asserted in test_coco_eval_cpu.py.
def _gt(images, cats, anns):
    return {"images": [{"id": i} for i in images], "categories": [{"id": c} for c in cats],
            "annotations": [dict(id=n + 1, image_id=a[0], category_id=a[1], bbox=list(a[2]), area=a[3], iscrowd=a[4] if len(a) > 4 else 0)
                            for n, a in enumerate(anns)]}


def _rows(*r):
    return np.array(r, np.float32).reshape(-1, 7)


def _edge_wh():
    """float32 w, h whose float32 product is exactly 1024 while the exact (double) product exceeds 1024"""
    w = np.float32(32) + np.float32(2.0 ** -18)
    h = np.float32(32) - np.float32(2.0 ** -19)
    assert np.float32(w * h) == np.float32(1024) and float(w) * float(h) > 1024
    return float(w), float(h)


def hand_cases():
    ew, eh = _edge_wh()
    return {
        "perfect": (_gt([1], [3], [(1, 3, (10, 10, 20, 20), 400.0)]), _rows([1, 10, 10, 20, 20, 0.9, 3])),
        "iou_062": (_gt([1], [1], [(1, 1, (0, 0, 100, 100), 10000.0)]), _rows([1, 0, 0, 62, 100, 0.9, 1])),
        "crowd": (_gt([1], [1], [(1, 1, (0, 0, 50, 50), 2500.0), (1, 1, (200, 200, 100, 100), 10000.0, 1)]),
                  _rows([1, 210, 210, 30, 30, 0.95, 1], [1, 250, 250, 20, 20, 0.9, 1], [1, 0, 0, 50, 50, 0.8, 1])),
        "areas": (_gt([1], [1], [(1, 1, (0, 0, 30, 30), 900.0), (1, 1, (100, 100, 80, 80), 5000.0), (1, 1, (300, 300, 150, 150), 20000.0),
                                 (1, 1, (500, 0, 30, 30), 1024.0)]),
                  _rows([1, 0, 0, 30, 30, 0.5, 1], [1, 100, 100, 80, 80, 0.6, 1], [1, 300, 300, 150, 150, 0.7, 1],
                        [1, 500, 0, 30, 30, 0.4, 1])),
        "area_edge_f32": (_gt([1], [1], [(1, 1, (0, 0, 30, 30), 900.0)]),
                          _rows([1, 400, 400, ew, eh, 0.9, 1], [1, 0, 0, 30, 30, 0.5, 1])),
        "tie_fp_first": (_gt([1, 2], [1], [(2, 1, (0, 0, 10, 10), 100.0)]),
                         _rows([2, 0, 0, 10, 10, 0.5, 1], [1, 50, 50, 10, 10, 0.5, 1])),
        "tie_tp_first": (_gt([1, 2], [1], [(1, 1, (0, 0, 10, 10), 100.0)]),
                         _rows([2, 50, 50, 10, 10, 0.5, 1], [1, 0, 0, 10, 10, 0.5, 1])),
        "iou_tie_later": (_gt([1], [1], [(1, 1, (0, 0, 10, 20), 200.0), (1, 1, (0, 0, 20, 10), 200.0)]),
                          _rows([1, 0, 0, 10, 10, 0.9, 1], [1, 0, 10, 10, 10, 0.8, 1])),
        "no_det_image": (_gt([1, 2], [1], [(1, 1, (0, 0, 10, 10), 100.0), (2, 1, (0, 0, 10, 10), 100.0)]),
                         _rows([1, 0, 0, 10, 10, 0.5, 1])),
        "max_dets": (_gt([1], [1, 2], [(1, 1, (0, 0, 10, 10), 100.0), (1, 2, (0, 0, 10, 10), 100.0)]),
                     np.concatenate([_rows(*[[1, 100 + 2 * i, 100, 5, 5, 0.9 - i * 0.001, 1] for i in range(150)]),
                                     _rows([1, 0, 0, 10, 10, 0.9 - 120 * 0.001, 1]),
                                     _rows(*[[1, 100 + 2 * i, 100, 5, 5, 0.9 - i * 0.01, 2] for i in range(20)]),
                                     _rows([1, 0, 0, 10, 10, 0.9 - 4.5 * 0.01, 2])])),
        "crowd_only": (_gt([1], [1, 2], [(1, 1, (0, 0, 10, 10), 100.0), (1, 2, (0, 0, 50, 50), 2500.0, 1)]),
                       _rows([1, 0, 0, 10, 10, 0.9, 1], [1, 0, 0, 50, 50, 0.9, 2])),
        "unknown_cat": (_gt([1, 2], [1], [(1, 1, (0, 0, 10, 10), 100.0), (2, 1, (0, 0, 10, 10), 100.0)]),
                        _rows([1, 0, 0, 10, 10, 0.5, 1], [2, 0, 0, 10, 10, 0.5, 9])),
    }

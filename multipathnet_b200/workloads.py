"""Seeded synthetic workloads for the five BASELINE.json configs (SURVEY 8d).

No dataset or proposal file is reachable (no network, data/ absent from the reference tree),
so images are uniform noise pushed through the model's transformer and proposals are random
boxes of the stated shape distribution. Everything is a pure function of the seed.
"""
from __future__ import annotations

import numpy as np

ROSS_MEAN = (102.9801, 115.9465, 122.7717)             # model_utils.lua:138-140
IMAGENET_MEAN = (0.48462227599918, 0.45624044862054, 0.40588363755159)   # model_utils.lua:143-155
IMAGENET_STD = (0.22889466674951, 0.22446679341259, 0.22495548344775)


def raw_image(h: int, w: int, seed: int) -> np.ndarray:
    """3 x H x W float in [0,1], RGB — what loaders/loader.lua:79 hands to detect()."""
    return np.random.default_rng(seed).random((3, h, w), dtype=np.float32)


def transform(im: np.ndarray, kind: str) -> np.ndarray:
    """fbcoco.ImageTransformer:updateOutput (modules/ImageTransformer.lua:19-33)."""
    if kind == "ross":                                  # swap {3,2,1}, x255, minus mean
        out = im[[2, 1, 0]].astype(np.float32) * np.float32(255.0)
        for c in range(3):
            out[c] -= np.float32(ROSS_MEAN[c])
        return out
    if kind == "inception":                             # ImageTransformer({1,1,1}, nil, 2): x2, minus 1 (inceptionv3.lua)
        return im.astype(np.float32) * np.float32(2.0) - np.float32(1.0)
    out = im.astype(np.float32).copy()
    for c in range(3):
        out[c] = (out[c] - np.float32(IMAGENET_MEAN[c])) / np.float32(IMAGENET_STD[c])
    return out


def random_boxes(n: int, img_h: int, img_w: int, seed: int, wmin=16, wmax=None, hmin=16, hmax=None) -> np.ndarray:
    """cfg 2: w ~ U[16, 0.8W], h ~ U[16, 0.8H], top-left uniform s.t. the box stays inside; 1-based [x1,y1,x2,y2]."""
    rng = np.random.default_rng(seed)
    wmax = wmax or 0.8 * img_w
    hmax = hmax or 0.8 * img_h
    w = rng.uniform(wmin, wmax, n)
    h = rng.uniform(hmin, hmax, n)
    x1 = 1 + rng.uniform(0, 1, n) * (img_w - w - 1)
    y1 = 1 + rng.uniform(0, 1, n) * (img_h - h - 1)
    return np.stack([x1, y1, x1 + w, y1 + h], 1).astype(np.float32)


def sharpmask_boxes(n: int, img_h: int, img_w: int, seed: int) -> np.ndarray:
    """cfg 3/4 'SharpMask-shaped' proposals (builder's definition, SURVEY 8d): longest side 128/2^s,
    s in {-2.5..0.5 step .5} (demo.lua:23-25,49-50) x U[.75,1.25], aspect exp(U[ln 1/3, ln 3]), clipped."""
    rng = np.random.default_rng(seed)
    s = rng.choice(np.arange(-2.5, 0.51, 0.5), n)
    L = 128.0 / (2.0 ** s) * rng.uniform(0.75, 1.25, n)
    ar = np.exp(rng.uniform(np.log(1 / 3), np.log(3), n))
    w = np.where(ar >= 1, L, L * ar)
    h = np.where(ar >= 1, L / ar, L)
    cx = rng.uniform(1, img_w, n)
    cy = rng.uniform(1, img_h, n)
    x1 = np.clip(cx - w / 2, 1, img_w - 2); x2 = np.clip(cx + w / 2, x1 + 1, img_w)
    y1 = np.clip(cy - h / 2, 1, img_h - 2); y2 = np.clip(cy + h / 2, y1 + 1, img_h)
    return np.stack([x1, y1, x2, y2], 1).astype(np.float32)


# inn.ROIPooling module-op shapes: name -> (N, C, H, W, R, pooled size, spatial scale, Foveal region of the rois)
ROI_POOL_CASES = {
    "S1": (1, 512, 38, 50, 40, 7, 1 / 16, 0),       # the reference's ROI test, modules/test.lua:60-83 (rois randn*50)
    "S2": (2, 512, 14, 14, 2, 7, 1 / 16, 0),        # utils.testModel's input at the pool: boxes {i,1,1,100,100}
    "S3": (2, 512, 38, 63, 128, 7, 1 / 16, 0),      # Fast R-CNN training batch (train.lua: 2 images, 128 rois)
    "S4": (4, 256, 200, 250, 64, 7, 1 / 4, 3),      # MultiPathNet training at conv3: the x4 Foveal region
    "R1000": (1, 512, 38, 50, 1000, 7, 1 / 16, 0),  # one 600 x 800 test image, 1000 proposals
}


def roi_pool_case(name: str, foveal=None, seed: int = 0):
    """seeded randn feature map and rois of one ROI_POOL_CASES shape -> (fmap, rois R x 5, pooled size, scale).
    Batch indices cycle through the N images. A case with a Foveal region needs `foveal` (R x 5 -> 4R x 5, e.g.
    Context.foveal) to derive it."""
    N, C, H, W, R, P, scale, region = ROI_POOL_CASES[name]
    rng = np.random.default_rng(seed)
    fmap = rng.standard_normal((N, C, H, W), dtype=np.float32)
    if name == "S1":
        rois = (rng.standard_normal((R, 5)) * 50).astype(np.float32)
    elif name == "S2":
        rois = np.zeros((R, 5), np.float32); rois[:, 1:] = [1, 1, 100, 100]
    else:
        rois = np.zeros((R, 5), np.float32)
        rois[:, 1:] = random_boxes(R, int(round(H / scale)), int(round(W / scale)), seed + 1)
    rois[:, 0] = np.arange(R) % N + 1
    if region:
        if foveal is None:
            raise ValueError(f"{name} pools a Foveal region: pass foveal=")
        rois = np.ascontiguousarray(foveal(rois)[region::4])
    return fmap, rois, P, scale


def nms_sweep_boxes(n: int, ncls: int, seed: int, img_h=600, img_w=800, ties=False) -> np.ndarray:
    """cfg 5: ncls x n x 5 scored boxes; distinct scores unless ties=True (scores rounded to 1/20)."""
    rng = np.random.default_rng(seed)
    out = np.empty((ncls, n, 5), np.float32)
    for c in range(ncls):
        out[c, :, :4] = random_boxes(n, img_h, img_w, seed * 1000 + c, wmax=0.4 * img_w, hmax=0.4 * img_h)
        if ties:
            out[c, :, 4] = np.round(rng.random(n) * 20) / 20
        else:
            sc = rng.permutation(n).astype(np.float64) + rng.random(n) * 0.5      # distinct by construction
            out[c, :, 4] = (sc / n).astype(np.float32)
            assert len(np.unique(out[c, :, 4])) == n
    return out


def coco_eval_set(n_images: int, n_cats: int, anns_per_image: float, dets_per_image: int, seed: int, crowd_p: float = 0.02,
                  unknown_cat_p: float = 0.01, tie_p: float = 0.3):
    """A synthetic COCO evaluation set: (annotation json as a dict, D x 7 float32 result rows as testCoco/init.lua builds
    them). Image ids are sparse and unsorted in the json, category ids have gaps, category frequencies are skewed (1/rank).
    Boxes span all three area buckets; the json "area" is below the box area, as a segment's is. Rows mix jittered true
    positives, duplicates, false positives, a share of scores rounded to 1/64 (ties within and across images) and a share of
    rows with a category id the json does not have."""
    rng = np.random.default_rng(seed)
    image_ids = rng.choice(np.arange(1, 20 * n_images + 2), n_images, replace=False).astype(np.int64)
    cat_ids = np.sort(rng.choice(np.arange(1, 2 * n_cats + 1), n_cats, replace=False)).astype(np.int64)
    unknown_cat = int(cat_ids.max()) + 7
    pc = 1.0 / np.arange(1, n_cats + 1)
    pc /= pc.sum()

    def boxes(n):
        w = np.exp(rng.uniform(np.log(4), np.log(400), n)); h = w * np.exp(rng.uniform(-0.7, 0.7, n))
        x = rng.uniform(0, 640 - np.minimum(w, 600)); y = rng.uniform(0, 480 - np.minimum(h, 460))
        return np.stack([x, y, w, h], 1)

    anns, rows, next_id = [], [], 1
    for iid in image_ids:
        ng = int(rng.poisson(anns_per_image))
        gb = np.round(boxes(ng), 2)
        gc = cat_ids[rng.choice(n_cats, ng, p=pc)]
        for j in range(ng):
            area = float(gb[j, 2] * gb[j, 3] * rng.uniform(0.5, 1.0))
            anns.append({"id": next_id, "image_id": int(iid), "category_id": int(gc[j]), "bbox": [float(v) for v in gb[j]],
                         "area": area, "iscrowd": int(rng.random() < crowd_p)})
            next_id += 1
        tp = rng.random(ng) < 0.8
        tb = gb[tp] + rng.normal(0, 0.08, (int(tp.sum()), 4)) * np.repeat(gb[tp, 2:], 2, 1)
        tcat = gc[tp]
        dup = rng.random(len(tb)) < 0.25
        db = np.concatenate([tb, tb[dup] + rng.normal(0, 2, (int(dup.sum()), 4))])
        dc = np.concatenate([tcat, tcat[dup]])
        n_fp = max(dets_per_image - len(db), 0)
        db = np.concatenate([db, boxes(n_fp)])[:dets_per_image]
        dc = np.concatenate([dc, cat_ids[rng.choice(n_cats, n_fp, p=pc)]])[:dets_per_image]
        dc = np.where(rng.random(len(dc)) < unknown_cat_p, unknown_cat, dc)
        sc = rng.random(len(db))
        sc = np.where(rng.random(len(db)) < tie_p, np.round(sc * 64) / 64, sc)
        r = np.empty((len(db), 7), np.float32)
        r[:, 0] = iid; r[:, 1:5] = db; r[:, 5] = sc; r[:, 6] = dc
        rows.append(r)
    gt = {"images": [{"id": int(i)} for i in image_ids], "categories": [{"id": int(c)} for c in rng.permutation(cat_ids)],
          "annotations": anns}
    return gt, np.concatenate(rows, 0)

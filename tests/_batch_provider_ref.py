"""numpy restatement of the training feed (DataSetJSON.lua, BatchProviderROI.lua, BatchProviderBase.lua, utils.lua), written
from the reference independently of csrc/roidb_rule.cuh: fp32 numpy ops for Torch's FloatTensor ops, Python floats for
Lua numbers."""
import math

import numpy as np

from _train_ref import philox4x32_10

f32 = np.float32
DRAW_IMAGE, DRAW_FLIP, DRAW_BG, DRAW_FG = 1, 2, 3, 4


def gt_rows(anns, min_area=0.0, num_classes=None):
    """anns: list of (x, y, w, h, area, class_id, crowd, difficult) -> (gt boxes G x 4, classes, crowd boxes)"""
    gt, cls, crowd = [], [], []
    for x, y, w, h, area, c, is_crowd, diff in anns:
        if not area > min_area:
            continue
        b = np.array([x, y, w, h], np.float64).astype(f32)
        box = np.array([b[0], b[1], (b[2] + b[0]) + f32(1), (b[3] + b[1]) + f32(1)], f32)
        if is_crowd:
            crowd.append(box)
        if not diff and not is_crowd:
            gt.append(box)
            cls.append(int(c))
    return np.array(gt, f32).reshape(-1, 4), np.array(cls, np.int32), np.array(crowd, f32).reshape(-1, 4)


def filter_proposals(boxes, scores, best_number, min_area=0.0):
    boxes = np.asarray(boxes, f32).reshape(-1, 4)
    if min_area != 0:
        s = (boxes[:, 2] - boxes[:, 0]) * (boxes[:, 3] - boxes[:, 1])
        keep = s > f32(min_area)
        boxes = boxes[keep]
        scores = None if scores is None else np.asarray(scores, f32)[keep]
    if scores is not None and boxes.shape[0] > best_number:
        idx = np.argsort(-np.asarray(scores, f32), kind="stable")[:best_number]
        boxes = boxes[idx]
    return boxes


def boxoverlap(a, b):
    """utils.boxoverlap(a, b) for rows a (n x 4 fp32) and one box b"""
    a = np.asarray(a, f32).reshape(-1, 4)
    x1 = np.maximum(a[:, 0], b[0]); y1 = np.maximum(a[:, 1], b[1])
    x2 = np.minimum(a[:, 2], b[2]); y2 = np.minimum(a[:, 3], b[3])
    w = (x2 - x1) + f32(1); h = (y2 - y1) + f32(1)
    inter = w * h
    aarea = ((a[:, 2] - a[:, 0]) + f32(1)) * ((a[:, 3] - a[:, 1]) + f32(1))
    barea = (float(b[2]) - float(b[0]) + 1.0) * (float(b[3]) - float(b[1]) + 1.0)
    with np.errstate(divide="ignore", invalid="ignore"):
        o = inter / ((aarea + f32(barea)) - inter)
    o[(w < 0) | (h < 0)] = 0
    return o.astype(f32)


def intersection(a, b):
    a = np.asarray(a, f32).reshape(-1, 4)
    x1 = np.maximum(a[:, 0], b[0]); y1 = np.maximum(a[:, 1], b[1])
    x2 = np.minimum(a[:, 2], b[2]); y2 = np.minimum(a[:, 3], b[3])
    inter = ((x2 - x1) + f32(1)) * ((y2 - y1) + f32(1))
    aarea = ((a[:, 2] - a[:, 0]) + f32(1)) * ((a[:, 3] - a[:, 1]) + f32(1))
    with np.errstate(divide="ignore", invalid="ignore"):
        return (inter / aarea).astype(f32)


def attach(gt, cls, crowd, props):
    """attachProposals -> (all_boxes, overlap, correspondance (1-based, 0 none), label)"""
    allb = np.concatenate([gt, props], 0).astype(f32)
    n, G = allb.shape[0], gt.shape[0]
    if G > 0:
        O = np.stack([boxoverlap(allb, gt[g]) for g in range(G)], 1)
        ov = O.max(1).astype(f32)
        corr = (O.argmax(1) + 1).astype(np.int32)           # argmax: first maximum
        corr[ov == 0] = 0
    else:
        ov, corr = np.zeros(n, f32), np.zeros(n, np.int32)
    label = np.where(corr > 0, cls[np.maximum(corr - 1, 0)] if G else 0, 0).astype(np.int32)
    if crowd.shape[0] > 0 and n > 0:
        inter = np.stack([intersection(allb, c) for c in crowd], 0).max(0)
        mask = inter > f32(0.7)
        mask[:G] = False
        ov = ov.copy(); ov[mask] = -1
    return allb, ov, corr, label


def lists(ov, fg, lo, hi):
    """(bg rows, fg rows) in row order"""
    return (np.nonzero((ov >= f32(lo)) & (ov < f32(hi)))[0].astype(np.int32), np.nonzero(ov >= f32(fg))[0].astype(np.int32))


def convert_f32(b, t):
    """utils.convertTo's 2-D branch on n x 4 fp32 rows"""
    b, t = np.asarray(b, f32), np.asarray(t, f32)
    xc = (b[:, 0] + b[:, 2]) * f32(0.5); yc = (b[:, 1] + b[:, 3]) * f32(0.5)
    w = b[:, 2] - b[:, 0]; h = b[:, 3] - b[:, 1]
    xtc = (t[:, 0] + t[:, 2]) * f32(0.5); ytc = (t[:, 1] + t[:, 3]) * f32(0.5)
    wt = t[:, 2] - t[:, 0]; ht = t[:, 3] - t[:, 1]
    return np.stack([(xtc - xc) / w, (ytc - yc) / h, np.log((wt / w).astype(np.float64)).astype(f32),
                     np.log((ht / h).astype(np.float64)).astype(f32)], 1).astype(f32)


def convert_f64(b, t):
    """utils.convertTo's 1-D branch (Lua numbers) on one row, stored into fp32"""
    b, t = [float(v) for v in b], [float(v) for v in t]
    xc, yc = (b[0] + b[2]) * 0.5, (b[1] + b[3]) * 0.5
    w, h = b[2] - b[0], b[3] - b[1]
    xtc, ytc = (t[0] + t[2]) * 0.5, (t[1] + t[3]) * 0.5
    wt, ht = t[2] - t[0], t[3] - t[1]
    return np.array([(xtc - xc) / w, (ytc - yc) / h, math.log(wt / w), math.log(ht / h)], np.float64).astype(f32)


def regression_stats(rows_per_image):
    """setupData from [(all_boxes, corr, fg rows)] of the first images: mean and unbiased std in double, rounded to fp32"""
    vals = [convert_f32(b[fg], b[c[fg] - 1]) for b, c, fg in rows_per_image if len(fg)]
    v = np.concatenate(vals, 0).astype(np.float64)
    return v.mean(0), v.std(0, ddof=1)


def draw_u32(seed, step, slot, set_, purpose, draws):
    d = np.asarray(draws, np.uint64).reshape(-1)
    n = d.shape[0]
    out = philox4x32_10([d, np.full(n, step, np.uint64), np.full(n, slot, np.uint64), np.full(n, (set_ << 8) | purpose, np.uint64)],
                        (seed & 0xFFFFFFFF, seed >> 32))
    return out[0]


def rand_int(u, n):
    """torch.random(n) as restated: 1 + floor(u * n / 2^32)"""
    return (1 + ((np.asarray(u, np.uint64) * np.uint64(n)) >> np.uint64(32))).astype(np.int64)


def plan(n_bg, n_fg, seed, step, set_, n_slots):
    out = []
    for k in range(n_slots):
        bg = fg = cur = -1
        d = 0
        while bg < 0 or fg < 0:
            cur = int(rand_int(draw_u32(seed, step, k, set_, DRAW_IMAGE, [d]), len(n_bg))[0]) - 1
            d += 1
            if n_bg[cur] > 0:
                bg = cur
            if n_fg[cur] > 0:
                fg = cur
        flip = int(rand_int(draw_u32(seed, step, k, set_, DRAW_FLIP, [0]), 2)[0]) - 1
        out.append((cur, bg, fg, flip))
    return np.array(out, np.int32)


def train_size(H0, W0, scale, max_size):
    s = scale / min(H0, W0)
    im_s = [H0 * s, W0 * s]
    for dim in range(2):
        if im_s[dim] > max_size:
            rat = im_s[dim] / max_size
            im_s = [im_s[0] / rat, im_s[1] / rat]
            s = s / rat
    return int(im_s[0]), int(im_s[1]), s


def train_box(b, scale, width, flip):
    d = ((np.asarray(b, f32) - f32(1)) * f32(scale)) + f32(1)
    if flip:
        t = float(d[0])
        d = d.copy()
        d[0] = f32(width - float(d[2]) + 1.0)
        d[2] = f32(width - t + 1.0)
    return d.astype(f32)


def sample_rows(rois, gtboxes, labels, im_scale, width, flip, mean, std, C):
    """boxes and R x 4C targets of drawn rows (raw boxes, label 1 = bg)"""
    R = len(labels)
    boxes, tg = np.zeros((R, 4), f32), np.zeros((R, 4 * C), f32)
    for r in range(R):
        roi = train_box(rois[r], im_scale, width, flip)
        boxes[r] = roi
        if labels[r] > 1:
            gt = train_box(gtboxes[r], im_scale, width, flip)
            t = convert_f64(roi, gt)
            tg[r, 4 * (labels[r] - 1):4 * labels[r]] = (t - np.asarray(mean, f32)) / np.asarray(std, f32)
    return boxes, tg


def sample(db, seed, step, set_, n_slots, bg_each, fg_each, sizes, mean, std, C, scale=600, max_size=1000):
    """one step from a restated roidb: db[i] = (all_boxes, corr, label, [(bg, fg) per set]); sizes[i] = (H0, W0)
    -> plan, per slot (h, w), boxes, labels, targets, rows per slot"""
    n_bg = [len(d[3][set_][0]) for d in db]
    n_fg = [len(d[3][set_][1]) for d in db]
    P = plan(n_bg, n_fg, seed, step, set_, n_slots)
    out_b, out_l, out_t, hw, rpi = [], [], [], [], []
    for k, (img, bgs, fgs, flip) in enumerate(P):
        h, w, s = train_size(*sizes[img], scale, max_size)
        hw.append((h, w))
        bg, fg = db[bgs][3][set_][0], db[fgs][3][set_][1]
        nb, nf = min(bg_each, len(bg)), min(fg_each, len(fg))
        pb = rand_int(draw_u32(seed, step, k, set_, DRAW_BG, np.arange(nb)), len(bg)) - 1
        pf = rand_int(draw_u32(seed, step, k, set_, DRAW_FG, np.arange(nf)), len(fg)) - 1
        rb, rf = bg[pb], fg[pf]
        allb_b, allb_f, corr_f, lab_f = db[bgs][0], db[fgs][0], db[fgs][1], db[fgs][2]
        rois = np.concatenate([allb_b[rb], allb_f[rf]], 0)
        gts = np.concatenate([np.zeros((nb, 4), f32), allb_f[corr_f[rf] - 1]], 0)
        labels = np.concatenate([np.ones(nb, np.int32), 1 + lab_f[rf]]).astype(np.int32)
        b, t = sample_rows(rois, gts, labels, s, w, flip, mean, std, C)
        out_b.append(b); out_l.append(labels); out_t.append(t); rpi.append(nb + nf)
    return P, np.array(hw), np.concatenate(out_b), np.concatenate(out_l), np.concatenate(out_t), np.array(rpi)


def synthetic_coco(n_images, num_classes, seed, props_per_image=60, gt_per_image=4, crowd_every=3, empty_every=7):
    """a COCO-like dataset with crowds, images without GT, an image with GT but no proposals, tied GT boxes; returns
    (gt dict, proposals dict as t7.proposals_from_t7 returns, image sizes (H, W))"""
    rng = np.random.default_rng(seed)
    images, anns, boxes, scores, sizes = [], [], [], [], []
    aid = 1
    for i in range(n_images):
        H, W = int(rng.integers(120, 260)), int(rng.integers(120, 300))
        sizes.append((H, W))
        images.append({"id": 1000 + 3 * i, "file_name": f"img_{i:05d}.jpg", "height": H, "width": W})
        ng = 0 if i % empty_every == 3 else int(rng.integers(1, gt_per_image + 1))
        for g in range(ng):
            w, h = float(rng.uniform(10, W / 2)), float(rng.uniform(10, H / 2))
            x, y = float(rng.uniform(0, W - w)), float(rng.uniform(0, H - h))
            anns.append({"id": aid, "image_id": 1000 + 3 * i, "category_id": 10 + 2 * int(rng.integers(0, num_classes)),
                         "bbox": [x, y, w, h], "area": w * h * float(rng.uniform(0.5, 1.0)), "iscrowd": 0})
            aid += 1
            if g == 0 and i % 5 == 1:                      # an exact duplicate of GT box 1: a tie, the lower index wins
                anns.append(dict(anns[-1], id=aid, category_id=10 + 2 * ((int(rng.integers(0, num_classes)) + 1) % num_classes)))
                aid += 1
        if i % crowd_every == 2:
            w, h = float(rng.uniform(30, W / 1.5)), float(rng.uniform(30, H / 1.5))
            anns.append({"id": aid, "image_id": 1000 + 3 * i, "category_id": 10, "bbox": [float(rng.uniform(0, W - w)),
                         float(rng.uniform(0, H - h)), w, h], "area": w * h, "iscrowd": 1})
            aid += 1
        npr = 0 if i % 11 == 5 else props_per_image
        gtb = [a["bbox"] for a in anns if a["image_id"] == 1000 + 3 * i]
        b = []
        for p in range(npr):
            if gtb and p % 3 == 0:                         # jittered copies of GT boxes: overlaps across the thresholds
                x, y, w, h = gtb[p % len(gtb)]
                j = rng.normal(0, 0.15, 4) * [w, h, w, h]
                x1, y1 = x + j[0], y + j[1]
                b.append([x1, y1, x1 + w + j[2], y1 + h + j[3]])
            else:
                x1, y1 = rng.uniform(0, W - 12), rng.uniform(0, H - 12)
                b.append([x1, y1, rng.uniform(x1 + 4, W), rng.uniform(y1 + 4, H)])
        boxes.append(np.array(b, np.float32).reshape(-1, 4))
        sc = rng.random(npr).astype(np.float32)
        sc[: npr // 4] = 0.5                               # ties in the score sort
        scores.append(sc)
    cats = [{"id": 10 + 2 * c, "name": f"c{c}"} for c in range(num_classes)]
    gt = {"images": images[::-1], "annotations": anns, "categories": cats}   # json order differs from id order
    props = {"boxes": boxes[::-1], "scores": scores[::-1], "images": [im["file_name"] for im in images][::-1]}
    return gt, props, sizes


def restate_roidb(gt, props, num_classes, thresholds, best_number=1000, min_area=0.0, min_proposal_area=0.0):
    """the RoiDB of (gt, props) restated: per image in ascending id order (all_boxes, corr, label, [(bg, fg)...], overlap)"""
    cat_index = {c["id"]: k + 1 for k, c in enumerate(sorted(gt["categories"], key=lambda c: c["id"]))}
    pidx = {f: k for k, f in enumerate(props["images"])}
    out = []
    for im in sorted(gt["images"], key=lambda im: im["id"]):
        anns = [(*a["bbox"], a["area"], cat_index[a["category_id"]], a.get("iscrowd", 0), a.get("difficult", 0))
                for a in gt["annotations"] if a["image_id"] == im["id"]]
        g, c, cr = gt_rows(anns, min_area)
        k = pidx[im["file_name"]]
        p = filter_proposals(props["boxes"][k], props["scores"][k] if "scores" in props else None, best_number, min_proposal_area)
        allb, ov, corr, lab = attach(g, c, cr, p)
        out.append((allb, corr, lab, [lists(ov, *t) for t in thresholds], ov))
    return out

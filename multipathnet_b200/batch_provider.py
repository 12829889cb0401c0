"""The training feed on the device: DataSetJSON's proposals and ground truth (DataSetJSON.lua) and BatchProviderROI's
minibatches (BatchProviderROI.lua, BatchProviderBase.lua).

`RoiDB` matches every image's proposals to its ground truth once, on the device (attachProposals), and keeps the fg / bg
row lists of each threshold set there. `BatchProviderROI.sample(step)` draws one step's images, flips, ROIs, labels and
normalised regression targets from it and leaves the batch on the device, where `Trainer.step_batch` trains on it.
`sample_integral(step)` first draws the step's threshold set, as train.lua picks one of its loaders per step. The
rules and where they differ from a literal reading of the reference are listed in DESIGN section 4.
"""
from __future__ import annotations

import ctypes as C
import math
import weakref
from dataclasses import dataclass
from typing import Callable, Dict, Sequence, Tuple, Union

import numpy as np

from ._lib import CImageTransform, Context, MpnError, _ptr, _vp
from .coco_eval import CocoGroundTruth


class RoiDB:
    """DataSetJSON:loadROIDB + attachProposals for every image, on the device.

    gt: a COCO annotation dict (images, categories, annotations); images are taken in ascending id order, class_id is the
    1-based index of the category in ascending id order, an annotation may carry "difficult" (default 0).
    proposals: what `t7.proposals_from_t7` returns ({'boxes', 'scores' (optional), 'images' = file names}), matched to the
    images by file name; an image without an entry is refused, naming it.
    thresholds: one (fg, bg_lo, bg_hi) per set; fg rows have overlap >= fg, bg rows bg_lo <= overlap < bg_hi."""

    def __init__(self, ctx: Context, gt: Dict, proposals: Dict, num_classes: int,
                 thresholds: Sequence[Tuple[float, float, float]] = ((0.5, 0.1, 0.5),), best_number: int = 1000,
                 min_area: float = 0, min_proposal_area: float = 0):
        self.ctx, self.num_classes = ctx, int(num_classes)
        g = CocoGroundTruth.from_dict(gt)
        by_id = {int(im["id"]): im for im in gt["images"]}
        self.file_names = [str(by_id[int(i)]["file_name"]) for i in g.image_ids]
        n = len(self.file_names)
        anns = gt.get("annotations", [])
        order = np.argsort(g.gt_img, kind="stable")                    # annotations grouped by image, json order within
        ann_off = np.zeros(n + 1, np.int64)
        np.add.at(ann_off, g.gt_img.astype(np.int64) + 1, 1)
        ann_off = np.cumsum(ann_off)
        xywh = np.ascontiguousarray(g.gt_box[order], np.float64)
        area = np.ascontiguousarray(g.gt_area[order], np.float64)
        cls = np.ascontiguousarray(g.gt_cat[order] + 1, np.int32)
        difficult = np.array([int(a.get("difficult", 0)) != 0 for a in anns], bool).reshape(-1)
        flags = np.ascontiguousarray((g.gt_crowd[order] != 0).astype(np.int32) | (difficult[order].astype(np.int32) << 1), np.int32)

        idx = {str(f): k for k, f in enumerate(proposals.get("images", []))}
        boxes, scores = proposals["boxes"], proposals.get("scores")
        prop_off = np.zeros(n + 1, np.int64)
        sel = []
        for i, f in enumerate(self.file_names):
            if f not in idx:
                raise MpnError(f"RoiDB: image {f} is not in the proposals")
            k = idx[f]
            sel.append(k)
            prop_off[i + 1] = prop_off[i] + np.asarray(boxes[k]).reshape(-1, 4).shape[0]
        pb = np.ascontiguousarray(np.concatenate([np.asarray(boxes[k], np.float32).reshape(-1, 4) for k in sel] or [np.zeros((0, 4))]),
                                  np.float32)
        ps = None
        if scores is not None:
            ps = np.ascontiguousarray(np.concatenate([np.asarray(scores[k], np.float32).reshape(-1) for k in sel] or [np.zeros(0)]),
                                      np.float32)
            if ps.shape[0] != pb.shape[0]:
                raise MpnError("RoiDB: proposal scores and boxes differ in length")
        thr = np.ascontiguousarray(np.asarray(thresholds, np.float32).reshape(-1, 3))
        self.thresholds = [tuple(float(v) for v in t) for t in thr]
        h = _vp()
        ctx.check(ctx.lib.mpn_roidb_create(ctx.h, n, _ptr(ann_off), _ptr(xywh), _ptr(area), _ptr(cls), _ptr(flags), float(min_area),
                                           _ptr(prop_off), _ptr(pb), _ptr(ps), int(best_number), float(min_proposal_area),
                                           self.num_classes, thr.shape[0], _ptr(thr), C.byref(h)), "mpn_roidb_create")
        self.h = h
        self.n_images = n
        self.serial = 0                                                # bumped by every sample: its buffers are reused
        counts = np.empty((thr.shape[0], 2, n), np.int32)
        rows = C.c_int64()
        ctx.check(ctx.lib.mpn_roidb_counts(self.h, _ptr(counts), C.byref(rows)), "mpn_roidb_counts")
        self.counts, self.n_rows = counts, int(rows.value)     # counts[set, 0 bg / 1 fg, image]
        ctx._models.append(weakref.ref(self))

    def image_rows(self, i: int):
        """image i's all_boxes (GT rows first), overlap, correspondance (1-based, 0 = none) and label rows, and its GT count"""
        n, g = C.c_int64(), C.c_int32()
        lib = self.ctx.lib
        self.ctx.check(lib.mpn_roidb_image_rows(self.h, int(i), None, None, None, None, 0, C.byref(n), C.byref(g)), "image_rows")
        b, o = np.empty((n.value, 4), np.float32), np.empty(n.value, np.float32)
        c, lab = np.empty(n.value, np.int32), np.empty(n.value, np.int32)
        self.ctx.check(lib.mpn_roidb_image_rows(self.h, int(i), _ptr(b), _ptr(o), _ptr(c), _ptr(lab), n.value, None, None), "image_rows")
        return b, o, c, lab, int(g.value)

    def rows(self, set_: int, kind: int, i: int) -> np.ndarray:
        """the bg (kind 0) or fg (kind 1) rows of image i in threshold set set_, indices into image_rows(i), row order"""
        n = C.c_int64()
        self.ctx.check(self.ctx.lib.mpn_roidb_list(self.h, set_, kind, int(i), None, 0, C.byref(n)), "mpn_roidb_list")
        out = np.empty(n.value, np.int32)
        self.ctx.check(self.ctx.lib.mpn_roidb_list(self.h, set_, kind, int(i), _ptr(out), out.size, None), "mpn_roidb_list")
        return out

    def close(self):
        if getattr(self, "h", None):
            if getattr(self.ctx, "h", None):
                self.ctx.lib.mpn_roidb_destroy(self.h)
            self.h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def sample_plan(counts_bg, counts_fg, seed: int, step: int, set_: int, n_slots: int) -> np.ndarray:
    """permuteIdx + the flips of one step (mpn_sample_plan, host): n_slots x (image, bg source, fg source, flip)"""
    from ._lib import load_library
    bg, fg = (np.ascontiguousarray(a, np.int32) for a in (counts_bg, counts_fg))
    out = np.empty((4, n_slots), np.int32)
    rc = load_library().mpn_sample_plan(_ptr(bg), _ptr(fg), bg.shape[0], int(seed) & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFF,
                                        int(set_), int(n_slots), _ptr(out[0]), _ptr(out[1]), _ptr(out[2]), _ptr(out[3]))
    if rc != 0:
        raise MpnError("sample plan: no image of the set has a bg row, or none has a fg row" if rc == -3 else "sample plan: bad arguments")
    return np.ascontiguousarray(out.T)


def integral_thresholds(K: int, bg_lo: float = 0.1, bg_hi: float = 0.5) -> Tuple[Tuple[float, float, float], ...]:
    """the threshold sets of the integral loss' K loaders (donkey.lua:38-45): loader i + 1 takes fg = bg_hi = bg_hi + i / 20
    and bg_lo, i = 0 .. K-1, as (fg, bg_lo, bg_hi) rows for RoiDB"""
    if K < 1:
        raise MpnError("integral_thresholds: K must be >= 1")
    return tuple((bg_hi + i / 20, bg_lo, bg_hi + i / 20) for i in range(int(K)))


def integral_set(seed: int, step: int, n_sets: int) -> int:
    """the threshold set of one step of integral training (mpn_integral_set, host): train.lua's
    `loaders[torch.random(#loaders)]` as a Philox draw keyed by (seed, step), 0-based"""
    from ._lib import load_library
    out = C.c_int32()
    if load_library().mpn_integral_set(int(seed) & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFF, int(n_sets), C.byref(out)) != 0:
        raise MpnError("integral_set: n_sets must be >= 1")
    return int(out.value)


def train_images_size(H0: int, W0: int, scale: float, max_size: float) -> Tuple[int, int, float]:
    """getImages' training size rule (mpn_train_images_size) -> (h, w, im_scale)"""
    from ._lib import load_library
    h, w, s = C.c_int32(), C.c_int32(), C.c_double()
    if load_library().mpn_train_images_size(int(H0), int(W0), float(scale), float(max_size), C.byref(h), C.byref(w), C.byref(s)) != 0:
        raise MpnError("train_images_size: bad arguments")
    return int(h.value), int(w.value), float(s.value)


@dataclass
class Batch:
    """One step's minibatch on the device, in buffers the RoiDB owns: valid until its next sample."""
    roidb: RoiDB
    plan: np.ndarray             # n x (image, bg source, fg source, flip)
    image_hw: np.ndarray         # n x 2: the scaled images' h, w
    rois_per_image: np.ndarray   # n
    num_classes: int             # C of the targets (dataset classes + 1)
    serial: int = 0              # which of the RoiDB's samples this is
    set: int = 0                 # the threshold set the rows were drawn from (an integral model trains head `set` on it)

    def check_current(self):
        if self.serial != self.roidb.serial:
            raise MpnError("this batch was overwritten by a later sample of its RoiDB")

    @property
    def R(self) -> int:
        return int(self.rois_per_image.sum())

    def to_host(self):
        """(images [3 x h x w fp32], boxes R x 4, labels R, targets R x 4C) copied back from the device"""
        self.check_current()
        ims = [np.empty((3, int(h), int(w)), np.float32) for h, w in self.image_hw]
        boxes, labels = np.empty((self.R, 4), np.float32), np.empty(self.R, np.int32)
        targets = np.empty((self.R, 4 * self.num_classes), np.float32)
        ptrs = (_vp * len(ims))(*[im.ctypes.data for im in ims])
        ctx = self.roidb.ctx
        ctx.check(ctx.lib.mpn_roidb_batch_host(self.roidb.h, ptrs, _ptr(boxes), _ptr(labels), _ptr(targets)), "mpn_roidb_batch_host")
        return ims, boxes, labels, targets


class BatchProviderROI:
    """fbcoco.BatchProviderROI over a RoiDB. images(i) returns image i (0-based, RoiDB order) decoded as H x W x 3 uint8 RGB.
    transformer: "ross" | "imagenet" (ModelSpec.transformer) or a CImageTransform. Per step and image slot: bg rows first,
    then fg rows, min(batch_size - fg_fraction * batch_size, n_bg) and min(fg_fraction * batch_size, n_fg) of them, each
    drawn with replacement; the draws are Philox4x32-10 keyed by (seed, step, slot, set, purpose, draw), not Torch's
    generator, so the same (seed, step, set) gives the same batch."""

    def __init__(self, roidb: RoiDB, images: Callable[[int], np.ndarray], transformer: Union[str, CImageTransform],
                 imgs_per_batch: int = 2, batch_size: int = 128, fg_fraction: float = 0.25, scale: float = 600,
                 max_size: float = 1000, seed: int = 555):
        if not 1 <= imgs_per_batch <= 32:
            raise MpnError("imgs_per_batch must lie in 1..32")
        self.roidb, self.images = roidb, images
        self.tf = transformer if isinstance(transformer, CImageTransform) else CImageTransform.of(transformer)
        self.imgs_per_batch, self.scale, self.max_size, self.seed = int(imgs_per_batch), float(scale), float(max_size), int(seed)
        fg_each = float(fg_fraction) * float(batch_size)                 # BatchProviderROI.lua:74-75, Lua numbers
        self.fg_each = int(math.floor(fg_each))                          # `for i = 1, math.min(num_max, n)`
        self.bg_each = int(math.floor(float(batch_size) - fg_each))
        self.bbox_regr = None

    def setup_data(self) -> Tuple[np.ndarray, np.ndarray]:
        """setupData: mean and std (fp32, 4 each) of the regression values of loader 1's fg rows in the first 1000 images;
        they are what ModelSpec.bbox_mean / bbox_std take, and what sample normalises the targets with"""
        mean, std = np.empty(4, np.float32), np.empty(4, np.float32)
        db = self.roidb
        db.ctx.check(db.ctx.lib.mpn_roidb_regression_stats(db.h, 0, 1000, _ptr(mean), _ptr(std)), "mpn_roidb_regression_stats")
        self.bbox_regr = (mean, std)
        return mean, std

    def plan(self, step: int, set_: int = 0) -> np.ndarray:
        db = self.roidb
        return sample_plan(db.counts[set_, 0], db.counts[set_, 1], self.seed, step, set_, self.imgs_per_batch)

    def sample(self, step: int, set_: int = 0) -> Batch:
        if self.bbox_regr is None:
            raise MpnError("sample: call setup_data() first (the targets are normalised by its mean / std)")
        db = self.roidb
        if not 0 <= set_ < len(db.thresholds):
            raise MpnError(f"sample: threshold set {set_} out of range")
        plan = self.plan(step, set_)
        ims = [np.ascontiguousarray(self.images(int(i)), np.uint8) for i in plan[:, 0]]
        for im in ims:
            if im.ndim != 3 or im.shape[2] != 3:
                raise MpnError("sample: images(i) must return H x W x 3 uint8")
        n = len(ims)
        ptrs = (_vp * n)(*[im.ctypes.data for im in ims])
        hw0 = np.ascontiguousarray([[im.shape[0], im.shape[1]] for im in ims], np.int32)
        hw = np.empty((n, 2), np.int32)
        rpi = np.empty(n, np.int32)
        mean, std = self.bbox_regr
        C_ = db.num_classes + 1
        db.ctx.check(db.ctx.lib.mpn_roidb_sample(db.h, set_, self.seed & 0xFFFFFFFFFFFFFFFF, int(step) & 0xFFFFFFFF, n, _ptr(plan), ptrs,
                                                 _ptr(hw0), C.byref(self.tf), self.scale, self.max_size, self.bg_each, self.fg_each,
                                                 _ptr(mean), _ptr(std), C_, _ptr(hw), _ptr(rpi)), "mpn_roidb_sample")
        db.serial += 1
        return Batch(db, plan, hw, rpi, C_, db.serial, int(set_))

    def sample_integral(self, step: int) -> Batch:
        """one step of integral training: the step's threshold set drawn over the RoiDB's sets (`integral_set`), then
        `sample(step, set)`; Trainer.step_batch trains the class head of that set"""
        return self.sample(step, integral_set(self.seed, step, len(self.roidb.thresholds)))

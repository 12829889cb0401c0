"""fbcoco.Tester_FRCNN mirror (Tester_FRCNN.lua:24-187) over the C ABI.

testOne with the default options is ONE library call (trunk, heads, decode, clamp, per-class gather and batched NMS on the
GPU). With the optional test-time features of the reference — iterative localisation (`test_num_iterative_loc`,
nn.SelectBoxes + detect(..., recompute_features=false), :82-89), `test_use_rbox_scores` (:91-97), bbox voting with
`test_bbox_voting_score_pow` (:118-124) — it is ONE call as well, mpn_model_test_one: every pass, nn.SelectBoxes, the join,
the NMS over the joined rows and the voting stay on the device (SURVEY 8f-2/3). `device_tail=False` (or a backend without
`test_one`, e.g. the CPU oracle of the tests) keeps them as host-side glue around the ABI calls, exactly where the
reference has them in Lua; both paths give the same bits. keepTopKPerImage / transposeBoxes (:163-187) mirror utils.lua."""
from __future__ import annotations

from typing import List, Optional

import numpy as np

from .image_detect import ImageDetect
from .modules import SelectBoxes
from . import utils as U


class _AbiBackend:
    """The calls testOne needs, bound to a Model / Context (the product path). Tests may inject another object with the
    same four methods (e.g. the CPU oracle) to check the host logic without a GPU."""

    def __init__(self, model):
        self.model, self.ctx = model, model.ctx

    def detect_nms(self, img, boxes, im_scale, W0, H0, thresh, nms_thresh):
        return self.model.detect_nms(img, boxes, im_scale, W0, H0, thresh, nms_thresh)

    def detect(self, img, boxes, im_scale, recompute_features):
        return self.model.detect(img, boxes, im_scale, recompute_features)

    def nms_batched(self, sb, offsets, thr):
        return self.ctx.nms_batched(sb, offsets, thr)

    def bbox_vote(self, nms_boxes, scored_boxes, thr):
        return U.bbox_vote(self.ctx, nms_boxes, scored_boxes, thr)

    def test_one(self, img, boxes, im_scale, W0, H0, **kw):
        return self.model.test_one(img, boxes, im_scale, W0, H0, **kw)

    def detect_nms_batch(self, ims, boxes_list, transformer, scale, max_size, thresh, nms_thresh):
        return self.model.detect_nms_batch(ims, boxes_list, transformer, scale, max_size, thresh, nms_thresh)

    def max_rois(self) -> int:
        return self.model.limits[0]


class Tester:
    def __init__(self, model, transformer, scale=None, max_size=None, nms_thresh: float = 0.3,
                 bbox_vote_thresh: float = 0.5, score_thresh: float = -1.5, bbox_voting: bool = False,
                 num_iterative_loc: int = 1, use_rbox_scores: bool = False, bbox_voting_score_pow: float = 1.0,
                 backend=None, device_tail: bool = True):
        self.detec = ImageDetect(model, transformer, scale, max_size)
        self.model = model
        self.be = backend if backend is not None else _AbiBackend(model)
        self.nms_thresh = nms_thresh                 # opt.test_nms_threshold (Tester_FRCNN.lua:28)
        self.bbox_vote_thresh = bbox_vote_thresh     # the reference reads an unset field here (SURVEY 8f-2); intended 0.5
        self.thresh = score_thresh                   # Tester_FRCNN.lua:50
        self.bbox_voting = bbox_voting               # opt.test_bbox_voting
        self.bbox_voting_score_pow = bbox_voting_score_pow
        self.num_iter = int(num_iterative_loc)       # opt.test_num_iterative_loc (Tester_FRCNN.lua:26)
        self.use_rbox_scores = bool(use_rbox_scores)
        if self.use_rbox_scores and self.num_iter < 2:
            raise ValueError("test_use_rbox_scores needs test_num_iterative_loc > 1")     # assert(#all_output > 1), :92
        self.boxselect: Optional[SelectBoxes] = None
        self.raw = None
        self.device_tail = bool(device_tail) and hasattr(self.be, "test_one")

    # ---- Tester_FRCNN.lua:54-139
    def testOne(self, im, boxes) -> List[np.ndarray]:
        """-> img_boxes: list over foreground classes of K_j x 5 [x1,y1,x2,y2,score] after NMS (and voting)."""
        boxes = np.ascontiguousarray(boxes, np.float32)
        img, im_scale = self.detec.getImages(im)
        H0, W0 = im.shape[1], im.shape[2]
        if self.num_iter == 1 and not (self.device_tail and self.bbox_voting and self.bbox_voting_score_pow == 1.0):
            scores, bboxes, keeps = self.be.detect_nms(img, boxes, im_scale, W0, H0, self.thresh, self.nms_thresh)
            self.raw = (scores, bboxes)
            out = []
            for j, k in enumerate(keeps, start=1):
                sb = np.concatenate([bboxes[k, 4 * j:4 * j + 4], scores[k, j:j + 1]], axis=1).astype(np.float32)
                out.append(self._vote(sb, scores, bboxes, j))
            return out
        if self.device_tail and (self.bbox_voting_score_pow == 1.0 or not self.bbox_voting):
            # all passes, nn.SelectBoxes, join, per-class gather, NMS and voting in one library call (mpn_model_test_one)
            output, bbox_pred, keeps, voted = self.be.test_one(
                img, boxes, im_scale, W0, H0, num_iter=self.num_iter, use_rbox_scores=self.use_rbox_scores, bbox_voting=self.bbox_voting,
                score_thresh=self.thresh, nms_thr=self.nms_thresh, vote_thr=self.bbox_vote_thresh, vote_score_pow=self.bbox_voting_score_pow)
            self.raw = (output, bbox_pred)
            if voted is not None:
                return voted
            return [np.concatenate([bbox_pred[k, 4 * j:4 * j + 4], output[k, j:j + 1]], axis=1).astype(np.float32) for j, k in enumerate(keeps, start=1)]
        # ---- iterative localisation: every pass re-uses the cached trunk features (recompute_features = false)
        all_output, all_bbox = [], []
        output, bbox_pred = self.be.detect(img, boxes, im_scale, True)
        bbox_pred = self._clamp(bbox_pred, W0, H0)                                          # :75-78 (first pass only, as the reference)
        all_output.append(output); all_bbox.append(bbox_pred)
        for _ in range(2, self.num_iter + 1):
            self.boxselect = self.boxselect or SelectBoxes()
            new_boxes = self.boxselect.forward([output, bbox_pred])
            output, bbox_pred = self.be.detect(None, new_boxes, im_scale, False)
            all_output.append(output); all_bbox.append(bbox_pred)
        if self.use_rbox_scores:        # scores of pass n+1 for the boxes of pass n: one pass worth of boxes is lost (:91-97)
            all_output.pop(0)
            all_bbox.pop()
        output = U.joinTable(all_output, 0)
        bbox_pred = U.joinTable(all_bbox, 0)
        self.raw = (output, bbox_pred)
        num_classes = output.shape[1] - 1
        segs, offs = [], [0]
        for j in range(1, num_classes + 1):
            sel = output[:, j] > self.thresh
            sb = np.concatenate([bbox_pred[sel, 4 * j:4 * j + 4], output[sel, j:j + 1]], axis=1).astype(np.float32)
            segs.append(sb); offs.append(offs[-1] + sb.shape[0])
        allsb = np.concatenate(segs, 0) if offs[-1] else np.zeros((0, 5), np.float32)
        keeps = self.be.nms_batched(allsb, offs, self.nms_thresh) if offs[-1] else [np.zeros(0, np.int32)] * num_classes
        out = []
        for j in range(1, num_classes + 1):
            sb = segs[j - 1][np.asarray(keeps[j - 1], np.int64)] if segs[j - 1].shape[0] else segs[j - 1]
            out.append(self._vote(sb, output, bbox_pred, j))
        return out

    def testMany(self, ims, boxes_list) -> List[List[np.ndarray]]:
        """[testOne(im, boxes) for each image], bit for bit. Where testOne takes the single detect + NMS path (one
        localisation pass, no voting), consecutive images whose proposals fit the model's max_rois go through one
        batched library call (mpn_model_detect_nms_batch); otherwise, and for a backend without it, image by image."""
        if len(ims) != len(boxes_list):
            raise ValueError("testMany: one box array per image")
        boxes_list = [np.ascontiguousarray(b, np.float32).reshape(-1, 4) for b in boxes_list]
        if self.num_iter != 1 or self.bbox_voting or not hasattr(self.be, "detect_nms_batch"):
            return [self.testOne(im, b) for im, b in zip(ims, boxes_list)]
        cap = self.be.max_rois()
        out: List[List[np.ndarray]] = []
        i = 0
        while i < len(ims):
            j, n = i, 0
            while j < len(ims) and n + boxes_list[j].shape[0] <= cap:
                n += boxes_list[j].shape[0]
                j += 1
            if j == i:                      # one image over max_rois: testOne refuses it as it does today
                out.append(self.testOne(ims[i], boxes_list[i]))
                i += 1
                continue
            res = self.be.detect_nms_batch(ims[i:j], boxes_list[i:j], self.detec.image_transformer, self.detec.scale[0],
                                           self.detec.max_size, self.thresh, self.nms_thresh)
            for scores, bboxes, keeps in res:
                out.append([np.concatenate([bboxes[k, 4 * c:4 * c + 4], scores[k, c:c + 1]], axis=1).astype(np.float32)
                            for c, k in enumerate(keeps, start=1)])
                self.raw = (scores, bboxes)
            i = j
        return out

    @staticmethod
    def _clamp(bbox_pred, W0, H0):
        b = np.array(bbox_pred, np.float32, copy=True).reshape(-1, 2)
        np.clip(b[:, 0], 1, W0, out=b[:, 0]); np.clip(b[:, 1], 1, H0, out=b[:, 1])
        return b.reshape(bbox_pred.shape)

    def _vote(self, nms_boxes, scores, bboxes, j):
        if not self.bbox_voting or not len(nms_boxes):
            return nms_boxes
        sel = scores[:, j] > self.thresh
        allsb = np.concatenate([bboxes[sel, 4 * j:4 * j + 4], scores[sel, j:j + 1]], axis=1).astype(np.float32)
        allsb[:, 4] = np.power(allsb[:, 4], np.float32(self.bbox_voting_score_pow))           # :119-121
        return self.be.bbox_vote(nms_boxes, allsb, self.bbox_vote_thresh)

    # ---- Tester_FRCNN.lua:141-187 (the dataset loop itself stays with the caller: no dataset code here)
    @staticmethod
    def keepTopKPerImage(aboxes_t: List[List[np.ndarray]], k: int = 100):
        return [U.keep_top_k(per_img, k)[0] for per_img in aboxes_t]

    def transposeBoxes(self, aboxes_t: List[List[np.ndarray]]):
        return U.transposeBoxes(aboxes_t, len(aboxes_t[0]) if aboxes_t else 0)

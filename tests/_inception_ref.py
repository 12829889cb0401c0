"""fp64 restatement of model:forward / ImageDetect:detect / Tester_FRCNN:testOne for graphs with Inception-v3's layers:
convolutions with their own horizontal pad (Layer.padw), windowed average pools (include- or exclude-pad, as
nn.SpatialAveragePooling), and branches that write channel slices of one concatenation slot (Layer.out_c_off /
out_c_total, what nn.Concat(2) / nn.DepthConcat(2) return). Everything else follows oracle/graphs.py and the C
restatement in oracle/ref.py (ROI pooling, softmax, decode, clamp, NMS). The dense layers run in torch float64, on
cuda when it is there (the full-size graph is two TFLOP per 1000 ROIs), so the result is the exact product up to fp64."""
from __future__ import annotations

import numpy as np
import torch
import torch.nn.functional as F

from oracle import ref as O
from multipathnet_b200 import models
from multipathnet_b200._lib import (Head, Layer, ModelSpec, Tower, MPN_LAYER_AVGPOOL, MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_CONV,
                                    MPN_LAYER_FLATTEN, MPN_LAYER_MAXPOOL)


def _dev():
    return torch.device("cuda") if torch.cuda.is_available() else torch.device("cpu")


def _t(a, dev=None):
    return torch.as_tensor(np.ascontiguousarray(a, dtype=np.float64), device=dev or _dev())


def layer(L, x, weights, res=None):
    """one layer on NCHW float64 x (2-D after a FLATTEN)"""
    if L.kind == MPN_LAYER_CONV:
        w, b = _t(weights[L.weight], x.device), (_t(weights[L.bias], x.device) if L.bias >= 0 else None)
        if x.dim() == 2:
            y = F.linear(x, w.reshape(L.cout, -1), b)
        else:
            y = F.conv2d(x, w.reshape(L.cout, L.cin, L.kh, L.kw), b, stride=L.stride, padding=(L.pad, L.padw))
        if res is not None:
            y = y + res
        return F.relu(y) if L.relu else y
    if L.kind == MPN_LAYER_MAXPOOL:
        return F.max_pool2d(x, (L.kh, L.kw), L.stride, L.pad, ceil_mode=bool(L.ceil_mode))
    if L.kind == MPN_LAYER_AVGPOOL_WIN:
        return F.avg_pool2d(x, (L.kh, L.kw), L.stride, L.pad, ceil_mode=bool(L.ceil_mode), count_include_pad=not L.exclude_pad)
    if L.kind == MPN_LAYER_AVGPOOL:
        return x.mean(dim=(2, 3))
    if L.kind == MPN_LAYER_FLATTEN:
        return x.reshape(x.shape[0], -1)
    raise ValueError(L.kind)


def run_layers(layers, slots, weights):
    """slots: {slot: tensor}; a concatenation slot is assembled from its branches in place"""
    for L in layers:
        y = layer(L, slots[L.in_slot], weights, slots[L.residual_slot] if L.residual_slot >= 0 else None)
        if L.out_c_total > 0:
            if L.out_slot not in slots:
                slots[L.out_slot] = torch.full((y.shape[0], L.out_c_total) + tuple(y.shape[2:]), float("nan"), dtype=y.dtype,
                                               device=y.device)
            slots[L.out_slot][:, L.out_c_off:L.out_c_off + y.shape[1]] = y
        else:
            slots[L.out_slot] = y
    return slots


def trunk_forward(spec, image_chw):
    with torch.no_grad():
        return run_layers(spec.trunk_layers, {0: _t(image_chw)[None]}, spec.weights)


def pooled_rows(spec, trunk_slots, rois, tower=0):
    """the ROI-pooled rows of a tower (fp32, the C restatement of inn.ROIPooling): R x C x PH x PW"""
    t = spec.towers[tower]
    out = []
    for slot, scale in t.levels:
        fm = trunk_slots[slot].float().cpu().numpy()
        out.append(O.roi_pool(fm, np.ascontiguousarray(rois, np.float32), t.pooled_w, t.pooled_h, np.float32(scale), spec.roi_variant))
    return np.concatenate(out, axis=1)


def heads_forward(spec, trunk_slots, rois, pooled=None):
    """(cls logits or probabilities, float64; bbox after BBoxNorm, fp32); single-tower graphs, region 0 (Inception-v3)"""
    assert len(spec.towers) == 1 and spec.towers[0].region == 0 and not spec.towers[0].normalize
    t = spec.towers[0]
    with torch.no_grad():
        x = pooled if pooled is not None else pooled_rows(spec, trunk_slots, rois)
        feat = run_layers(t.layers, {0: _t(x)}, spec.weights)[t.out_slot].reshape(x.shape[0], -1)
        cls = [F.linear(feat[:, h.col_begin:h.col_begin + h.col_len], _t(spec.weights[h.weight]), _t(spec.weights[h.bias]))
               for h in spec.cls_heads]
        hb = spec.bbox_head
        bbox = F.linear(feat[:, hb.col_begin:hb.col_begin + hb.col_len], _t(spec.weights[hb.weight]), _t(spec.weights[hb.bias]))
        bbox = bbox.cpu().numpy()
        if len(cls) > 1:
            c = np.mean(np.stack([torch.softmax(c, 1).cpu().numpy() for c in cls], 0), axis=0)
        else:
            c = cls[0].cpu().numpy()
        if spec.has_bbox_norm:
            bbox = O.bbox_norm(bbox.astype(np.float32), spec.bbox_mean, spec.bbox_std)
        return c, bbox


def detect(spec, image_chw, boxes, im_scale):
    """ImageDetect:detect after getImages: (scores R x C, bboxes R x 4C), fp32 at the end (softmax, decode: oracle/ref.py)"""
    rois = O.project_rois(boxes, np.float32(im_scale))
    cls, bbox = heads_forward(spec, trunk_forward(spec, image_chw), rois)
    bboxes = O.convert_from(bbox.astype(np.float32), boxes)
    c = cls.astype(np.float32)
    scores = c if (spec.no_softmax or len(spec.cls_heads) > 1) else O.softmax(c)
    return scores, bboxes


def test_one(spec, image_chw, boxes, im_scale, W0, H0, score_thresh=-1.5, nms_thr=0.3):
    scores, bboxes = detect(spec, image_chw, boxes, im_scale)
    bboxes = O.clamp_boxes(bboxes, W0, H0)
    keeps = []
    for j in range(1, scores.shape[1]):
        sel = np.nonzero(scores[:, j] > score_thresh)[0]
        sb = np.concatenate([bboxes[sel, 4 * j:4 * j + 4], scores[sel, j:j + 1]], 1).astype(np.float32)
        keeps.append(sel[O.nms(sb, nms_thr)].astype(np.int32))
    return scores, bboxes, keeps


def tiny_spec(seed=3, xp=1):
    """one of each block kind at narrow widths: a K-tail Cin (40, 24), include- and exclude-pad pools, a nested concat"""
    W = models._W(seed)
    g = models._Graph(W, 1)
    x = g.conv(0, 3, 32, 3, 3, stride=2, gain=0.5)
    x = g.conv(x, 32, 40, 3, 3, ph=1, pw=1)
    o = g.slot()
    g.conv(x, 40, 16, 1, 1, dst=(o, 0, 64))
    g.conv(g.conv(x, 40, 24, 1, 1), 24, 16, 1, 7, pw=3, dst=(o, 16, 64))
    g.conv(g.conv(x, 40, 16, 1, 1), 16, 16, 7, 1, ph=3, dst=(o, 32, 64))
    g.conv(g.pool(MPN_LAYER_AVGPOOL_WIN, x, 3, 1, 1, exclude_pad=xp), 40, 16, 1, 1, dst=(o, 48, 64))
    o2 = g.slot()
    g.conv(o, 64, 32, 3, 3, stride=2, dst=(o2, 0, 96))
    g.pool(MPN_LAYER_MAXPOOL, o, 3, 2, 0, dst=(o2, 32, 96))
    t = models._Graph(W, 1)
    o3 = t.slot()
    b = t.conv(0, 96, 32, 1, 1)
    t.conv(b, 32, 16, 1, 3, pw=1, dst=(o3, 0, 64))
    t.conv(b, 32, 16, 3, 1, ph=1, dst=(o3, 16, 64))
    t.conv(t.pool(MPN_LAYER_AVGPOOL_WIN, 0, 3, 1, 1, exclude_pad=1 - xp), 96, 32, 1, 1, dst=(o3, 32, 64))
    out = t.slot()
    t.layers.append(Layer(MPN_LAYER_AVGPOOL, o3, out))
    tower = Tower(region=0, levels=[(o2, 1.0 / 8)], pooled_w=5, pooled_h=5, normalize=0, layers=t.layers, out_slot=out)
    wc, bc = W.linear(5, 64, std=0.1, zero_bias=True)
    wb, bb = W.linear(20, 64, std=0.01, zero_bias=True)
    return ModelSpec(name="inception_tiny", trunk_layers=g.layers, towers=[tower], cls_heads=[Head(0, 64, 5, wc, bc)],
                     bbox_head=Head(0, 64, 20, wb, bb), num_classes=5, weights=W.arrays, transformer="inception", taps={"top": o2})


def evaluate_nn(m, x):
    """a torch nn graph (T7Object tree) evaluated module by module in eval mode, fp32 on the CPU: tests/_nn_interp.py
    plus what inceptionv3.lua adds (nn.Concat / nn.DepthConcat(2), a pad per axis, windowed SpatialAveragePooling)"""
    from multipathnet_b200.t7 import _base, _children
    import _nn_interp as NI
    b, kids = _base(m.typename), _children(m)
    if b in ("Sequential", "NoBackprop"):
        for c in kids:
            x = evaluate_nn(c, x)
        return x
    if b == "ConcatTable":
        return [evaluate_nn(c, x) for c in kids]
    if b == "ParallelTable":
        return [evaluate_nn(c, xi) for c, xi in zip(kids, x)]
    if b in ("Concat", "DepthConcat"):
        return torch.cat([evaluate_nn(c, x) for c in kids], dim=int(m.dimension) - 1)
    if b in ("SpatialConvolution", "SpatialConvolutionMM"):
        bias = None if m.get("bias") is None else NI._t(m.bias)
        return F.conv2d(x, NI._t(m.weight), bias, stride=(int(m.dH), int(m.dW)), padding=(int(m.get("padH", 0)), int(m.get("padW", 0))))
    if b == "SpatialAveragePooling":
        return F.avg_pool2d(x, (int(m.kH), int(m.kW)), (int(m.dH), int(m.dW)), (int(m.get("padH", 0)), int(m.get("padW", 0))),
                            ceil_mode=bool(m.get("ceil_mode", False)), count_include_pad=bool(m.get("count_include_pad", True)))
    assert b not in ("DataParallelTable", "ModelParallelTable", "ModeSwitch"), b
    return NI.evaluate(m, x)

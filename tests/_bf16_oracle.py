"""The bf16 inference numerics (mpn_ctx_set_option "bf16") restated on the CPU: the graphs of oracle/graphs.py with the
input and the weight of every convolution / Linear rounded to bf16 (round to nearest even) before the fp32 op, except the
first trunk layer (the one that reads the image, slot 0), which keeps its fp32-faithful kernels on the device.

That is exactly the device's operand rounding: a layer's A operand is the hi plane hi = rn_bf16(x) of the stored fp32
value x, its B operand the hi plane of the fp32 weight. rn_bf16 is monotonic, so it commutes with the max pools between
the convolutions. Residual inputs, ROI pooling, the L2 normalisation and everything after the heads stay fp32, as on
the device (they read hi + lo, or fp32).

fp64_sums=True sums every convolution / Linear in fp64 before rounding to fp32: the same bf16 operands, another
summation order. How far that moves the outputs is the order sensitivity of the graph in this mode (a reordered fp32
sum flips the bf16 rounding of ~1e-4 of a layer's outputs, and the graph amplifies those one-ulp changes); no oracle
can pin the device closer than that."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import graphs as G, ref as O


def rn_bf16(t):
    """fp32 -> nearest bf16 (ties to even) -> fp32"""
    return t.to(torch.bfloat16).to(torch.float32)


def _conv2d(x, w, b, fp64, **k):
    if not fp64:
        return F.conv2d(x, w, b, **k)
    return F.conv2d(x.double(), w.double(), None if b is None else b.double(), **k).float()


def _linear(x, w, b, fp64):
    if not fp64:
        return F.linear(x, w, b)
    return F.linear(x.double(), w.double(), None if b is None else b.double()).float()


def _run_layers(layers, slots, weights, trunk, fp64=False):
    for L in layers:
        x = slots[L.in_slot]
        if L.kind == G.CONV:
            w = G._t(weights[L.weight])
            if not (trunk and L.in_slot == 0):
                x, w = rn_bf16(x), rn_bf16(w)
            b = G._t(weights[L.bias]) if L.bias >= 0 else None
            if x.dim() == 2:
                y = _linear(x, w.reshape(L.cout, -1), b, fp64)
            else:
                g = getattr(L, "groups", 1)
                y = _conv2d(x, w.reshape(L.cout, L.cin // g, L.kh, L.kw), b, fp64, stride=L.stride, padding=L.pad, groups=g)
            if L.residual_slot >= 0:
                y = y + slots[L.residual_slot]
            if L.relu:
                y = F.relu(y)
            slots[L.out_slot] = y
        else:
            G._run_layers([L], slots, weights)
    return slots


def trunk_forward(spec, image_chw, fp64_sums=False):
    with torch.no_grad():
        return _run_layers(spec.trunk_layers, {0: G._t(image_chw)[None]}, spec.weights, trunk=True, fp64=fp64_sums)


def heads_forward(spec, trunk_slots, rois, fp64_sums=False):
    """graphs.heads_forward with bf16 operands in the towers and the heads"""
    rois = np.ascontiguousarray(rois, np.float32)
    R = rois.shape[0]
    with torch.no_grad():
        fov = O.foveal(rois).reshape(R, 4, 5) if any(t.region > 0 for t in spec.towers) else None
        feats = []
        for t in spec.towers:
            reg = rois if t.region == 0 else np.ascontiguousarray(fov[:, t.region, :])
            pooled = []
            for slot, scale in t.levels:
                p = O.roi_pool(trunk_slots[slot].numpy(), reg, t.pooled_w, t.pooled_h, np.float32(scale), spec.roi_variant)
                if t.normalize:
                    p = O.l2_normalize(p.reshape(R, -1)).reshape(p.shape)
                pooled.append(p)
            x = np.concatenate(pooled, axis=1)
            if t.normalize:
                x = x * np.float32(1000.0)
            slots = _run_layers(t.layers, {0: G._t(x)}, spec.weights, trunk=False, fp64=fp64_sums)
            feats.append(slots[t.out_slot].reshape(R, -1))
        cat = torch.cat(feats, dim=1)

        def linear(h):
            return _linear(rn_bf16(cat[:, h.col_begin:h.col_begin + h.col_len]), rn_bf16(G._t(spec.weights[h.weight])),
                           G._t(spec.weights[h.bias]), fp64_sums)
        cls = [linear(h) for h in spec.cls_heads]
        bbox = linear(spec.bbox_head).numpy()
        if len(cls) > 1:
            c = np.mean(np.stack([O.softmax(c.numpy()) for c in cls], 0), axis=0, dtype=np.float32)
        else:
            c = cls[0].numpy()
        if spec.has_bbox_norm:
            bbox = O.bbox_norm(bbox, spec.bbox_mean, spec.bbox_std)
        return c, bbox


def detect(spec, image_chw, boxes, im_scale, fp64_sums=False):
    rois = O.project_rois(boxes, np.float32(im_scale))
    cls, bbox = heads_forward(spec, trunk_forward(spec, image_chw, fp64_sums), rois, fp64_sums)
    bboxes = O.convert_from(bbox, boxes)
    scores = cls if (spec.no_softmax or len(spec.cls_heads) > 1) else O.softmax(cls)
    return scores, bboxes


def test_one(spec, image_chw, boxes, im_scale, W0, H0, fp64_sums=False):
    """detect + clamp (the keep lists are checked against nms.c on the device's own outputs, not here)"""
    scores, bboxes = detect(spec, image_chw, boxes, im_scale, fp64_sums)
    return scores, O.clamp_boxes(bboxes, W0, H0)

"""The fp8 inference numerics (mpn_ctx_set_option "fp8") restated on the CPU: the graphs of oracle/graphs.py with the
fp8 operand rule applied to every convolution / Linear the mode covers: every trunk layer but the first (the one that
reads the image, slot 0) and every tower layer. The cls / bbox heads keep fp32 operands, as the device's three-product
default does.

Operand rule (csrc/fp8_e4m3.cuh): h = rn_bf16(x) (the hi plane), q = rn_e4m3(2^e * h) with e the largest integer such that
max|h| * 2^e <= 448, clamped to [-60, 60] (0 for an all-zero group); one e per output channel of a weight and one per sample
of an activation (dim 0: the image in the trunk, the ROI in the towers). The layer computes sum(q_a * q_w) * 2^-(e_a + e_w)
+ bias. Rounding uses torch.float8_e4m3fn (round to nearest even on the CPU; NaN above 464, which the rule never reaches).

fp64_sums=True sums in fp64 before rounding to fp32: the same operands, another summation order, i.e. the order sensitivity
of the graph in this mode (see tests/_bf16_oracle.py). That sensitivity understates what the device can reach: the e4m3
tensor-core product keeps fewer bits than an fp32 sum (measured 3-7e-5 normwise per layer on an H100, DESIGN 4), and a
change that size flips the e4m3 rounding of the next layer's operands far more often than a reordered fp32 sum does.
sum_noise=eps adds to every fp8 layer's sum, before the scale, seeded Gaussian noise of standard deviation eps * max|sum|:
the graph's sensitivity to an accumulator of the device's precision."""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import graphs as G, ref as O


def scale_exponents(h):
    """per dim-0 group of h (fp32): the largest e with max|h| * 2^e <= 448, clamped to [-60, 60]; 0 for max|h| = 0"""
    amax = h.abs().reshape(h.shape[0], -1).amax(dim=1).double()
    m, k = torch.frexp(amax)                                  # amax = m * 2^k, m in [0.5, 1)
    e = torch.where(m <= 0.875, 9 - k, 8 - k).clamp(-60, 60)
    return torch.where(amax > 0, e, torch.zeros_like(e)).to(torch.int64)


def quantize(x):
    """(codes as fp32 values, exponents) of x under the operand rule, groups along dim 0"""
    h = x.to(torch.bfloat16).to(torch.float32)
    e = scale_exponents(h)
    sc = torch.ldexp(torch.ones_like(e, dtype=torch.float32), e.to(torch.float32)).reshape(-1, *([1] * (h.dim() - 1)))
    q = (h * sc).to(torch.float8_e4m3fn).to(torch.float32)
    return q, e


def _scaled(y, ea, ew, b):
    """y * 2^-(e_a[sample] + e_w[channel]) (exact), then + bias"""
    shape = [1] * y.dim()
    ea = ea.reshape(-1, *shape[1:]); ew = ew.reshape(1, -1, *shape[2:])
    y = y * torch.ldexp(torch.ones(1), -(ea + ew).to(torch.float32))
    return y if b is None else y + b.reshape(1, -1, *shape[2:])


_NOISE = {"eps": 0.0, "gen": None}


def fp8_layer(x, w, b, fp64, **k):
    """conv (x 4-D) or Linear (x 2-D) with fp8 operands; w [Cout][...]"""
    qx, ea = quantize(x)
    qw, ew = quantize(w)
    if fp64:
        qx, qw = qx.double(), qw.double()
    y = F.linear(qx, qw.reshape(qw.shape[0], -1)) if x.dim() == 2 else F.conv2d(qx, qw, **k)
    y = y.float()
    if _NOISE["eps"] > 0:
        y = y + torch.randn(y.shape, generator=_NOISE["gen"]) * (_NOISE["eps"] * float(y.abs().max()))
    return _scaled(y, ea, ew, b)


def _run_layers(layers, slots, weights, trunk, fp64=False):
    for L in layers:
        x = slots[L.in_slot]
        if L.kind == G.CONV:
            w = G._t(weights[L.weight])
            b = G._t(weights[L.bias]) if L.bias >= 0 else None
            if trunk and L.in_slot == 0:
                y = F.conv2d(x, w.reshape(L.cout, L.cin, L.kh, L.kw), b, stride=L.stride, padding=L.pad)
            elif x.dim() == 2:
                y = fp8_layer(x, w.reshape(L.cout, -1), b, fp64)
            else:
                y = fp8_layer(x, w.reshape(L.cout, L.cin, L.kh, L.kw), b, fp64, stride=L.stride, padding=L.pad)
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
    """graphs.heads_forward with fp8 operands in the towers; fp32 heads"""
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
            x, w, b = cat[:, h.col_begin:h.col_begin + h.col_len], G._t(spec.weights[h.weight]), G._t(spec.weights[h.bias])
            if fp64_sums:
                return F.linear(x.double(), w.double(), b.double()).float()
            return F.linear(x, w, b)
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


def test_one(spec, image_chw, boxes, im_scale, W0, H0, fp64_sums=False, sum_noise=0.0):
    """detect + clamp (the keep lists are checked against nms.c on the device's own outputs, not here)"""
    _NOISE["eps"], _NOISE["gen"] = sum_noise, torch.Generator().manual_seed(0)
    try:
        scores, bboxes = detect(spec, image_chw, boxes, im_scale, fp64_sums)
    finally:
        _NOISE["eps"] = 0.0
    return scores, O.clamp_boxes(bboxes, W0, H0)

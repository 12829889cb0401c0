"""CPU emulation of the engine's bf16-split arithmetic on the default workload (no GPU): how far can the number of bf16
products per MAC be cut, layer by layer, before scores / boxes leave the 1e-3 end-to-end tolerance?

Every conv / Linear input x and weight w is split like the engine does (hi = bf16(x), lo = bf16(x - hi)); a layer then
accumulates a chosen subset of {hi*hi, lo*hi, hi*lo} in fp32 (PyTorch CPU).  "3" = what the engine issues today,
"w1" = drop hi_x*lo_w (weights effectively bf16), "x1" = drop lo_x*hi_w (activations effectively bf16), "1" = hi*hi only;
"f16w" / "f16x" / "f16x3" = the same with fp16 parts (2 / 2 / 3 products), "tf32" = one kind::tf32 pass.
Activations between layers are re-split (hi + lo = 16 mantissa bits), as in HBM.
TEST / ANALYSIS TOOL: imports oracle/ (reference-side arithmetic for the non-GEMM ops); not product code.

  python tools/split_emulation.py [--small]     # --small: 300x400 image, 300 ROIs (about a minute on 8 cores)
"""
import argparse
import os
import sys
import time

import numpy as np
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from multipathnet_b200 import models, workloads as wl          # noqa: E402
from multipathnet_b200._lib import MPN_LAYER_CONV, MPN_LAYER_FLATTEN, MPN_LAYER_MAXPOOL   # noqa: E402
from oracle import graphs as G, ref as O                        # noqa: E402


def split(t):
    hi = t.to(torch.bfloat16).to(torch.float32)
    lo = (t - hi).to(torch.bfloat16).to(torch.float32)
    return hi, lo


def split16(t):
    hi = t.to(torch.float16).to(torch.float32)
    lo = (t - hi).to(torch.float16).to(torch.float32)
    return hi, lo


def tf32(t):                                   # round to a 10-bit mantissa (tensor-core tf32 operand precision)
    i = t.contiguous().view(torch.int32)
    i = (i + 0x00000FFF + ((i >> 13) & 1)) & ~0x00001FFF
    return i.view(torch.float32)


def products(x, w, op, mode):
    """the fp32 sum of the operand-part products a mode issues"""
    if mode == "tf32":                         # one pass at half the bf16 rate = the cost of 2 bf16 products
        return op(tf32(x), tf32(w))
    if mode in ("f16w", "f16x", "f16x3"):      # fp16 parts (11-bit mantissa each; needs |x| < 65504)
        xh, xl = split16(x)
        wh, wl_ = split16(w)
        y = op(xh, wh)
        if mode in ("f16w", "f16x3"):
            y = y + op(xl, wh)
        if mode in ("f16x", "f16x3"):
            y = y + op(xh, wl_)
        return y
    xh, xl = split(x)
    wh, wl_ = split(w)
    y = op(xh, wh)
    if mode in ("3", "w1"):
        y = y + op(xl, wh)
    if mode in ("3", "x1"):
        y = y + op(xh, wl_)
    return y


def layer(x, w, b, L, mode, linear):
    op = (lambda a, ww: F.linear(a, ww)) if linear else (lambda a, ww: F.conv2d(a, ww, None, stride=L.stride, padding=L.pad))
    y = products(x, w, op, mode)
    y = y + (b if linear else b.view(1, -1, 1, 1))
    if L.relu:
        y = F.relu(y)
    h, l = split(y)
    return h + l


def run_layers(layers, x, weights, modes, names, prefix):
    slots = {0: x}
    for i, L in enumerate(layers):
        x = slots[L.in_slot]
        if L.kind == MPN_LAYER_CONV:
            w = torch.from_numpy(weights[L.weight])
            b = torch.from_numpy(weights[L.bias])
            lin = x.dim() == 2
            name = f"{prefix}{i}"
            names.append(name)
            y = layer(x, w.reshape(L.cout, -1) if lin else w.reshape(L.cout, L.cin, L.kh, L.kw), b, L, modes(name), lin)
        elif L.kind == MPN_LAYER_MAXPOOL:
            y = F.max_pool2d(x, L.kh, L.stride, L.pad, ceil_mode=bool(L.ceil_mode))
        elif L.kind == MPN_LAYER_FLATTEN:
            y = x.reshape(x.shape[0], -1)
        else:
            raise ValueError(L.kind)
        slots[L.out_slot] = y
    return slots


def emulate(spec, img, boxes, modes):
    names = []
    with torch.no_grad():
        ts = run_layers(spec.trunk_layers, torch.from_numpy(img)[None], spec.weights, modes, names, "conv")
        t = spec.towers[0]
        rois = O.project_rois(boxes, np.float32(1.0))
        pooled = O.roi_pool(ts[t.levels[0][0]].numpy(), rois, t.pooled_w, t.pooled_h, np.float32(t.levels[0][1]), spec.roi_variant)
        hs = run_layers(t.layers, torch.from_numpy(pooled), spec.weights, modes, names, "fc")
        feat = hs[t.out_slot]
        outs = []
        for nm, hd in (("cls", spec.cls_heads[0]), ("bbox", spec.bbox_head)):
            names.append(nm)
            y = products(feat, torch.from_numpy(spec.weights[hd.weight]), F.linear, modes(nm))
            outs.append((y + torch.from_numpy(spec.weights[hd.bias])).numpy())
    cls, bbox = outs
    bbox = O.bbox_norm(bbox, spec.bbox_mean, spec.bbox_std)
    return O.softmax(cls), O.convert_from(bbox, boxes), names


def rel(a, b):
    return float(np.abs(a.astype(np.float64) - b).max() / np.abs(b).max())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--small", action="store_true")
    a = ap.parse_args()
    H, W, R = (300, 400, 300) if a.small else (600, 800, 1000)
    spec = models.vgg16_fast_rcnn(21, seed=1234)
    img = wl.transform(wl.raw_image(H, W, 2), spec.transformer)
    boxes = wl.random_boxes(R, H, W, 2)
    t0 = time.time()
    ref_s, ref_b = G.detect(spec, img, boxes, 1.0)
    print(f"# fp32 oracle: {time.time() - t0:.1f} s; {H}x{W}, {R} ROIs", flush=True)
    trunk = [f"conv{i}" for i, L in enumerate(spec.trunk_layers) if L.kind == MPN_LAYER_CONV]
    configs = {
        "all 3 products (engine today)": {},
        "fc6 w1": {"fc1": "w1"}, "fc6 x1": {"fc1": "x1"}, "fc6 1": {"fc1": "1"},
        "fc6+fc7 w1": {"fc1": "w1", "fc2": "w1"}, "fc6+fc7 x1": {"fc1": "x1", "fc2": "x1"},
        "fc6+fc7+heads w1": {"fc1": "w1", "fc2": "w1", "cls": "w1", "bbox": "w1"},
        "trunk w1": {n: "w1" for n in trunk}, "trunk x1": {n: "x1" for n in trunk},
        "fc6 f16w (2 products, fp16 parts, weights one fp16)": {"fc1": "f16w"},
        "fc6+fc7 f16w": {"fc1": "f16w", "fc2": "f16w"}, "fc6+fc7 f16x": {"fc1": "f16x", "fc2": "f16x"},
        "trunk f16w": {n: "f16w" for n in trunk}, "everything f16w": "f16w", "everything f16x3": "f16x3",
        "fc6 tf32 (1 pass at half rate)": {"fc1": "tf32"}, "everything tf32": "tf32",
        "everything w1": "w1", "everything x1": "x1", "everything 1 (plain bf16)": "1",
    }
    print("| products per MAC | scores rel err | boxes rel err |\n|---|---|---|")
    for name, cfg in configs.items():
        modes = (lambda n, c=cfg: c) if isinstance(cfg, str) else (lambda n, c=cfg: c.get(n, "3"))
        t0 = time.time()
        s, b, names = emulate(spec, img, boxes, modes)
        print(f"| {name} | {rel(s, ref_s):.2e} | {rel(b, ref_b):.2e} |   # {time.time() - t0:.0f} s", flush=True)


if __name__ == "__main__":
    main()

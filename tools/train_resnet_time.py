"""Times the fixed-batch-norm ResNet training step (layer2 .. layer4 and the heads, the README's `model=resnet` recipe)
on the recipe's minibatch (scale 800, max_size 1000, 4 images, 64 ROIs per image): resnet18_fast_rcnn(81, integral_k=6,
fixed_bn=True) and resnet50_fast_rcnn(81, integral_k=6, fixed_bn=True), the trunk training from layer2. Per model, CUDA
events around --iters back-to-back steps after --warmup steps, then the library's phase events (mpn_model_train_phase_ms:
trunks + ROI pooling, per-ROI forward + criteria, backward, update), medians over --iters more steps, and the device
memory in use after the steps (cudaMemGetInfo: the library's own allocations are not torch's). The backward's dgrad and
wgrad FLOPs are counted from the shapes here, over the measured backward phase. Writes profiles/h100_train_resnet.json
(or --out) with the GPU's name and power limit read in the same run.
    python tools/train_resnet_time.py [--out FILE] [--iters 20] [--warmup 3]"""
import argparse
import ctypes as Cc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import MPN_LAYER_AVGPOOL, MPN_LAYER_CONV
from train_time import gpu_info

SIZES = ((800, 1000), (800, 1000), (666, 1000), (800, 800))
PER_IMAGE = 64
SEED = 555


def backward_flops(spec, sizes, R):
    """dgrad + wgrad FLOPs of one step's backward (2 * MACs), counted from the shapes: each trained convolution's wgrad,
    its dgrad unless its input is the frozen part's output, per image for the trunk range and per ROI for the tower; the
    heads' dW and their dX into the tower's columns"""
    k0 = spec.trunk_train_from
    frozen = spec.trunk_layers[k0].in_slot
    fl = {"trunk_dw": 0.0, "trunk_dx": 0.0, "tower_dw": 0.0, "tower_dx": 0.0, "heads": 0.0}
    for H, W in sizes:
        shp = {0: (H, W)}
        for L in spec.trunk_layers:
            h, w = shp[L.in_slot]
            ho, wo = ((h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1) if L.kind == MPN_LAYER_CONV else \
                (models._pool_out(h, L.kh, L.stride, L.pad, L.ceil_mode), models._pool_out(w, L.kw, L.stride, L.pad, L.ceil_mode))
            shp[L.out_slot] = (ho, wo)
        for L in spec.trunk_layers[k0:]:
            ho, wo = shp[L.out_slot]
            mac = L.cin * L.cout * L.kh * L.kw * ho * wo
            fl["trunk_dw"] += 2.0 * mac
            if L.in_slot != frozen:
                fl["trunk_dx"] += 2.0 * mac
    t = spec.towers[0]
    shp = {0: (t.pooled_h, t.pooled_w)}
    for L in t.layers:
        h, w = shp[L.in_slot]
        if L.kind == MPN_LAYER_AVGPOOL:
            shp[L.out_slot] = (1, 1)
            continue
        ho, wo = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1
        shp[L.out_slot] = (ho, wo)
        mac = R * L.cin * L.cout * L.kh * L.kw * ho * wo
        fl["tower_dw"] += 2.0 * mac
        fl["tower_dx"] += 2.0 * mac
    for hd in (spec.cls_heads[0], spec.bbox_head):
        fl["heads"] += 2 * 2.0 * R * hd.col_len * hd.cout
    fl["total"] = sum(fl.values())
    return fl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train_resnet.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    info = gpu_info()
    ctx = mpn.Context(0)
    max_h, max_w = max(h for h, _ in SIZES), max(w for _, w in SIZES)
    n, R = len(SIZES), PER_IMAGE * len(SIZES)
    res = {"tool": "train_resnet_time", **info, "images": [list(s) for s in SIZES], "rois_per_image": PER_IMAGE,
           "iters": args.iters, "warmup": args.warmup, "models": {}}
    for name, build in (("resnet18_fast_rcnn", models.resnet18_fast_rcnn), ("resnet50_fast_rcnn", models.resnet50_fast_rcnn)):
        spec = build(81, seed=1234, integral_k=6, fixed_bn=True)
        free0, total = torch.cuda.mem_get_info()
        m = mpn.Model(ctx, spec, max_rois=R, max_h=max_h, max_w=max_w)
        tr = mpn.Trainer(m, seed=SEED, train_trunk=True, integral=True)
        rng = np.random.default_rng(0)
        ims = [torch.from_numpy(wl.transform(wl.raw_image(h, w, i), spec.transformer)).cuda() for i, (h, w) in enumerate(SIZES)]
        boxes = torch.from_numpy(np.concatenate([wl.random_boxes(PER_IMAGE, h, w, i) for i, (h, w) in enumerate(SIZES)]).astype(np.float32)).cuda()
        C = spec.num_classes
        labels = torch.from_numpy(rng.integers(1, C + 1, R).astype(np.int32)).cuda()
        tg = torch.zeros((R, 4 * C), dtype=torch.float32, device="cuda")
        losses = torch.zeros(3, dtype=torch.float32, device="cuda")
        ptrs = (Cc.c_void_p * n)(*[im.data_ptr() for im in ims])
        hw = np.array([v for s in SIZES for v in s], np.int32)
        cnt = np.full(n, PER_IMAGE, np.int32)

        def step():
            ctx.check(ctx.lib.mpn_model_train_step_dev(m.h, n, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
                                                       boxes.data_ptr(), labels.data_ptr(), tg.data_ptr(), losses.data_ptr()), "train_step_dev")
        for _ in range(args.warmup):
            step()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            step()
        b.record()
        b.synchronize()
        finite = bool(torch.isfinite(losses).all())
        ms = np.zeros(4, np.float32)
        phases = []
        for _ in range(args.iters):
            step()
            ctx.check(ctx.lib.mpn_model_train_phase_ms(m.h, ms.ctypes.data_as(mpn._lib._f32p)), "train_phase_ms")
            phases.append(ms.copy())
        ph = np.median(np.stack(phases), 0)
        free1, _ = torch.cuda.mem_get_info()
        fl = backward_flops(spec, SIZES, R)
        res["models"][name] = {
            "step_ms": round(a.elapsed_time(b) / args.iters, 3), "losses_finite": finite,
            "phase_ms_median": {"trunk_pool": round(float(ph[0]), 3), "forward_criteria": round(float(ph[1]), 3),
                                "backward": round(float(ph[2]), 3), "update": round(float(ph[3]), 3)},
            "device_mem_in_use_gb": round((free0 - free1) / 1e9, 2),
            "backward_gflop_counted": {k: round(v / 1e9, 1) for k, v in fl.items()},
            "backward_tflops_achieved": round(fl["total"] / (float(ph[2]) * 1e-3) / 1e12, 1)}
        tr.close(); m.close()
        del ims, boxes, labels, tg, losses
        torch.cuda.synchronize()
    res["note"] = ("CUDA events over --iters steps after --warmup; phase times are the library's events inside each step; the "
                   "backward FLOPs are counted from the shapes (dgrad + wgrad, BF16X3 issues three tensor-core products per "
                   "counted MAC), over the measured backward phase")
    d = os.path.dirname(args.out)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(res) + "\n")
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()

"""Times the fixed-batch-norm Inception-v3 training step (Mixed_7a .. 7c and the heads, the trunk frozen: inceptionv3.lua's
classifier, modules 26..30) on the COCO recipe's minibatch (scale 800, max_size 1000, 4 images, 64 ROIs per image):
inception_v3_fast_rcnn(81, integral_k=6, fixed_bn=True), in the default numerics and in bf16 training
(Trainer(bf16=True)), two models in one process whose steps alternate. Per model, CUDA events around each of --iters
steps after --warmup steps each, then the library's phase events of each step (mpn_model_train_phase_ms: trunks + ROI
pooling, per-ROI forward + criteria, backward, update), medians over the steps, and the device memory in use once its
steps ran (cudaMemGetInfo before the model was built and after its steps: the library's allocations are not torch's).
The backward's dgrad and wgrad FLOPs are counted from the shapes. Writes profiles/h100_train_inception.json (or --out)
with the GPU's name and power limit read in the same run.
    python tools/train_inception_time.py [--out FILE] [--iters 20] [--warmup 3]"""
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
from multipathnet_b200._lib import MPN_LAYER_CONV
from train_time import gpu_info

SIZES = ((800, 1000), (800, 1000), (666, 1000), (800, 800))
PER_IMAGE = 64
SEED = 555


def backward_flops(spec, R):
    """dgrad + wgrad FLOPs of one step's backward (2 * MACs), counted from the shapes: every tower convolution's wgrad and,
    unless it reads the pooled map (the trunk is frozen), its dgrad; the heads' dW and their dX into the tower's columns"""
    t = spec.towers[0]
    shp = {0: (t.pooled_h, t.pooled_w)}
    fl = {"tower_dw": 0.0, "tower_dx": 0.0, "heads": 0.0}
    for L in t.layers:
        h, w = shp[L.in_slot]
        if L.kind != MPN_LAYER_CONV:
            shp[L.out_slot] = (1, 1) if L.kind == models.MPN_LAYER_AVGPOOL else \
                (models._pool_out(h, L.kh, L.stride, L.pad, L.ceil_mode), models._pool_out(w, L.kw, L.stride, L.pad, L.ceil_mode))
            continue
        ho, wo = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.padw - L.kw) // L.stride + 1
        shp[L.out_slot] = (ho, wo)
        mac = R * L.cin * L.cout * L.kh * L.kw * ho * wo
        fl["tower_dw"] += 2.0 * mac
        if L.in_slot != 0:
            fl["tower_dx"] += 2.0 * mac
    for hd in (spec.cls_heads[0], spec.bbox_head):
        fl["heads"] += 2 * 2.0 * R * hd.col_len * hd.cout
    fl["total"] = sum(fl.values())
    return fl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train_inception.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    info = gpu_info()
    ctx = mpn.Context(0)
    max_h, max_w = max(h for h, _ in SIZES), max(w for _, w in SIZES)
    n, R = len(SIZES), PER_IMAGE * len(SIZES)
    spec = models.inception_v3_fast_rcnn(81, seed=1234, integral_k=6, fixed_bn=True)
    rng = np.random.default_rng(0)
    ims = [torch.from_numpy(wl.transform(wl.raw_image(h, w, i), spec.transformer)).cuda() for i, (h, w) in enumerate(SIZES)]
    boxes = torch.from_numpy(np.concatenate([wl.random_boxes(PER_IMAGE, h, w, i) for i, (h, w) in enumerate(SIZES)]).astype(np.float32)).cuda()
    C = spec.num_classes
    labels = torch.from_numpy(rng.integers(1, C + 1, R).astype(np.int32)).cuda()
    tg = torch.zeros((R, 4 * C), dtype=torch.float32, device="cuda")
    ptrs = (Cc.c_void_p * n)(*[im.data_ptr() for im in ims])
    hw = np.array([v for s in SIZES for v in s], np.int32)
    cnt = np.full(n, PER_IMAGE, np.int32)
    torch.cuda.synchronize()
    runs = {}
    for name, bf16 in (("default", False), ("bf16", True)):
        free0, _ = torch.cuda.mem_get_info()
        m = mpn.Model(ctx, spec, max_rois=R, max_h=max_h, max_w=max_w)
        tr = mpn.Trainer(m, seed=SEED, integral=True, bf16=bf16)
        runs[name] = dict(m=m, tr=tr, free0=free0, losses=torch.zeros(3, dtype=torch.float32, device="cuda"), ms=[], ph=[])

    def step(r):
        ctx.check(ctx.lib.mpn_model_train_step_dev(r["m"].h, n, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
                                                   boxes.data_ptr(), labels.data_ptr(), tg.data_ptr(), r["losses"].data_ptr()), "train_step_dev")
    for r in runs.values():
        for _ in range(args.warmup):
            step(r)
    torch.cuda.synchronize()
    ms = np.zeros(4, np.float32)
    for _ in range(args.iters):
        for r in runs.values():
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            step(r)
            b.record()
            b.synchronize()
            r["ms"].append(a.elapsed_time(b))
            ctx.check(ctx.lib.mpn_model_train_phase_ms(r["m"].h, ms.ctypes.data_as(mpn._lib._f32p)), "train_phase_ms")
            r["ph"].append(ms.copy())
    fl = backward_flops(spec, R)
    res = {"tool": "train_inception_time", **info, "model": "inception_v3_fast_rcnn(81, integral_k=6, fixed_bn=True)",
           "images": [list(s) for s in SIZES], "rois_per_image": PER_IMAGE, "iters": args.iters, "warmup": args.warmup,
           "backward_gflop_counted": {k: round(v / 1e9, 1) for k, v in fl.items()}, "numerics": {}}
    free1, _ = torch.cuda.mem_get_info()
    for name, r in runs.items():
        ph = np.median(np.stack(r["ph"]), 0)
        res["numerics"][name] = {
            "step_ms_median": round(float(np.median(r["ms"])), 3), "step_ms_min": round(float(np.min(r["ms"])), 3),
            "losses_finite": bool(torch.isfinite(r["losses"]).all()),
            "phase_ms_median": {"trunk_pool": round(float(ph[0]), 3), "forward_criteria": round(float(ph[1]), 3),
                                "backward": round(float(ph[2]), 3), "update": round(float(ph[3]), 3)},
            "backward_tflops_achieved": round(fl["total"] / (float(ph[2]) * 1e-3) / 1e12, 1)}
    # each model's share once all steps ran: the bf16 model's is what closing it frees, the default's the rest
    order = list(runs)
    r0, r1 = runs[order[0]], runs[order[1]]
    r1["tr"].close(); r1["m"].close()
    torch.cuda.synchronize()
    free2, _ = torch.cuda.mem_get_info()
    res["numerics"][order[0]]["device_mem_in_use_gb"] = round((r0["free0"] - free2) / 1e9, 2)
    res["numerics"][order[1]]["device_mem_in_use_gb"] = round((free2 - free1) / 1e9, 2)
    r0["tr"].close(); r0["m"].close()
    res["note"] = ("default and bf16 steps alternate, each timed by CUDA events after --warmup steps of both; phase times are the "
                   "library's events inside each step, medians over --iters; device memory in use is each model's share after "
                   "all its steps (built, trained, not yet closed); the backward FLOPs are counted from the shapes (dgrad + "
                   "wgrad; BF16X3 issues three tensor-core products per counted MAC, bf16 one), over the measured backward phase")
    d = os.path.dirname(args.out)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(res) + "\n")
    print(json.dumps(res))
    ctx.close()


if __name__ == "__main__":
    main()

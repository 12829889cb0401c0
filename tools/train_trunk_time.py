"""Times the training step of vgg16_fast_rcnn(21) with the trunk frozen and with it training from conv3_1
(Trainer(train_trunk=True)): two images of 600 x 1000 and 600 x 800, 128 ROIs each. Two models are built and their steps
alternate in rounds: per round CUDA events around --iters back-to-back steps after --warmup steps, and the library's
phase events (mpn_model_train_phase_ms) over --iters more steps. The trunk backward's time is the trained run's backward
phase less the frozen run's; its counted work is the dgrad + wgrad FLOPs of conv3_1 .. conv5_3 (2x their forward FLOPs,
less conv3_1's dgrad). A step's peak device memory is read with cudaMemGetInfo around each model's construction and
first step: the library frees a buffer only to grow it, just before allocating the larger one, and never shrinks one, so
the memory it holds after a step is the step's peak. Writes profiles/h100_train_trunk.json (or --out) with the GPU's
name and power limit read in the same run.
    python tools/train_trunk_time.py [--iters 20] [--warmup 3] [--rounds 3]"""
import argparse
import ctypes as Cc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from tools.train_time import gpu_info


def trunk_backward_flops(spec, sizes):
    """2 x the forward FLOPs of every trained trunk convolution (dgrad + wgrad), less the lowest one's dgrad"""
    total = 0.0
    for H, W in sizes:
        h, w, first = H, W, True
        for L in spec.trunk_layers:
            if L.kind == mpn._lib.MPN_LAYER_MAXPOOL:
                h, w = (h + 1) // 2, (w + 1) // 2
                continue
            if L.in_slot == 0:
                continue
            if spec.trunk_layers.index(L) < spec.trunk_train_from:
                continue
            f = 2.0 * h * w * L.cin * L.cout * 9
            total += f if first else 2 * f
            first = False
    return total


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train_trunk.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    ctx = mpn.Context(0)
    spec = models.vgg16_fast_rcnn(21, seed=1234)
    sizes, per = ((600, 1000), (600, 800)), (128, 128)
    rng = np.random.default_rng(0)
    ims = [torch.from_numpy(wl.transform(wl.raw_image(h, w, i), spec.transformer)).cuda() for i, (h, w) in enumerate(sizes)]
    boxes = torch.from_numpy(np.concatenate([wl.random_boxes(n, h, w, i) for i, ((h, w), n) in enumerate(zip(sizes, per))]).astype(np.float32)).cuda()
    R, C = sum(per), spec.num_classes
    labels = torch.from_numpy(rng.integers(1, C + 1, R).astype(np.int32)).cuda()
    tg = torch.zeros((R, 4 * C), dtype=torch.float32, device="cuda")
    ptrs = (Cc.c_void_p * 2)(*[im.data_ptr() for im in ims])
    hw = np.array([s for hw_ in sizes for s in hw_], np.int32)
    cnt = np.array(per, np.int32)
    runs = {}
    for name, trunk in (("frozen", False), ("trunk", True)):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        m = mpn.Model(ctx, spec, max_rois=256, max_h=608, max_w=1008)
        tr = mpn.Trainer(m, train_trunk=trunk)
        losses = torch.zeros(3, dtype=torch.float32, device="cuda")

        def step(m=m, losses=losses):
            ctx.check(ctx.lib.mpn_model_train_step_dev(m.h, 2, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
                                                       boxes.data_ptr(), labels.data_ptr(), tg.data_ptr(), losses.data_ptr()), "train_step_dev")
        step()
        ctx.synchronize()
        runs[name] = {"m": m, "tr": tr, "step": step, "losses": losses, "mem_gb": (free0 - torch.cuda.mem_get_info()[0]) / 1e9,
                      "step_ms": [], "phases": []}

    def time_ms(fn):
        for _ in range(args.warmup):
            fn()
        torch.cuda.synchronize()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(args.iters):
            fn()
        b.record()
        b.synchronize()
        return a.elapsed_time(b) / args.iters

    ms = np.zeros(4, np.float32)
    for _ in range(args.rounds):
        for name in ("frozen", "trunk"):
            r = runs[name]
            r["step_ms"].append(time_ms(r["step"]))
            for _ in range(args.iters):
                r["step"]()
                ctx.check(ctx.lib.mpn_model_train_phase_ms(r["m"].h, ms.ctypes.data_as(mpn._lib._f32p)), "train_phase_ms")
                r["phases"].append(ms.copy())
    out = {"tool": "train_trunk_time", **gpu_info(), "shape": "vgg16_fast_rcnn(21), 600x1000 + 600x800, 128 ROIs each",
           "iters": args.iters, "warmup": args.warmup, "rounds": args.rounds}
    for name, r in runs.items():
        ph = np.median(np.stack(r["phases"]), 0)
        out[name] = {"step_ms_per_round": [round(x, 3) for x in r["step_ms"]], "step_ms_median": round(float(np.median(r["step_ms"])), 3),
                     "phase_ms_median": {"trunk_pool": round(float(ph[0]), 3), "forward_criteria": round(float(ph[1]), 3),
                                         "backward": round(float(ph[2]), 3), "update": round(float(ph[3]), 3)},
                     "device_mem_peak_gb": round(r["mem_gb"], 2), "losses_finite": bool(torch.isfinite(r["losses"]).all())}
    tb = out["trunk"]["phase_ms_median"]["backward"] - out["frozen"]["phase_ms_median"]["backward"]
    fl = trunk_backward_flops(spec, sizes)
    out["trunk_backward_ms"] = round(tb, 3)
    out["trunk_backward_tflop_counted"] = round(fl / 1e12, 4)
    out["trunk_backward_tflops"] = round(fl / 1e12 / (tb / 1e3), 1) if tb > 0 else None
    out["note"] = ("trunk backward = the trained run's backward phase less the frozen run's (ROI backward, gates, pool backward, "
                   "transposes, bias sums and the dgrad / wgrad GEMMs); TFLOP/s = counted dgrad + wgrad FLOPs over that time; "
                   "memory = cudaMemGetInfo difference across building the model and its first step, the step's peak: the library frees "
                   "a buffer only to grow it, before allocating the larger one, and never shrinks one")
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(out) + "\n")
    print(json.dumps(out))
    for r in runs.values():
        r["tr"].close(); r["m"].close()
    ctx.close()


if __name__ == "__main__":
    main()

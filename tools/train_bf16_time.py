"""Times the default training step (BF16X3: three bf16 products per MAC) against the bf16 one (Trainer(bf16=True): one
bf16 product per MAC in every forward and backward GEMM) on the recipe sizes:
  vgg_trunk:   vgg16_fast_rcnn(21), trunk training from conv3_1, 600 x 1000 + 600 x 800, 128 ROIs each;
  mpn_phase1 / mpn_phase2: vgg16_multipathnet(81, integral_k=6) before and after set_phase2, and
  resnet18 / resnet50: resnetXX_fast_rcnn(81, integral_k=6, fixed_bn=True) with the trunk training, all on the COCO
  recipe's four-image minibatch (800 x 1000, 800 x 1000, 666 x 1000, 800 x 800), 64 ROIs each.
Per config the two modes' models are built side by side and their steps alternate in rounds: per round CUDA events
around --iters back-to-back steps after --warmup steps, and the library's phase events (mpn_model_train_phase_ms) over
--iters more steps. Peak device memory as tools/train_trunk_time.py reads it: cudaMemGetInfo across building a model
and its first step (the library only grows buffers). Writes profiles/h100_train_bf16.json (or --out) with the GPU's
name, power limit and max SM clock read in the same run.
    python tools/train_bf16_time.py [--iters 20] [--warmup 3] [--rounds 3] [--configs vgg_trunk,...]"""
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

COCO_SIZES, COCO_PER = ((800, 1000), (800, 1000), (666, 1000), (800, 800)), (64, 64, 64, 64)
CONFIGS = {
    "vgg_trunk": (lambda: models.vgg16_fast_rcnn(21, seed=1234), ((600, 1000), (600, 800)), (128, 128), dict(train_trunk=True), False),
    "mpn_phase1": (lambda: models.vgg16_multipathnet(81, seed=1234, integral_k=6), COCO_SIZES, COCO_PER, dict(phase2=True, integral=True), False),
    "mpn_phase2": (lambda: models.vgg16_multipathnet(81, seed=1234, integral_k=6), COCO_SIZES, COCO_PER, dict(phase2=True, integral=True), True),
    "resnet18": (lambda: models.resnet18_fast_rcnn(81, seed=1234, integral_k=6, fixed_bn=True), COCO_SIZES, COCO_PER,
                 dict(train_trunk=True, integral=True), False),
    "resnet50": (lambda: models.resnet50_fast_rcnn(81, seed=1234, integral_k=6, fixed_bn=True), COCO_SIZES, COCO_PER,
                 dict(train_trunk=True, integral=True), False),
}


def run_config(ctx, name, args):
    build, sizes, per, kw, phase2 = CONFIGS[name]
    spec = build()
    rng = np.random.default_rng(0)
    ims = [torch.from_numpy(wl.transform(wl.raw_image(h, w, i), spec.transformer)).cuda() for i, (h, w) in enumerate(sizes)]
    boxes = torch.from_numpy(np.concatenate([wl.random_boxes(n, h, w, i) for i, ((h, w), n) in enumerate(zip(sizes, per))]).astype(np.float32)).cuda()
    R, C = sum(per), spec.num_classes
    labels = torch.from_numpy(rng.integers(1, C + 1, R).astype(np.int32)).cuda()
    tg = torch.zeros((R, 4 * C), dtype=torch.float32, device="cuda")
    n = len(sizes)
    ptrs = (Cc.c_void_p * n)(*[im.data_ptr() for im in ims])
    hw = np.array([s for hw_ in sizes for s in hw_], np.int32)
    cnt = np.array(per, np.int32)
    max_h, max_w = max(h for h, _ in sizes), max(w for _, w in sizes)
    runs = {}
    for mode, bf16 in (("default", False), ("bf16", True)):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        m = mpn.Model(ctx, spec, max_rois=R, max_h=max_h, max_w=max_w)
        tr = mpn.Trainer(m, bf16=bf16, **kw)
        if phase2:
            tr.set_phase2()
        losses = torch.zeros(3, dtype=torch.float32, device="cuda")

        def step(m=m, losses=losses):
            ctx.check(ctx.lib.mpn_model_train_step_dev(m.h, n, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
                                                       boxes.data_ptr(), labels.data_ptr(), tg.data_ptr(), losses.data_ptr()), "train_step_dev")
        step()
        ctx.synchronize()
        runs[mode] = {"m": m, "tr": tr, "step": step, "losses": losses, "mem_gb": (free0 - torch.cuda.mem_get_info()[0]) / 1e9,
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
        for mode in ("default", "bf16"):
            r = runs[mode]
            r["step_ms"].append(time_ms(r["step"]))
            for _ in range(args.iters):
                r["step"]()
                ctx.check(ctx.lib.mpn_model_train_phase_ms(r["m"].h, ms.ctypes.data_as(mpn._lib._f32p)), "train_phase_ms")
                r["phases"].append(ms.copy())
    out = {"shape": f"{spec.name}, " + " + ".join(f"{h}x{w}" for h, w in sizes) + f", {per[0]} ROIs each" + (", phase 2" if phase2 else "")}
    for mode, r in runs.items():
        ph = np.median(np.stack(r["phases"]), 0)
        out[mode] = {"step_ms_per_round": [round(x, 3) for x in r["step_ms"]], "step_ms_median": round(float(np.median(r["step_ms"])), 3),
                     "phase_ms_median": {"trunk_pool": round(float(ph[0]), 3), "forward_criteria": round(float(ph[1]), 3),
                                         "backward": round(float(ph[2]), 3), "update": round(float(ph[3]), 3)},
                     "device_mem_peak_gb": round(r["mem_gb"], 3), "losses_finite": bool(torch.isfinite(r["losses"]).all())}
        r["tr"].close(); r["m"].close()
    out["speedup_step"] = round(out["default"]["step_ms_median"] / out["bf16"]["step_ms_median"], 3)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train_bf16.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    ctx = mpn.Context(0)
    out = {"tool": "train_bf16_time", **gpu_info(), "iters": args.iters, "warmup": args.warmup, "rounds": args.rounds,
           "note": ("default = BF16X3, bf16 = Trainer(bf16=True); step_ms from CUDA events over iters steps after warmup, per "
                    "round, the two modes alternating; phase medians from mpn_model_train_phase_ms; memory = cudaMemGetInfo "
                    "difference across building the model and its first step")}
    for name in args.configs.split(","):
        out[name] = run_config(ctx, name, args)
        print(name, json.dumps(out[name]), flush=True)
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(out) + "\n")
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()

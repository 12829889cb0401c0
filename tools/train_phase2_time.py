"""Times MultiPathNet's training step in phase 1 (towers and heads) and phase 2 (also the trunk from conv3_1, through the
towers' foveal, normalised ROI pooling backward) on the COCO recipe's minibatch (train_multipathnet_coco.sh): four images
of 800 x 1000, 800 x 1000, 666 x 1000 and 800 x 800, 64 ROIs each, vgg16_multipathnet(81, integral_k=6). Two models are
built, one left in phase 1 and one switched to phase 2 (Trainer(phase2=True), set_phase2); their steps alternate in
rounds: per round CUDA events around --iters back-to-back steps after --warmup steps, and the library's phase events
(mpn_model_train_phase_ms) over --iters more steps. Peak device memory as tools/train_trunk_time.py reads it. Then, in a
separate pass under torch.profiler, the ROI pooling backward's kernels of --profile-steps phase-2 steps are timed on
their own. Writes profiles/h100_train_phase2.json (or --out) with the GPU's name and power limit read in the same run.
    python tools/train_phase2_time.py [--iters 20] [--warmup 3] [--rounds 3] [--profile-steps 5]"""
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

ROI_KERNELS = ("roi_argmax_nhwc_kernel", "roi_norm_ab_kernel", "roi_backward_nhwc_kernel")


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--profile-steps", type=int, default=5)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train_phase2.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    ctx = mpn.Context(0)
    spec = models.vgg16_multipathnet(81, seed=1234, integral_k=6)
    sizes, per = ((800, 1000), (800, 1000), (666, 1000), (800, 800)), (64, 64, 64, 64)
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
    runs = {}
    for name in ("phase1", "phase2"):
        torch.cuda.synchronize()
        free0 = torch.cuda.mem_get_info()[0]
        m = mpn.Model(ctx, spec, max_rois=256, max_h=1000, max_w=1000)
        tr = mpn.Trainer(m, phase2=True, integral=True)
        if name == "phase2":
            tr.set_phase2()
        losses = torch.zeros(3, dtype=torch.float32, device="cuda")

        def step(m=m, losses=losses):
            ctx.check(ctx.lib.mpn_model_train_step_dev(m.h, n, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
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
        for name in ("phase1", "phase2"):
            r = runs[name]
            r["step_ms"].append(time_ms(r["step"]))
            for _ in range(args.iters):
                r["step"]()
                ctx.check(ctx.lib.mpn_model_train_phase_ms(r["m"].h, ms.ctypes.data_as(mpn._lib._f32p)), "train_phase_ms")
                r["phases"].append(ms.copy())
    out = {"tool": "train_phase2_time", **gpu_info(),
           "shape": "vgg16_multipathnet(81, integral_k=6), 800x1000 + 800x1000 + 666x1000 + 800x800, 64 ROIs each",
           "iters": args.iters, "warmup": args.warmup, "rounds": args.rounds}
    for name, r in runs.items():
        ph = np.median(np.stack(r["phases"]), 0)
        out[name] = {"step_ms_per_round": [round(x, 3) for x in r["step_ms"]], "step_ms_median": round(float(np.median(r["step_ms"])), 3),
                     "phase_ms_median": {"trunk_pool": round(float(ph[0]), 3), "forward_criteria": round(float(ph[1]), 3),
                                         "backward": round(float(ph[2]), 3), "update": round(float(ph[3]), 3)},
                     "device_mem_peak_gb": round(r["mem_gb"], 2), "losses_finite": bool(torch.isfinite(r["losses"]).all())}
    out["phase2_extra_backward_ms"] = round(out["phase2"]["phase_ms_median"]["backward"] - out["phase1"]["phase_ms_median"]["backward"], 3)
    # the ROI pooling backward's kernels on their own, in a separate traced pass
    r = runs["phase2"]
    torch.cuda.synchronize()
    with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.profile_steps):
            r["step"]()
        torch.cuda.synchronize()
    per_kernel = {k: 0.0 for k in ROI_KERNELS}
    calls = {k: 0 for k in ROI_KERNELS}
    for e in prof.key_averages():
        for k in ROI_KERNELS:
            if k in e.key:
                per_kernel[k] += e.device_time_total / 1e3        # us -> ms
                calls[k] += e.count
    out["roi_backward_ms_per_step"] = {k: round(v / args.profile_steps, 3) for k, v in per_kernel.items()}
    out["roi_backward_launches_per_step"] = {k: calls[k] // args.profile_steps for k in ROI_KERNELS}
    out["roi_backward_ms_per_step_total"] = round(sum(per_kernel.values()) / args.profile_steps, 3)
    out["note"] = ("phase 2's extra backward = its backward phase less phase 1's (the towers' first-layer dX, the ROI pooling "
                   "backward of 11 (tower, level) jobs per image, the trunk's gates, pool backward and dgrad / wgrad GEMMs); "
                   "memory = cudaMemGetInfo difference across building the model and its first step, the step's peak; "
                   "ROI backward kernels from torch.profiler in a separate pass after the timed rounds")
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(out) + "\n")
    print(json.dumps(out))
    for r in runs.values():
        r["tr"].close(); r["m"].close()
    ctx.close()


if __name__ == "__main__":
    main()

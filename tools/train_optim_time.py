"""Times the training step under each optim method (Trainer(method=...): sgd, adam, adamax, adagrad, rmsprop) on two
workloads:
  mpn_phase1: vgg16_multipathnet(81, integral_k=6) on the COCO recipe's four-image minibatch (800 x 1000, 800 x 1000,
              666 x 1000, 800 x 800), 64 ROIs each, phase 1;
  vgg_trunk:  vgg16_fast_rcnn(21), trunk training from conv3_1, 600 x 1000 + 600 x 800, 128 ROIs each.
Per round the methods take turns: each builds its model and trainer, takes --warmup steps, CUDA events around --iters
back-to-back steps, then the library's phase events (mpn_model_train_phase_ms) over --iters more steps, and is closed
(two MultiPathNet trainers do not fit side by side with their states). Peak device memory: cudaMemGetInfo across
building the model and its first step, in the first round. The update phase's counted bytes are, per trained element,
the fp32 master read and written, the gradient read, each state read and written, and for a weight its forward split
planes written (hi + lo, 4 bytes); the W^T / rotated dgrad planes are not counted. Writes profiles/h100_train_optim.json
(or --out) with the GPU's name, power limit and max SM clock read in the same run.
    python tools/train_optim_time.py [--iters 10] [--warmup 3] [--rounds 2] [--configs mpn_phase1,vgg_trunk]"""
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

METHODS = ("sgd", "adam", "adamax", "adagrad", "rmsprop")
COCO_SIZES, COCO_PER = ((800, 1000), (800, 1000), (666, 1000), (800, 800)), (64, 64, 64, 64)
CONFIGS = {
    "mpn_phase1": (lambda: models.vgg16_multipathnet(81, seed=1234, integral_k=6), COCO_SIZES, COCO_PER, dict(phase2=True, integral=True)),
    "vgg_trunk": (lambda: models.vgg16_fast_rcnn(21, seed=1234), ((600, 1000), (600, 800)), (128, 128), dict(train_trunk=True)),
}


def update_bytes(spec, trained, n_states):
    """the update phase's counted bytes (see the module docstring)"""
    total = 0
    for i in trained:
        n = int(np.prod(np.shape(spec.weights[i])))
        total += n * (8 + 4 + 8 * n_states) + (n * 4 if np.ndim(spec.weights[i]) > 1 else 0)
    return total


def run_config(ctx, name, args):
    build, sizes, per, kw = CONFIGS[name]
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
    res = {mth: {"step_ms": [], "phases": []} for mth in METHODS}
    ms = np.zeros(4, np.float32)
    for rnd in range(args.rounds):
        for mth in METHODS:
            torch.cuda.synchronize()
            free0 = torch.cuda.mem_get_info()[0]
            m = mpn.Model(ctx, spec, max_rois=R, max_h=max_h, max_w=max_w)
            tr = mpn.Trainer(m, method=mth, **kw)
            losses = torch.zeros(3, dtype=torch.float32, device="cuda")

            def step():
                ctx.check(ctx.lib.mpn_model_train_step_dev(m.h, n, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
                                                           boxes.data_ptr(), labels.data_ptr(), tg.data_ptr(), losses.data_ptr()), "train_step_dev")
            step()
            ctx.synchronize()
            r = res[mth]
            if rnd == 0:
                r["mem_gb"] = (free0 - torch.cuda.mem_get_info()[0]) / 1e9
                r["update_bytes"] = update_bytes(spec, tr.trained, tr._n_states)
            for _ in range(args.warmup):
                step()
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                step()
            b.record()
            b.synchronize()
            r["step_ms"].append(a.elapsed_time(b) / args.iters)
            for _ in range(args.iters):
                step()
                ctx.check(ctx.lib.mpn_model_train_phase_ms(m.h, ms.ctypes.data_as(mpn._lib._f32p)), "train_phase_ms")
                r["phases"].append(ms.copy())
            last = [tr._get(i, 0) for i in tr.trained[-2:]]                   # the bbox head: the same bits in every round
            r["finite"] = bool(torch.isfinite(losses).all()) and all(np.isfinite(w).all() for w in last)
            r.setdefault("bits", []).append(hash(b"".join(w.tobytes() for w in last)))
            tr.close(); m.close()
            del tr, m
            torch.cuda.synchronize()
    out = {"shape": f"{spec.name}, " + " + ".join(f"{h}x{w}" for h, w in sizes) + f", {per[0]} ROIs each"}
    for mth, r in res.items():
        ph = np.median(np.stack(r["phases"]), 0)
        out[mth] = {"step_ms_per_round": [round(x, 3) for x in r["step_ms"]], "step_ms_median": round(float(np.median(r["step_ms"])), 3),
                    "phase_ms_median": {"trunk_pool": round(float(ph[0]), 3), "forward_criteria": round(float(ph[1]), 3),
                                        "backward": round(float(ph[2]), 3), "update": round(float(ph[3]), 3)},
                    "update_counted_gb": round(r["update_bytes"] / 1e9, 3),
                    "update_counted_gb_per_s": round(r["update_bytes"] / 1e9 / (float(ph[3]) / 1e3), 1),
                    "device_mem_peak_gb": round(r["mem_gb"], 3), "finite": r["finite"], "same_bits_every_round": len(set(r["bits"])) == 1}
    out["update_vs_sgd"] = {mth: round(out[mth]["phase_ms_median"]["update"] / out["sgd"]["phase_ms_median"]["update"], 3) for mth in METHODS}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train_optim.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    ctx = mpn.Context(0)
    out = {"tool": "train_optim_time", **gpu_info(), "iters": args.iters, "warmup": args.warmup, "rounds": args.rounds,
           "note": ("step_ms from CUDA events over iters steps after warmup, per round, the methods taking turns; phase medians "
                    "from mpn_model_train_phase_ms; memory = cudaMemGetInfo difference across building the model and its first "
                    "step; update GB/s = counted bytes over the update phase's median")}
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

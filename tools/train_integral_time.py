"""Times the training step with the integral loss against the plain step, on the recipe's minibatch
(scripts/train_multipathnet_coco.sh: scale 800, max_size 1000, 4 images, 64 ROIs per image): vgg16_multipathnet(81,
integral_k=6), whose step trains the head of the step's threshold set (mpn_integral_set) and updates the five idle
heads with a zero gradient, and vgg16_multipathnet(81) (one class head) on the same batches. The two alternate --rounds
times in one run; per round and model, CUDA events around --iters back-to-back steps after --warmup steps, then the
library's phase events (mpn_model_train_phase_ms: trunks + ROI pooling, per-ROI forward + criteria, backward, update),
medians over --iters more steps. The idle heads' update traffic is counted from the shapes (per weight element: read w
and buf, write w, buf, the split planes and the transposed planes). Writes profiles/h100_train_integral.json (or
--out DIR / FILE) with the GPU's name and power limit read in the same run.
    python tools/train_integral_time.py [--out DIR] [--rounds 3] [--iters 20] [--warmup 3]"""
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
from multipathnet_b200.batch_provider import integral_set
from train_time import gpu_info

SIZES = ((800, 1000), (800, 1000), (666, 1000), (800, 800))
PER_IMAGE = 64
K = 6
SEED = 555


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train_integral.json"))
    args = ap.parse_args()
    out = os.path.join(args.out, "h100_train_integral.json") if os.path.isdir(args.out) or not args.out.endswith(".json") else args.out
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    info = gpu_info()
    ctx = mpn.Context(0)
    specs = {"integral_k6": models.vgg16_multipathnet(81, seed=1234, integral_k=K), "plain": models.vgg16_multipathnet(81, seed=1234)}
    max_h, max_w = max(h for h, _ in SIZES), max(w for _, w in SIZES)
    n, R = len(SIZES), PER_IMAGE * len(SIZES)
    runs = {}
    for name, spec in specs.items():
        m = mpn.Model(ctx, spec, max_rois=R, max_h=max_h, max_w=max_w)
        runs[name] = (m, mpn.Trainer(m, seed=SEED, integral=len(spec.cls_heads) > 1), spec)
    spec = specs["plain"]
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
    counter = {k: 0 for k in runs}

    def step(name):
        m, tr, s = runs[name]
        if len(s.cls_heads) > 1:                          # the step's threshold set picks the trained head
            ctx.check(ctx.lib.mpn_model_train_select_head(m.h, integral_set(SEED, counter[name], len(s.cls_heads))), "select_head")
        counter[name] += 1
        ctx.check(ctx.lib.mpn_model_train_step_dev(m.h, n, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
                                                   boxes.data_ptr(), labels.data_ptr(), tg.data_ptr(), losses.data_ptr()), "train_step_dev")

    rounds = []
    finite = True
    for r in range(args.rounds):
        row = {}
        for name in runs:
            for _ in range(args.warmup):
                step(name)
            torch.cuda.synchronize()
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
            for _ in range(args.iters):
                step(name)
            b.record()
            b.synchronize()
            finite = finite and bool(torch.isfinite(losses).all())
            ms = np.zeros(4, np.float32)
            phases = []
            for _ in range(args.iters):
                step(name)
                ctx.check(ctx.lib.mpn_model_train_phase_ms(runs[name][0].h, ms.ctypes.data_as(mpn._lib._f32p)), "train_phase_ms")
                phases.append(ms.copy())
            ph = np.median(np.stack(phases), 0)
            row[name] = {"step_ms": round(a.elapsed_time(b) / args.iters, 3),
                         "phase_ms_median": {"trunk_pool": round(float(ph[0]), 3), "forward_criteria": round(float(ph[1]), 3),
                                             "backward": round(float(ph[2]), 3), "update": round(float(ph[3]), 3)}}
        rounds.append(row)
    med = {name: {"step_ms": round(float(np.median([r[name]["step_ms"] for r in rounds])), 3),
                  "phase_ms_median": {p: round(float(np.median([r[name]["phase_ms_median"][p] for r in rounds])), 3)
                                      for p in rounds[0][name]["phase_ms_median"]}} for name in runs}
    ch = specs["integral_k6"].cls_heads[0]
    idle_elems = (K - 1) * ch.cout * ch.col_len
    idle_bytes = idle_elems * 24 + (K - 1) * ch.cout * 12       # weights: w, buf r/w + split + W^T planes; biases: w, buf r/w
    res = {"tool": "train_integral_time", **info,
           "shape": f"vgg16_multipathnet(81), integral_k={K} vs 1 class head; images {list(SIZES)}, {PER_IMAGE} ROIs each (R = {R})",
           "rounds": args.rounds, "iters": args.iters, "warmup": args.warmup, "losses_finite": finite,
           "per_round": rounds, "median_over_rounds": med,
           "step_ms_delta": round(med["integral_k6"]["step_ms"] - med["plain"]["step_ms"], 3),
           "update_ms_delta": round(med["integral_k6"]["phase_ms_median"]["update"] - med["plain"]["phase_ms_median"]["update"], 3),
           "idle_head_update_elems_counted": idle_elems, "idle_head_update_mb_counted": round(idle_bytes / 1e6, 1),
           "note": "phase times are the library's events inside each step; the idle-head bytes are counted from the shapes, "
                   "not measured; the integral model trains the head mpn_integral_set draws for each step"}
    d = os.path.dirname(out)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(out, "w") as f:
        f.write(json.dumps(res) + "\n")
    print(json.dumps(res))
    for m, tr, _ in runs.values():
        tr.close(); m.close()
    ctx.close()


if __name__ == "__main__":
    main()

"""Times data-parallel training (Trainer(replicas=...), train.lua's train_nGPU) against one trainer, on two workloads:
vgg16_multipathnet(81, integral_k=6) phase 1 on the COCO recipe's minibatch (scripts/train_multipathnet_coco.sh: 4 images
of up to 800 x 1000, 64 ROIs each) and VGG-16 Fast R-CNN with its trunk (vgg.lua's recipe: 2 images of 600 x 1000, 64
ROIs each). K = 1 and K = 2 replicas on device 0 alternate --rounds times in one run; with two or more GPUs, K = 2 on
devices 0 and 1 joins the rotation. Per round and setup: CUDA events around --iters back-to-back steps after --warmup
steps (every step ends in a host synchronise, so the window holds every replica's work), and the median of the
reduction's own events (mpn_model_train_allreduce_ms). The reduction's bytes are counted from the shapes: G, the bytes of
the gradients a step sums, and the HBM traffic of K replicas on one device, per gradient element (K - 1) peer copies
into the stage (read + write), the ordered sum (K reads, one write) and (K - 1) copies of the gather (read + write).
Writes profiles/h100_train_dp.json (or --out DIR / FILE) with the GPU's name and power limit read in the same run.
    python tools/train_dp_time.py [--out DIR] [--rounds 3] [--iters 10] [--warmup 2]"""
import argparse
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
from train_time import gpu_info

SEED = 555
WORKLOADS = {
    "multipathnet_integral6_phase1": dict(sizes=((800, 1000), (800, 1000), (666, 1000), (800, 800)), per_image=64,
                                          spec=lambda: models.vgg16_multipathnet(81, seed=1234, integral_k=6), kw=dict(integral=True)),
    "vgg16_fast_rcnn_trunk": dict(sizes=((600, 1000), (600, 800)), per_image=64,
                                  spec=lambda: models.vgg16_fast_rcnn(81, seed=1234), kw=dict(train_trunk=True)),
}


def minibatch(spec, sizes, per_image, seed=0):
    rng = np.random.default_rng(seed)
    ims = [wl.transform(wl.raw_image(h, w, i), spec.transformer) for i, (h, w) in enumerate(sizes)]
    rois = [wl.random_boxes(per_image, h, w, i).astype(np.float32) for i, (h, w) in enumerate(sizes)]
    R, C = per_image * len(sizes), spec.num_classes
    labels = rng.integers(1, C + 1, R).astype(np.int32)
    tg = np.zeros((R, 4 * C), np.float32)
    for r in range(R):
        if labels[r] > 1:
            tg[r, 4 * labels[r] - 4:4 * labels[r]] = rng.standard_normal(4) * 0.5
    return ims, rois, labels, tg


def reduced_elems(tr):
    """the gradient elements a step sums: every trained tensor but the class heads the step did not train"""
    spec = tr.model.spec
    idle = {i for k, h in enumerate(spec.cls_heads) if k != tr.head for i in (h.weight, h.bias) if i >= 0}
    return int(sum(np.asarray(spec.weights[i]).size for i in tr.trained if i not in idle))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train_dp.json"))
    args = ap.parse_args()
    out = os.path.join(args.out, "h100_train_dp.json") if os.path.isdir(args.out) or not args.out.endswith(".json") else args.out
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    info = gpu_info()
    n_gpus = torch.cuda.device_count()
    placements = {"K1": [0], "K2_one_gpu": [0, 0]}
    if n_gpus >= 2:
        placements["K2_two_gpus"] = [0, 1]
    results = {}
    for wname, W in WORKLOADS.items():
        spec = W["spec"]()
        sizes, per_image = W["sizes"], W["per_image"]
        max_h, max_w = max(h for h, _ in sizes), max(w for _, w in sizes)
        R = per_image * len(sizes)
        batch = minibatch(spec, sizes, per_image)
        runs = {}
        for pname, devs in placements.items():
            ctxs = [mpn.Context(d, own_stream=True) for d in devs]
            ms = [mpn.Model(c, spec, max_rois=R, max_h=max_h, max_w=max_w) for c in ctxs]
            runs[pname] = (ctxs, mpn.Trainer(ms[0], replicas=ms[1:], seed=SEED, **W["kw"]))
        rounds, finite = [], True
        for _ in range(args.rounds):
            row = {}
            for pname, (ctxs, tr) in runs.items():
                for _ in range(args.warmup):
                    tr.step(*batch)
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                red, losses = [], None
                for _ in range(args.iters):
                    losses = tr.step(*batch)
                    if len(tr.models) > 1:
                        red.append(tr.allreduce_ms())
                b.record()
                b.synchronize()
                finite = finite and bool(np.isfinite(losses).all())
                row[pname] = {"step_ms": round(a.elapsed_time(b) / args.iters, 3)}
                if red:
                    row[pname]["allreduce_ms_median"] = round(float(np.median(red)), 3)
            rounds.append(row)
        res = {}
        for pname, (ctxs, tr) in runs.items():
            r = {"step_ms_median": round(float(np.median([x[pname]["step_ms"] for x in rounds])), 3)}
            if len(tr.models) > 1:
                K = len(tr.models)
                g = 4 * reduced_elems(tr)
                t = float(np.median([x[pname]["allreduce_ms_median"] for x in rounds]))
                traffic = g * ((K - 1) * 2 + (K + 1) + (K - 1) * 2)
                r.update(allreduce_ms_median=round(t, 3), gradient_gb_counted=round(g / 1e9, 3),
                         gradient_gb_per_s=round(g / t / 1e6, 1))
                if pname.endswith("one_gpu"):
                    r.update(hbm_traffic_gb_counted=round(traffic / 1e9, 3), hbm_gb_per_s=round(traffic / t / 1e6, 1))
            res[pname] = r
        results[wname] = {"shape": f"{spec.name}: images {list(sizes)}, {per_image} ROIs each (R = {R}); options {W['kw']}",
                          "per_round": rounds, "median_over_rounds": res, "losses_finite": finite}
        for ctxs, tr in runs.values():
            tr.close()
            for m in tr.models:
                m.close()
            for c in ctxs:
                c.close()
    doc = {"tool": "train_dp_time", **info, "gpus_visible": n_gpus, "rounds": args.rounds, "iters": args.iters, "warmup": args.warmup,
           "workloads": results,
           "note": "step_ms: CUDA events around back-to-back Trainer.step calls (host arrays, uploads included), each of which "
                   "ends in a host synchronise; allreduce_ms: the reduction's events on replica 0's stream; bytes counted "
                   "from the shapes, not measured. Multi-GPU scaling is measured only when gpus_visible > 1."}
    d = os.path.dirname(out)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(out, "w") as f:
        f.write(json.dumps(doc) + "\n")
    print(json.dumps(doc))


if __name__ == "__main__":
    main()

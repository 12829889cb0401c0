"""Times SVD-compressed detection (models.svd_compress, utils.SVDlinear) against the uncompressed model on one GPU, in one
process, and writes one JSON line per config plus one for the Linears.

  * detect + NMS, device-resident (mpn_model_detect_nms_dev), cfg 2 (VGG-16 Fast R-CNN, 600 x 800, 1000 ROIs, C = 21) and
    cfg 3 (MultiPathNet, 81 classes, 1000 SharpMask-shaped ROIs): uncompressed, ranks (1024, 256), and for cfg 2 also the
    factored model with fc6's first factor taken off the fp16-weight scheme ("fc_w16" = 0: three bf16 products per MAC,
    where the default is two with split-K). Every model is built and warmed up first; then the variants alternate
    --reps times, each timing --steps steps with CUDA events. Medians are reported.
  * fc6 / fc7 at R = 1000 against their factors, as a model plans each layer (Context.linear_bench: CUDA events over
    --iters launches, split-K reduce included), alternated --reps times, with achieved TFLOP/s from 2 R K N.
The GPU's name and power limit are read in the same process. Synthetic weights are not low-rank, so the outputs of the
compressed model are not compared with the uncompressed model's here: that says nothing about accuracy.
    python tools/svd_time.py [--steps 100] [--warmup 10] [--reps 3] [--iters 50] [--out profiles/h100_svd.json]"""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

RANKS = (1024, 256)
CONFIGS = {
    "vgg16_frcnn": dict(cfg=2, H=600, W=800, R=1000, C=21, boxes="random", model="vgg16_fast_rcnn"),
    "multipathnet": dict(cfg=3, H=600, W=800, R=1000, C=81, boxes="sharpmask", model="vgg16_multipathnet"),
}
# (name, N outputs, K inputs, w16 as the single-tower model plans it, biasless)
LINEARS = [("fc6", 4096, 25088, True, False), ("fc6_factor1", 1024, 25088, True, True), ("fc6_factor2", 4096, 1024, False, False),
           ("fc7", 4096, 4096, True, False), ("fc7_factor1", 256, 4096, False, True), ("fc7_factor2", 4096, 256, False, False)]


def gpu_info():
    """name, power limit and SM clocks of GPU 0 (read-only nvidia-smi query)"""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30, check=True).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit_w": float(q[1]), "sm_mhz": float(q[2]), "sm_max_mhz": float(q[3])}
    except (OSError, subprocess.SubprocessError, IndexError, ValueError) as e:
        return {"gpu": None, "power_limit_w": None, "sm_mhz": None, "sm_max_mhz": None, "nvidia_smi": str(e)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_svd.json"))
    args = ap.parse_args()
    if args.reps < 3:
        raise SystemExit("--reps must be at least 3")
    import torch
    import multipathnet_b200 as mpn
    from multipathnet_b200 import models, workloads as wl
    ctx = mpn.Context(0)                 # the legacy default stream: the one torch's events below are recorded on
    lines = []
    for name, c in CONFIGS.items():
        H, W, R, C = c["H"], c["W"], c["R"], c["C"]
        spec = getattr(models, c["model"])(C, seed=1234)
        t0 = time.time()
        svd = models.svd_compress(spec, RANKS)
        svd_s = time.time() - t0
        variants = {"uncompressed": (spec, -1), "svd": (svd, -1)}
        if c["cfg"] == 2:
            variants["svd_fc6_factor1_3prod"] = (svd, 0)
        boxes_fn = wl.sharpmask_boxes if c["boxes"] == "sharpmask" else wl.random_boxes
        img = torch.from_numpy(wl.transform(wl.raw_image(H, W, 2), spec.transformer)).cuda()
        boxes = torch.from_numpy(boxes_fn(R, H, W, 2)).cuda()
        sc = torch.empty((R, C), dtype=torch.float32, device="cuda")
        bb = torch.empty((R, 4 * C), dtype=torch.float32, device="cuda")
        kp = torch.empty((C - 1, R), dtype=torch.int32, device="cuda")
        ct = torch.empty((C - 1,), dtype=torch.int32, device="cuda")
        built = {}
        for v, (s, w16) in variants.items():
            ctx.set_option("fc_w16", w16)          # read when the model plans: at its first call below
            try:
                m = mpn.Model(ctx, s, max_rois=R + 48, max_h=H + 8, max_w=W)
                for _ in range(args.warmup):
                    m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, sc, bb, kp, ct)
                torch.cuda.synchronize()
            finally:
                ctx.set_option("fc_w16", -1)
            built[v] = (m, m.last_flops()[1] / R)
        runs = {v: [] for v in variants}
        for _ in range(args.reps):
            for v, (m, _) in built.items():
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(args.steps):
                    m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, sc, bb, kp, ct)
                b.record()
                b.synchronize()
                runs[v].append(a.elapsed_time(b) / args.steps)
        info = gpu_info()
        med = {v: float(np.median(r)) for v, r in runs.items()}
        line = {"tool": "svd_time", "config": name, "cfg": c["cfg"], "ranks": list(RANKS), "R": R, "steps": args.steps,
                "warmup": args.warmup, "reps": args.reps, **info, "svd_compress_s": svd_s,
                "head_gflop_per_roi": {v: f / 1e9 for v, (_, f) in built.items()},
                "ms_per_step": runs, "median_ms_per_step": med,
                "speedup_svd": med["uncompressed"] / med["svd"]}
        for m, _ in built.values():
            m.close()
        print(json.dumps(line), flush=True)
        lines.append(line)
    R = 1000
    ms = {n: [] for n, *_ in LINEARS}
    plan = {}
    for n, N, K, w16, nb in LINEARS:                   # warm-up and plan
        _, bn, sk = ctx.linear_bench(R, N, K, w16, nb, iters=3)
        plan[n] = {"N": N, "K": K, "w16": w16, "biasless": nb, "bn": bn, "splitk": sk}
    for _ in range(args.reps):
        for n, N, K, w16, nb in LINEARS:
            ms[n].append(ctx.linear_bench(R, N, K, w16, nb, iters=args.iters)[0])
    info = gpu_info()
    layers = {}
    for n, N, K, *_ in LINEARS:
        t = float(np.median(ms[n]))
        layers[n] = {**plan[n], "ms": ms[n], "median_ms": t, "tflops": 2.0 * R * K * N / (t * 1e-3) / 1e12}
    fc6f = layers["fc6_factor1"]["median_ms"] + layers["fc6_factor2"]["median_ms"]
    fc7f = layers["fc7_factor1"]["median_ms"] + layers["fc7_factor2"]["median_ms"]
    line = {"tool": "svd_time", "config": "linears", "R": R, "iters": args.iters, "reps": args.reps, **info, "layers": layers,
            "fc6_ms": layers["fc6"]["median_ms"], "fc6_factors_ms": fc6f, "fc7_ms": layers["fc7"]["median_ms"], "fc7_factors_ms": fc7f}
    print(json.dumps(line), flush=True)
    lines.append(line)
    ctx.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

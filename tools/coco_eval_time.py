"""Time mpn_coco_eval (testCoco.evaluate's score on the device) on a seeded synthetic set at COCO val2014 scale:
40,504 images, 80 categories, ~7 annotations and 100 detection rows per image (workloads.coco_eval_set).

Three figures for the full set: the host clock around the synchronous call (median of --reps), CUDA events on the ctx's
stream around the call, and the sum of the evaluator's kernel and copy times from torch.profiler (a run of its own).
The numpy restatement of pycocotools (tests/_coco_eval_ref.py) is timed on a 5,000-image set of the same kind, whose
device result is checked against it. The GPU's name and power limit are read in the same run.

    python tools/coco_eval_time.py --out profiles/h100_coco_eval.json
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    name, power, sm = [s.strip() for s in q.stdout.strip().splitlines()[0].split(",")]
    return {"gpu": name, "power_limit": power, "sm_max_clock": sm}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=40504)
    ap.add_argument("--oracle-images", type=int, default=5000)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()

    import torch
    import multipathnet_b200 as mpn
    from multipathnet_b200 import coco_eval as CE, workloads as wl
    import _coco_eval_ref as R

    info = gpu_info()
    ctx = mpn.Context(0)
    res = {"tool": "tools/coco_eval_time.py", **info}

    t0 = time.perf_counter()
    gt_json, rows = wl.coco_eval_set(a.images, 80, 7, 100, a.seed)
    gt = CE.CocoGroundTruth.from_dict(gt_json)
    res["set"] = {"images": a.images, "categories": 80, "annotations": int(len(gt.gt_img)), "rows": int(rows.shape[0]),
                  "build_s": round(time.perf_counter() - t0, 2)}

    out = CE.coco_evaluate(ctx, gt, rows)                     # warm-up: module load, scratch allocation
    host = []
    for _ in range(a.reps):
        t = time.perf_counter()
        again = CE.coco_evaluate(ctx, gt, rows)
        host.append((time.perf_counter() - t) * 1e3)
        assert all(np.array_equal(out[k], again[k]) for k in out)
    ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    stream = torch.cuda.ExternalStream(ctx.stream_handle) if ctx.stream_handle else torch.cuda.default_stream()
    spans = []
    for _ in range(a.reps):
        ev0.record(stream)
        CE.coco_evaluate(ctx, gt, rows)
        ev1.record(stream)
        ev1.synchronize()
        spans.append(ev0.elapsed_time(ev1))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        CE.coco_evaluate(ctx, gt, rows)
        torch.cuda.synchronize()
    kern, copy = {}, 0.0
    for e in prof.events():
        if e.device_type.name != "CUDA":
            continue
        us = e.device_time if hasattr(e, "device_time") else e.cuda_time
        if "Memcpy" in e.name or "Memset" in e.name:
            copy += us / 1e3
        else:
            short = e.name.split("::")[-1].split("(")[0].split("<")[0]
            kern[short] = kern.get(short, 0.0) + us / 1e3
    res["full"] = {"host_ms_median": round(statistics.median(host), 2), "host_ms": [round(x, 2) for x in host],
                   "event_span_ms_median": round(statistics.median(spans), 2),
                   "kernel_ms_sum": round(sum(kern.values()), 3), "copy_ms_sum": round(copy, 3),
                   "kernel_ms": {k: round(v, 3) for k, v in sorted(kern.items(), key=lambda kv: -kv[1])},
                   "stats": [round(float(s), 6) for s in out["stats"]], "launches_per_call": None}
    n0 = ctx.launch_count
    CE.coco_evaluate(ctx, gt, rows)
    res["full"]["launches_per_call"] = ctx.launch_count - n0

    gt_s, rows_s = wl.coco_eval_set(a.oracle_images, 80, 7, 100, a.seed + 1)
    g_s = CE.CocoGroundTruth.from_dict(gt_s)
    dev = CE.coco_evaluate(ctx, g_s, rows_s)
    t = time.perf_counter()
    dev = CE.coco_evaluate(ctx, g_s, rows_s)
    dev_ms = (time.perf_counter() - t) * 1e3
    t = time.perf_counter()
    p, r, s = R.cocoeval(gt_s, rows_s)
    orc_s = time.perf_counter() - t
    res["subset"] = {"images": a.oracle_images, "rows": int(rows_s.shape[0]), "oracle_s": round(orc_s, 2), "device_host_ms": round(dev_ms, 2),
                     "precision_bit_equal": bool(np.array_equal(dev["precision"], p)), "recall_bit_equal": bool(np.array_equal(dev["recall"], r)),
                     "stats_max_abs_diff": float(np.max(np.abs(dev["stats"] - s)))}
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    ctx.close()


if __name__ == "__main__":
    main()

"""Times the inn.ROIPooling module ops on the GPU: the forward (mpn_roi_pool_dev) and the backward
(mpn_roi_pool_backward_dev) on device buffers, at the S3, S4 and R1000 shapes of workloads.ROI_POOL_CASES (variant 2).
Each op: CUDA events around --iters back-to-back launches after --warmup launches. The backward's achieved GB/s counts
its algorithmic bytes: grad_out and argmax read once, grad_data written once. Prints one JSON line, with the GPU's name
and power limit read in the same run.      python tools/roi_backward_time.py [--iters 200] [--warmup 10]"""
import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import workloads as wl


def gpu_info():
    """name, power limit and max SM clock of GPU 0 (read-only nvidia-smi query)"""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30, check=True).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit_w": float(q[1]), "sm_max_mhz": float(q[2])}
    except (OSError, subprocess.SubprocessError, IndexError, ValueError) as e:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None, "nvidia_smi": str(e)}


def time_ms(fn, iters, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(iters):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=10)
    args = ap.parse_args()
    if args.iters < 100:
        raise SystemExit("--iters must be at least 100")
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    ctx = mpn.Context(0)                     # the legacy default stream: the same stream torch's events are recorded on
    lib, variant = ctx.lib, 2
    res = {"tool": "roi_backward_time", "variant": variant, "iters": args.iters, "warmup": args.warmup, **gpu_info(), "cases": {}}
    for name in ("S3", "S4", "R1000"):
        fm, rois, P, scale = wl.roi_pool_case(name, foveal=ctx.foveal)
        N, C, H, W = fm.shape
        R = rois.shape[0]
        fm_d, r_d = torch.from_numpy(fm).cuda(), torch.from_numpy(rois).cuda()
        out_d = torch.empty((R, C, P, P), dtype=torch.float32, device="cuda")
        am_d = torch.empty((R, C, P, P), dtype=torch.int32, device="cuda")
        g_d = torch.from_numpy(np.random.default_rng(1).standard_normal((R, C, P, P), dtype=np.float32)).cuda()
        gd_d = torch.empty((N, C, H, W), dtype=torch.float32, device="cuda")

        def fwd():
            ctx.check(lib.mpn_roi_pool_dev(ctx.h, fm_d.data_ptr(), N, C, H, W, r_d.data_ptr(), R, P, P, scale, variant,
                                           out_d.data_ptr(), am_d.data_ptr()), "mpn_roi_pool_dev")

        def bwd():
            ctx.roi_pool_backward_dev(g_d, am_d, N, C, H, W, r_d, R, P, P, scale, variant, gd_d)

        fwd_ms = time_ms(fwd, args.iters, args.warmup)     # leaves the argmax the backward reads
        bwd_ms = time_ms(bwd, args.iters, args.warmup)
        nbytes = R * C * P * P * (4 + 4) + N * C * H * W * 4
        res["cases"][name] = {"shape": [N, C, H, W], "R": R, "pooled": P, "scale": scale,
                              "forward_us": round(1e3 * fwd_ms, 2), "backward_us": round(1e3 * bwd_ms, 2),
                              "backward_bytes": nbytes, "backward_gbps": round(nbytes / (bwd_ms * 1e-3) / 1e9, 1)}
    ctx.close()
    print(json.dumps(res))


if __name__ == "__main__":
    main()

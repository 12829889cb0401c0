"""Times the first layer of the VGG-16 trunk (conv1_1: 3x3, Cin 3, Cout 64, pad 1) on a device-resident
1 x 3 x H x W image, and prints one JSON line.

Three numbers, each from its own loop of --steps trunk forwards (mpn_model_trunk_dev) after --warmup:
  trunk_ms_per_step       CUDA events around the loop, profiling off (the whole trunk: conv1_1 + the wgmma layers)
  conv_direct_ms_per_step the per-category profile (ctx.profile_begin / profile_end); in the trunk the conv_direct
                          category holds conv1_1 and nothing else. records_per_step is the number of event pairs
                          the category recorded per step.
  kernel_us_per_launch    torch.profiler (CUDA activities) over the loop: mean device time of the first-layer kernel
The output the layer must write (H x W x 64 channels x hi + lo bf16 planes) over the kernel time gives its store
bandwidth, stated against the 3.35 TB/s HBM3 figure of the H100 SXM data sheet. The GPU's name, power limit and SM
clocks are read right after the timed loop.
    python tools/conv1_time.py [--steps 200] [--warmup 20] [--H 600] [--W 800] [--out FILE]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_PEAK_GBS = 3350.0     # H100 SXM data sheet, not measured


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
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--H", type=int, default=600)
    ap.add_argument("--W", type=int, default=800)
    ap.add_argument("--out", default=None, help="also append the JSON line to this file")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    import multipathnet_b200 as mpn
    from multipathnet_b200 import models, workloads as wl

    H, W = args.H, args.W
    ctx = mpn.Context(0)                  # the legacy default stream: the one torch's events below are recorded on
    spec = models.vgg16_fast_rcnn(21, seed=1234)
    m = mpn.Model(ctx, spec, max_rois=64, max_h=H, max_w=W)
    img = torch.from_numpy(wl.transform(wl.raw_image(H, W, 2), spec.transformer)).cuda().contiguous()

    def step():
        ctx.check(ctx.lib.mpn_model_trunk_dev(m.h, img.data_ptr(), H, W), "mpn_model_trunk_dev")

    for _ in range(args.warmup):
        step()
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(args.steps):
        step()
    b.record()
    b.synchronize()
    info = gpu_info()
    trunk_ms = a.elapsed_time(b) / args.steps

    ctx.profile_begin()
    for _ in range(args.steps):
        step()
    prof = ctx.profile_end()

    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as tp:
        for _ in range(args.steps):
            step()
        torch.cuda.synchronize()
    kern = {}
    for e in tp.events():
        if e.device_type == torch.autograd.DeviceType.CUDA and "conv1" in e.name:
            t = kern.setdefault(e.name, [0.0, 0])
            t[0] += e.device_time
            t[1] += 1
    if len(kern) != 1:
        raise SystemExit(f"expected one first-layer kernel in the trace, found {sorted(kern)}")
    kname, (kus, kn) = next(iter(kern.items()))
    us = kus / kn
    out_bytes = H * W * 64 * 2 * 2
    in_bytes = 3 * H * W * 4
    line = {"tool": "conv1_time", "H": H, "W": W, "steps": args.steps, "warmup": args.warmup, **info,
            "trunk_ms_per_step": trunk_ms,
            "conv_direct_ms_per_step": prof["conv_direct"][0] / args.steps,
            "conv_direct_records_per_step": prof["conv_direct"][1] / args.steps,
            "kernel": kname, "kernel_launches": kn, "kernel_us_per_launch": us,
            "output_bytes": out_bytes, "input_bytes": in_bytes,
            "output_gbs": out_bytes / (us * 1e-6) / 1e9,
            "hbm_floor_us": (out_bytes + in_bytes) / (HBM_PEAK_GBS * 1e9) * 1e6,
            "frac_of_hbm_peak": (out_bytes + in_bytes) / (us * 1e-6) / 1e9 / HBM_PEAK_GBS,
            "hbm_peak_source": "H100 SXM data sheet (3.35 TB/s), not measured"}
    print(json.dumps(line), flush=True)
    if args.out:
        with open(args.out, "a") as f:
            f.write(json.dumps(line) + "\n")
    m.close(); ctx.close()


if __name__ == "__main__":
    main()

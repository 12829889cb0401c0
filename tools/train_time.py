"""Times the training step of the per-ROI layers (mpn_model_train_step_dev) at the full-size shape: vgg16_multipathnet(81),
two images of 600 x 800 and 600 x 900, 128 ROIs each. The whole step: CUDA events around --iters back-to-back steps after
--warmup steps. Its phases: the library's own events inside each step (mpn_model_train_phase_ms: trunks + ROI pooling,
per-ROI forward + criteria, backward, update), medians over --iters more steps. The algorithmic work is counted from the
shapes: the per-ROI forward FLOPs, the backward GEMMs' FLOPs (dW for every trained layer, dX wherever a trained layer lies
below) over the backward phase's time, and the bytes the fused update moves over the update phase's time, both against
the H100 SXM data sheet (989 TFLOP/s dense bf16, 3.35 TB/s). Writes profiles/h100_train.json (or --out) with the GPU's
name and power limit read in the same run.      python tools/train_time.py [--iters 20] [--warmup 3]"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl


def gpu_info():
    """name, power limit and max SM clock of GPU 0 (read-only nvidia-smi query)"""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30, check=True).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit_w": float(q[1]), "sm_max_mhz": float(q[2])}
    except (OSError, subprocess.SubprocessError, IndexError, ValueError) as e:
        return {"gpu": torch.cuda.get_device_name(0), "power_limit_w": None, "sm_max_mhz": None, "nvidia_smi": str(e)}


def counted(spec, R):
    """(per-ROI forward FLOPs, backward GEMM FLOPs, update bytes) at R rows, from the shapes. The update as built: per weight
    element it reads w, g, buf and writes w, buf (fp32) and the hi / lo planes (2 x 2 bytes), plus the transposed hi / lo
    planes (2 x 2 bytes) of layers with a dX GEMM; per bias element 20 bytes."""
    fwd = bwd = upd = 0.0
    for T in spec.towers:
        first = True
        bins = T.pooled_h * T.pooled_w
        flat = False
        for L in T.layers:
            if L.kind == mpn._lib.MPN_LAYER_FLATTEN:
                flat = True
                continue
            rows = R * (1 if flat else bins)
            mac = float(rows) * L.cin * L.cout
            fwd += 2 * mac
            bwd += 2 * mac * (1 if first else 2)              # dW; dX too unless nothing trained lies below
            upd += L.cin * L.cout * (24 + (0 if first else 4)) + L.cout * 20
            first = False
    for h in (spec.cls_heads[0], spec.bbox_head):
        mac = float(R) * h.col_len * h.cout
        fwd += 2 * mac; bwd += 4 * mac
        upd += h.col_len * h.cout * 28 + h.cout * 20
    return fwd, bwd, upd


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_train.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    ctx = mpn.Context(0)                                   # the legacy default stream: torch's events are recorded on it
    spec = models.vgg16_multipathnet(81, seed=1234)
    m = mpn.Model(ctx, spec, max_rois=256, max_h=608, max_w=912)
    tr = mpn.Trainer(m)
    sizes, per = ((600, 800), (600, 900)), (128, 128)
    rng = np.random.default_rng(0)
    ims = [torch.from_numpy(wl.transform(wl.raw_image(h, w, i), spec.transformer)).cuda() for i, (h, w) in enumerate(sizes)]
    boxes = torch.from_numpy(np.concatenate([wl.random_boxes(n, h, w, i) for i, ((h, w), n) in enumerate(zip(sizes, per))]).astype(np.float32)).cuda()
    R, C = sum(per), spec.num_classes
    labels = torch.from_numpy(rng.integers(1, C + 1, R).astype(np.int32)).cuda()
    tg = torch.zeros((R, 4 * C), dtype=torch.float32, device="cuda")
    losses = torch.zeros(3, dtype=torch.float32, device="cuda")
    import ctypes as Cc
    ptrs = (Cc.c_void_p * 2)(*[im.data_ptr() for im in ims])
    hw = np.array([600, 800, 600, 900], np.int32); cnt = np.array(per, np.int32)

    def step():
        ctx.check(ctx.lib.mpn_model_train_step_dev(m.h, 2, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
                                                   boxes.data_ptr(), labels.data_ptr(), tg.data_ptr(), losses.data_ptr()), "train_step_dev")

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

    step_ms = time_ms(step, args.iters, args.warmup)
    ctx.synchronize()
    finite = bool(torch.isfinite(losses).all())
    phases = []
    ms = np.zeros(4, np.float32)
    for _ in range(args.iters):
        step()
        ctx.check(ctx.lib.mpn_model_train_phase_ms(m.h, ms.ctypes.data_as(mpn._lib._f32p)), "train_phase_ms")
        phases.append(ms.copy())
    ph = np.median(np.stack(phases), 0)
    fwd, bwd, upd = counted(spec, R)
    res = {"tool": "train_time", **gpu_info(), "shape": "vgg16_multipathnet(81), 600x800 + 600x900, 128 ROIs each",
           "R": R, "iters": args.iters, "warmup": args.warmup, "step_ms": round(step_ms, 3), "losses_finite": finite,
           "phase_ms_median": {"trunk_pool": round(float(ph[0]), 3), "forward_criteria": round(float(ph[1]), 3),
                               "backward": round(float(ph[2]), 3), "update": round(float(ph[3]), 3)},
           "per_roi_forward_tflop_counted": round(fwd / 1e12, 4), "backward_gemm_tflop_counted": round(bwd / 1e12, 4),
           "update_gb_counted": round(upd / 1e9, 2),
           "backward_tflops": round(bwd / 1e12 / (float(ph[2]) / 1e3), 1),
           "backward_frac_of_989": round(bwd / 1e12 / (float(ph[2]) / 1e3) / 989.0, 3),
           "update_gbps": round(upd / 1e9 / (float(ph[3]) / 1e3), 1),
           "update_frac_of_3350": round(upd / 1e9 / (float(ph[3]) / 1e3) / 3350.0, 3),
           "note": "backward rate = counted GEMM FLOPs over the whole backward phase (gates, transposes, bias sums included); "
                   "update rate = counted bytes over the update phase; data-sheet peaks, not measured ones"}
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(res) + "\n")
    print(json.dumps(res))
    tr.close(); m.close(); ctx.close()


if __name__ == "__main__":
    main()

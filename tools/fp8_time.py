"""Times the device-resident detect+NMS step (mpn_model_detect_nms_dev) in the default numerics, the opt-in bf16
numerics (mpn_ctx_set_option "bf16" = 1) and the opt-in fp8 numerics ("fp8" = 1), for the three detection configs of
bench.py (cfg 2 vgg16_frcnn, cfg 3 multipathnet, cfg 4 resnet50), and writes one JSON line per config.

Every run is its own process (a fresh context and model); the modes alternate default / bf16 / fp8 --reps times per
config. A run times --steps steps with CUDA events after --warmup steps, then the same number of steps under the
per-category profile (conv_gemm_tc = the wgmma engine, fp8_quantize = the fp8 operand quantizer), and reads the GPU's
name, power limit and SM clocks right after the timed loop. The score / box distance of a mode to the default is the
normwise max|mode - default| / max|default| of the last step.
    python tools/fp8_time.py [--steps 200] [--warmup 20] [--reps 2] [--out profiles/h100_fp8.json]"""
import argparse
import json
import os
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np

CONFIGS = {   # the workloads of bench.py
    "vgg16_frcnn": dict(cfg=2, H=600, W=800, R=1000, C=21, boxes="random", model="vgg16_fast_rcnn", kw={}),
    "multipathnet": dict(cfg=3, H=600, W=800, R=1000, C=81, boxes="sharpmask", model="vgg16_multipathnet", kw={}),
    "resnet50": dict(cfg=4, H=800, W=1000, R=2000, C=81, boxes="sharpmask", model="resnet50_fast_rcnn", kw={"integral_k": 6}),
}


def gpu_info():
    """name, power limit and SM clocks of GPU 0 (read-only nvidia-smi query)"""
    try:
        q = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader,nounits"],
                           capture_output=True, text=True, timeout=30, check=True).stdout.strip().split(", ")
        return {"gpu": q[0], "power_limit_w": float(q[1]), "sm_mhz": float(q[2]), "sm_max_mhz": float(q[3])}
    except (OSError, subprocess.SubprocessError, IndexError, ValueError) as e:
        return {"gpu": None, "power_limit_w": None, "sm_mhz": None, "sm_max_mhz": None, "nvidia_smi": str(e)}


MODES = ("default", "bf16", "fp8")


def child(name, mode, steps, warmup, dump):
    import torch
    import multipathnet_b200 as mpn
    from multipathnet_b200 import models, workloads as wl
    c = CONFIGS[name]
    H, W, R, C = c["H"], c["W"], c["R"], c["C"]
    ctx = mpn.Context(0)                 # the legacy default stream: the one torch's events below are recorded on
    if mode != "default":
        ctx.set_option(mode, 1)
    spec = getattr(models, c["model"])(C, seed=1234, **c["kw"])
    m = mpn.Model(ctx, spec, max_rois=R + 48, max_h=H + 8, max_w=W)
    boxes_fn = wl.sharpmask_boxes if c["boxes"] == "sharpmask" else wl.random_boxes
    imgs = [torch.from_numpy(wl.transform(wl.raw_image(H, W, s), spec.transformer)).cuda() for s in (2, 3)]
    boxes = [torch.from_numpy(boxes_fn(R, H, W, s)).cuda() for s in (2, 3)]
    sc = torch.empty((R, C), dtype=torch.float32, device="cuda")
    bb = torch.empty((R, 4 * C), dtype=torch.float32, device="cuda")
    kp = torch.empty((C - 1, R), dtype=torch.int32, device="cuda")
    ct = torch.empty((C - 1,), dtype=torch.int32, device="cuda")

    def step(i):
        m.detect_nms_dev(imgs[i % 2], H, W, boxes[i % 2], R, 1.0, W, H, -1.5, 0.3, sc, bb, kp, ct)

    for i in range(warmup):
        step(i)
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        step(i)
    b.record()
    b.synchronize()
    info = gpu_info()
    ms = a.elapsed_time(b) / steps
    ctx.profile_begin()
    for i in range(steps):
        step(i)
    prof = ctx.profile_end()
    torch.cuda.synchronize()
    np.save(os.path.join(dump, "scores.npy"), sc.cpu().numpy())       # last step: image / boxes seed 3
    np.save(os.path.join(dump, "bboxes.npy"), bb.cpu().numpy())
    m.close(); ctx.close()
    return {"ms_per_step": ms, "conv_gemm_tc_ms_per_step": prof["conv_gemm_tc"][0] / steps,
            "fp8_quantize_ms_per_step": prof["fp8_quantize"][0] / steps, **info}


def rel(a, b):
    return float(np.max(np.abs(a.astype(np.float64) - b)) / max(float(np.max(np.abs(b))), 1e-30))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200)
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--reps", type=int, default=2)
    ap.add_argument("--configs", default=",".join(CONFIGS))
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_fp8.json"))
    ap.add_argument("--child", nargs=3, metavar=("CONFIG", "MODE", "DUMP_DIR"), help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.child:
        print(json.dumps(child(args.child[0], args.child[1], args.steps, args.warmup, args.child[2])))
        return
    if args.steps < 200 or args.reps < 2:
        raise SystemExit("--steps must be at least 200 and --reps at least 2")
    out_f = open(args.out, "w")
    for name in args.configs.split(","):
        runs = {mode: [] for mode in MODES}
        with tempfile.TemporaryDirectory() as tmp:
            for rep in range(args.reps):
                for mode in MODES:
                    d = os.path.join(tmp, mode)
                    os.makedirs(d, exist_ok=True)
                    out = subprocess.run([sys.executable, os.path.abspath(__file__), "--steps", str(args.steps), "--warmup",
                                          str(args.warmup), "--child", name, mode, d],
                                         capture_output=True, text=True, check=True).stdout
                    runs[mode].append(json.loads(out.strip().splitlines()[-1]))
            dist = {f"{k}_{mode}_vs_default": rel(np.load(os.path.join(tmp, mode, f"{k}.npy")), np.load(os.path.join(tmp, "default", f"{k}.npy")))
                    for mode in MODES[1:] for k in ("scores", "bboxes")}
        keys = ("ms_per_step", "conv_gemm_tc_ms_per_step", "fp8_quantize_ms_per_step")
        med = {mode: {k: float(np.median([r[k] for r in rs])) for k in keys} for mode, rs in runs.items()}
        fp8_engine = med["fp8"]["conv_gemm_tc_ms_per_step"] + med["fp8"]["fp8_quantize_ms_per_step"]
        line = {"tool": "fp8_time", "config": name, "cfg": CONFIGS[name]["cfg"], "steps": args.steps, "warmup": args.warmup,
                "gpu": runs["default"][0]["gpu"], "power_limit_w": runs["default"][0]["power_limit_w"],
                "runs": runs, "median": med,
                "step_speedup_fp8_vs_bf16": med["bf16"]["ms_per_step"] / med["fp8"]["ms_per_step"],
                "step_speedup_fp8_vs_default": med["default"]["ms_per_step"] / med["fp8"]["ms_per_step"],
                "engine_speedup_fp8_vs_bf16": med["bf16"]["conv_gemm_tc_ms_per_step"] / fp8_engine, **dist}
        print(json.dumps(line), flush=True)
        out_f.write(json.dumps(line) + "\n")
        out_f.flush()
    out_f.close()


if __name__ == "__main__":
    main()

"""Times CaffeNet Fast R-CNN (models.alexnet_fast_rcnn(21)) on the device, every input and output a CUDA tensor:
  * device-resident detect + NMS (mpn_model_detect_nms_dev: one image of 600 x 1000) with 1000 and with 2000 ROIs (2000:
    the VOC 2007 scripts' proposal count), default (BF16X3) and bf16 numerics, their rounds alternated; CUDA events on
    the library's stream, medians of --rounds;
  * the trunk alone (mpn_model_trunk_dev), its FLOPs counted from the layer table (a grouped convolution's divided by
    its groups);
  * each kernel of one trunk pass (torch.profiler, CUDA activities, in a pass of its own after the timed rounds): conv2,
    conv4 and conv5 as their G engine launches with TFLOP/s counted from the shapes, and the two LRN launches with the
    bytes they move counted from the shapes against the H100 SXM data sheet's 3.35 TB/s.
conv2's groups read 48 channels: the engine pads K to 64 per tap, so a quarter of its MMA work is padding; its TFLOP/s
counts the useful FLOPs only. Writes profiles/h100_caffenet.json (or --out) with the GPU's name, power limit and max SM
clock, read in the same run.
    python tools/caffenet_time.py [--rounds 5] [--iters 10] [--warmup 2]"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200._lib import MPN_LAYER_CONV, MPN_LAYER_LRN
from tools.train_time import gpu_info

H, W, C = 600, 1000, 21
MODES = {"default": -1, "bf16": 1}
HBM_TBPS = 3.35


def trunk_shapes(spec):
    """(c, h, w) of every trunk slot at H x W"""
    shp = {0: (3, H, W)}
    for L in spec.trunk_layers:
        c, h, w = shp[L.in_slot]
        if L.kind == MPN_LAYER_CONV:
            shp[L.out_slot] = (L.cout, (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1)
        elif L.kind == MPN_LAYER_LRN:
            shp[L.out_slot] = (c, h, w)
        else:
            shp[L.out_slot] = (c, models._pool_out(h, L.kh, L.stride, L.pad, L.ceil_mode), models._pool_out(w, L.kw, L.stride, L.pad, L.ceil_mode))
    return shp


def trunk_kernels(ctx, m, img):
    """device time (ms) of every kernel of one trunk pass, in launch order: [(name, ms)]"""
    from torch.profiler import ProfilerActivity, profile
    ctx.check(ctx.lib.mpn_model_trunk_dev(m.h, img.data_ptr(), H, W), "trunk_dev")
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        ctx.check(ctx.lib.mpn_model_trunk_dev(m.h, img.data_ptr(), H, W), "trunk_dev")
        torch.cuda.synchronize()
    ev = [e for e in p.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name and "Memset" not in e.name]
    ev.sort(key=lambda e: e.time_range.start)
    return [(e.name, e.time_range.elapsed_us() / 1e3) for e in ev]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_caffenet.json"))
    a = ap.parse_args()
    assert torch.cuda.is_available(), "no GPU: nothing to measure"

    def time_ms(fn):
        for _ in range(a.warmup):
            fn()
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.iters):
            fn()
        e1.record()
        e1.synchronize()
        return e0.elapsed_time(e1) / a.iters

    ctx = mpn.Context(0)
    spec = models.alexnet_fast_rcnn(C, seed=1234)
    shp = trunk_shapes(spec)
    out = {"card": gpu_info(), "workload": f"alexnet_fast_rcnn({C}), {H} x {W}, device-resident", "rounds": a.rounds,
           "iters": a.iters, "timing": "CUDA events on the library's stream, median of the rounds; per-kernel times from "
                                       "torch.profiler in a separate pass",
           "flops": {"trunk_gflop": models.trunk_flops(spec, H, W) / 1e9, "per_roi_gflop": models.head_flops_per_roi(spec) / 1e9}}
    img = torch.from_numpy(wl.transform(wl.raw_image(H, W, 0), spec.transformer)).cuda()
    lib = ctx.lib
    res = {}
    for R in (1000, 2000):
        boxes = torch.from_numpy(wl.random_boxes(R, H, W, 0).astype(np.float32)).cuda()
        sc = torch.empty((R, C), dtype=torch.float32, device="cuda")
        bb = torch.empty((R, 4 * C), dtype=torch.float32, device="cuda")
        kp = torch.empty((C - 1, R), dtype=torch.int32, device="cuda")
        ct = torch.empty((C - 1,), dtype=torch.int32, device="cuda")
        mdl = {}
        for k, v in MODES.items():
            ctx.set_option("bf16", v)
            mdl[k] = mpn.Model(ctx, spec, max_rois=R, max_h=H, max_w=W)
        r = {k: {"detect_nms_ms": [], "trunk_ms": []} for k in MODES}
        for _ in range(a.rounds):
            for k, v in MODES.items():
                ctx.set_option("bf16", v)
                m = mdl[k]
                r[k]["detect_nms_ms"].append(time_ms(lambda: m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, sc, bb, kp, ct)))
                r[k]["trunk_ms"].append(time_ms(lambda: ctx.check(lib.mpn_model_trunk_dev(m.h, img.data_ptr(), H, W), "trunk_dev")))
        for k, v in MODES.items():
            e = {q: float(np.median(x)) for q, x in r[k].items()}
            e["rounds"] = r[k]
            e["trunk_tflops"] = out["flops"]["trunk_gflop"] / e["trunk_ms"]            # GFLOP / ms = TFLOP/s
            if R == 1000:
                ctx.set_option("bf16", v)
                ks = trunk_kernels(ctx, mdl[k], img)
                e["trunk_kernels"] = [(n[:60], round(ms, 4)) for n, ms in ks]
                conv = [ms for n, ms in ks if "conv_gemm_tc" in n]
                lrn = [ms for n, ms in ks if "lrn_split" in n]
                # trunk engine launches in order: conv2 x 2, conv3, conv4 x 2, conv5 x 2 (conv1 runs on the direct kernel)
                layers = {}
                if len(conv) == 7:
                    for name, idx, li in (("conv2", (0, 1), 3), ("conv3", (2,), 6), ("conv4", (3, 4), 7), ("conv5", (5, 6), 8)):
                        L = spec.trunk_layers[li]
                        _, h, w = shp[L.out_slot]
                        fl = 2.0 * (L.cin // L.groups) * L.cout * L.kh * L.kw * h * w
                        ms = sum(conv[i] for i in idx)
                        layers[name] = {"launches_ms": [conv[i] for i in idx], "ms": ms, "gflop": fl / 1e9, "tflops": fl / 1e9 / ms}
                    layers["conv2"]["note"] = "48-channel groups: K padded to 64 per tap, a quarter of the MMA work is padding"
                if len(lrn) == 2:
                    for name, li, ms in (("norm1", 2, lrn[0]), ("norm2", 5, lrn[1])):
                        c, h, w = shp[spec.trunk_layers[li].in_slot]
                        byts = 2 * 4.0 * c * h * w                     # read hi + lo, write hi + lo: 2 bytes each
                        layers[name] = {"ms": ms, "mbytes": byts / 1e6, "tbytes_per_s": byts / (ms / 1e3) / 1e12,
                                        "share_of_3.35_tbps": byts / (ms / 1e3) / 1e12 / HBM_TBPS}
                e["layers"] = layers
            res[f"R{R}/{k}"] = e
        for m in mdl.values():
            m.close()
    ctx.set_option("bf16", -1)
    out["results"] = res
    ctx.close()
    os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(json.dumps(out) + "\n")
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

"""Times Inception-v3 Fast R-CNN (models.inception_v3_fast_rcnn(21)) on the device, every input and output a CUDA tensor and
every time between CUDA events on the stream the library runs on (the legacy default stream of mpn.Context(0)):
  * device-resident detect + NMS (mpn_model_detect_nms_dev: one image of 600 x 1000) with 1000 and with 400 ROIs (400:
    the COCO eval recipe's test_best_proposals_number), default (BF16X3) and bf16 numerics, their rounds alternated;
  * the trunk alone (mpn_model_trunk_dev) and the per-ROI part alone (mpn_model_heads_dev: ROI pooling, Mixed_7a..7c,
    the average pool, the heads), with their FLOPs counted from the layer table;
  * per category of one 1000-ROI detect (mpn_ctx_profile): the engine's share, and the pools' (windowed average and
    max pools share the "pool" category) with the bytes they move counted from shapes;
  * the device memory the process holds after a 1000-ROI detect (cudaMemGetInfo: total - free).
Medians over --rounds; writes profiles/h100_inception.json (or --out) with the GPU's name, power limit and max SM clock.
    python tools/inception_time.py [--rounds 5] [--iters 10] [--warmup 2]"""
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
from multipathnet_b200._lib import MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_CONV, MPN_LAYER_MAXPOOL
from tools.train_time import gpu_info

H, W, C = 600, 1000, 21
MODES = {"default": -1, "bf16": 1}


def pool_bytes(spec, R):
    """bytes the windowed average and max pools of one detect read and write (split planes: 4 bytes per element), from shapes"""
    tot = 0.0
    for layers, shp in ((spec.trunk_layers, {0: (3, H, W)}), (spec.towers[0].layers, {0: (768, 17, 17)})):
        n = 1 if layers is spec.trunk_layers else R
        for L in layers:
            c, h, w = shp[L.in_slot]
            if L.kind == MPN_LAYER_CONV:
                oh, ow, oc = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.padw - L.kw) // L.stride + 1, L.cout
            elif L.kind in (MPN_LAYER_MAXPOOL, MPN_LAYER_AVGPOOL_WIN):
                oh, ow, oc = models._pool_out(h, L.kh, L.stride, L.pad, 0), models._pool_out(w, L.kw, L.stride, L.pad, 0), c
                tot += 4.0 * n * (c * h * w + oc * oh * ow)
            else:
                oh, ow, oc = 1, 1, c
            shp[L.out_slot] = (L.out_c_total or oc, oh, ow)
    return tot


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_inception.json"))
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
    spec = models.inception_v3_fast_rcnn(C, seed=1234)
    free0, total = torch.cuda.mem_get_info()
    out = {"card": gpu_info(), "workload": f"inception_v3_fast_rcnn({C}), {H} x {W}, device-resident", "rounds": a.rounds,
           "iters": a.iters, "timing": "CUDA events on the library's stream, median of the rounds",
           "flops": {"trunk_gflop": models.trunk_flops(spec, H, W) / 1e9, "per_roi_gflop": models.head_flops_per_roi(spec) / 1e9},
           "not_measured": ["the 1 x n / n x 1 layers' own share (no per-layer timing; they run in the conv_gemm_tc category)",
                            "avgpool_win_kernel apart from the max pools (both report as the pool category)"]}
    img = torch.from_numpy(wl.transform(wl.raw_image(H, W, 0), spec.transformer)).cuda()
    lib = ctx.lib
    res = {}
    for R in (1000, 400):
        boxes_np = wl.random_boxes(R, H, W, 0).astype(np.float32)
        boxes = torch.from_numpy(boxes_np).cuda()
        rois = torch.from_numpy(np.concatenate([np.ones((R, 1), np.float32), boxes_np], 1)).cuda()
        sc = torch.empty((R, C), dtype=torch.float32, device="cuda")
        bb = torch.empty((R, 4 * C), dtype=torch.float32, device="cuda")
        kp = torch.empty((C - 1, R), dtype=torch.int32, device="cuda")
        ct = torch.empty((C - 1,), dtype=torch.int32, device="cuda")
        mdl = {}
        for k, v in MODES.items():
            ctx.set_option("bf16", v)
            mdl[k] = mpn.Model(ctx, spec, max_rois=R, max_h=H, max_w=W)
        r = {k: {"detect_nms_ms": [], "trunk_ms": [], "per_roi_ms": []} for k in MODES}
        for _ in range(a.rounds):
            for k, v in MODES.items():
                ctx.set_option("bf16", v)
                m = mdl[k]
                r[k]["detect_nms_ms"].append(time_ms(lambda: m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, sc, bb, kp, ct)))
                r[k]["trunk_ms"].append(time_ms(lambda: ctx.check(lib.mpn_model_trunk_dev(m.h, img.data_ptr(), H, W), "trunk_dev")))
                r[k]["per_roi_ms"].append(time_ms(lambda: ctx.check(lib.mpn_model_heads_dev(m.h, rois.data_ptr(), R, sc.data_ptr(),
                                                                                              bb.data_ptr()), "heads_dev")))
        for k, v in MODES.items():
            ctx.set_option("bf16", v)
            m = mdl[k]
            e = {q: float(np.median(x)) for q, x in r[k].items()}
            e["rounds"] = r[k]
            e["trunk_tflops"] = out["flops"]["trunk_gflop"] / e["trunk_ms"]            # GFLOP / ms = TFLOP/s
            e["per_roi_tflops"] = out["flops"]["per_roi_gflop"] * R / e["per_roi_ms"]
            if R == 1000:
                m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, sc, bb, kp, ct)
                torch.cuda.synchronize()
                ctx.profile_begin()
                m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, sc, bb, kp, ct)
                prof = ctx.profile_end()
                e["profile_ms"] = {c: round(ms, 4) for c, (ms, n) in prof.items() if n}
                pb = pool_bytes(spec, R)
                e["pool_share"] = prof["pool"][0] / sum(ms for ms, _ in prof.values())
                e["pool_gbytes"] = pb / 1e9
                e["pool_tbytes_per_s"] = pb / (prof["pool"][0] / 1e3) / 1e12
                e["conv_gemm_tc_share"] = prof["conv_gemm_tc"][0] / sum(ms for ms, _ in prof.values())
            res[f"R{R}/{k}"] = e
        if R == 1000:
            torch.cuda.synchronize()
            free1, _ = torch.cuda.mem_get_info()
            out["device_memory_gb_two_models_1000_rois"] = (free0 - free1) / 1e9
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

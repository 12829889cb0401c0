"""Times Network-in-Network Fast R-CNN (models.nin_fast_rcnn(21)) on the device, every input and output a CUDA tensor and
every time between CUDA events on the stream the library runs on (the legacy default stream of mpn.Context(0)):
  * device-resident detect + NMS (mpn_model_detect_nms_dev: one image of 600 x 1000, 1000 ROIs) in the default (BF16X3)
    and the bf16 numerics, their rounds alternated;
  * the per-ROI part alone (mpn_model_heads_dev on the trunk features of one mpn_model_trunk_dev: ROI pooling, block 4,
    the average pool, the heads);
  * per category of one detect (mpn_ctx_profile: the direct first layer is the only conv_direct launch);
  * the tailed layers on the engine (mpn_conv_bench, CUDA events): block 1's 1x1 (96 -> 96 at 150 x 250) and block 2's
    5x5 (96 -> 256 at 75 x 125), each beside the same layer with 128 input channels, which costs the same K blocks: the
    tail's cost in time against its 25 % of padded MMA work;
  * one per-ROI training step (mpn_model_train_step_dev; fixed batch norm: block 4 and the heads) on the VOC recipe's
    minibatch, 2 images of 600 x 1000, 128 ROIs each, default and bf16.
Medians over --rounds; writes profiles/h100_nin.json (or --out) with the GPU's name, power limit and max SM clock.
    python tools/nin_time.py [--rounds 5] [--iters 20] [--warmup 3]"""
import argparse
import ctypes as Cc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from tools.train_time import gpu_info

H, W, R, C = 600, 1000, 1000, 21
MODES = {"default": -1, "bf16": 1}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_nin.json"))
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

    out = {"card": gpu_info(), "workload": f"nin_fast_rcnn({C}), {H} x {W}, {R} ROIs, device-resident", "rounds": a.rounds,
           "iters": a.iters, "timing": "CUDA events on the library's stream, median of the rounds"}
    ctx = mpn.Context(0)                 # the legacy default stream: the one torch's events are recorded on
    spec = models.nin_fast_rcnn(C, seed=1234)
    img = torch.from_numpy(wl.transform(wl.raw_image(H, W, 0), spec.transformer)).cuda()
    boxes_np = wl.random_boxes(R, H, W, 0).astype(np.float32)
    boxes = torch.from_numpy(boxes_np).cuda()
    rois = torch.from_numpy(np.concatenate([np.ones((R, 1), np.float32), boxes_np], 1)).cuda()   # scale 1: image coordinates
    sc = torch.empty((R, C), dtype=torch.float32, device="cuda")
    bb = torch.empty((R, 4 * C), dtype=torch.float32, device="cuda")
    kp = torch.empty((C - 1, R), dtype=torch.int32, device="cuda")
    ct = torch.empty((C - 1,), dtype=torch.int32, device="cuda")
    out["flops"] = {"trunk_gflop": models.trunk_flops(spec, H, W) / 1e9, "per_roi_block_tflop": models.head_flops_per_roi(spec) * R / 1e12}
    lib = ctx.lib
    mdl, res = {}, {k: {"detect_nms_ms": [], "per_roi_ms": []} for k in MODES}
    for k, v in MODES.items():
        ctx.set_option("bf16", v)
        mdl[k] = mpn.Model(ctx, spec, max_rois=R + 48, max_h=608, max_w=W)

    def detect(m):
        m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, sc, bb, kp, ct)

    def heads(m):
        ctx.check(lib.mpn_model_heads_dev(m.h, rois.data_ptr(), R, sc.data_ptr(), bb.data_ptr()), "heads_dev")

    for _ in range(a.rounds):
        for k, v in MODES.items():
            ctx.set_option("bf16", v)
            m = mdl[k]
            res[k]["detect_nms_ms"].append(time_ms(lambda: detect(m)))
            ctx.check(lib.mpn_model_trunk_dev(m.h, img.data_ptr(), H, W), "trunk_dev")
            res[k]["per_roi_ms"].append(time_ms(lambda: heads(m)))
    for k, v in MODES.items():
        ctx.set_option("bf16", v)
        detect(mdl[k])
        torch.cuda.synchronize()
        ctx.profile_begin()
        detect(mdl[k])
        prof = ctx.profile_end()
        r = res[k]
        out[k] = {"detect_nms_ms": float(np.median(r["detect_nms_ms"])), "per_roi_ms": float(np.median(r["per_roi_ms"])),
                  "detect_nms_ms_rounds": r["detect_nms_ms"], "per_roi_ms_rounds": r["per_roi_ms"],
                  "profile_ms": {c: round(ms, 4) for c, (ms, n) in prof.items() if n}, "first_layer_ms": prof["conv_direct"][0]}
        out[k]["per_roi_block_tflops"] = out["flops"]["per_roi_block_tflop"] / (out[k]["per_roi_ms"] / 1e3)
        mdl[k].close()
    layers = {"block1_1x1": (1, 96, 150, 250, 96, 1, 1, 0), "block2_5x5": (1, 96, 75, 125, 256, 5, 1, 2)}
    lt = {}
    for k, v in MODES.items():
        ctx.set_option("bf16", v)
        for name, (n, cin, h, w, cout, kk, s, p) in layers.items():
            t = {cin: [], 128: []}
            for _ in range(a.rounds):
                for c in (cin, 128):
                    t[c].append(ctx.conv_bench(n, c, h, w, cout, kk, s, p, iters=50)[0])
            ho, wo = (h + 2 * p - kk) // s + 1, (w + 2 * p - kk) // s + 1
            fl = 2.0 * cin * cout * kk * kk * ho * wo
            ms_t, ms_128 = float(np.median(t[cin])), float(np.median(t[128]))
            lt[f"{name}/{k}"] = {"ms": ms_t, "tflops": fl / (ms_t / 1e3) / 1e12, "ms_with_128_channels": ms_128,
                                 "ratio_to_128_channels": ms_t / ms_128, "padded_mma_share": 1 - cin / 128.0,
                                 "ms_rounds": t[cin], "ms_128_rounds": t[128]}
    out["tailed_layers"] = lt
    ctx.set_option("bf16", -1)
    # one per-ROI training step on the VOC recipe's minibatch, on device buffers
    tspec = models.nin_fast_rcnn(C, seed=1234, fixed_bn=True)
    rng = np.random.default_rng(0)
    ims = [torch.from_numpy(wl.transform(wl.raw_image(H, W, i), tspec.transformer)).cuda() for i in range(2)]
    tboxes = torch.from_numpy(np.concatenate([wl.random_boxes(128, H, W, i) for i in range(2)]).astype(np.float32)).cuda()
    labels = torch.from_numpy(rng.integers(1, C + 1, 256).astype(np.int32)).cuda()
    tg = torch.zeros((256, 4 * C), dtype=torch.float32, device="cuda")
    losses = torch.zeros(3, dtype=torch.float32, device="cuda")
    ptrs = (Cc.c_void_p * 2)(*[im.data_ptr() for im in ims])
    hw = np.array([H, W, H, W], np.int32)
    cnt = np.array([128, 128], np.int32)
    runs = {}
    for k in MODES:
        m = mpn.Model(ctx, tspec, max_rois=256, max_h=608, max_w=W)
        tr = mpn.Trainer(m, seed=1, bf16=k == "bf16")

        def step(m=m):
            ctx.check(lib.mpn_model_train_step_dev(m.h, 2, ptrs, hw.ctypes.data_as(mpn._lib._i32p), cnt.ctypes.data_as(mpn._lib._i32p),
                                                   tboxes.data_ptr(), labels.data_ptr(), tg.data_ptr(), losses.data_ptr()), "train_step_dev")
        runs[k] = (m, tr, step, [])
    for _ in range(a.rounds):
        for k in MODES:
            runs[k][3].append(time_ms(runs[k][2]))
    train = {}
    for k, (m, tr, _, ts) in runs.items():
        train[k] = {"step_ms": float(np.median(ts)), "rounds": ts}
        tr.close(); m.close()
    out["train_per_roi_step"] = {"minibatch": "2 images of 600 x 1000, 128 ROIs each", **train,
                                 "losses_finite": bool(torch.isfinite(losses).all())}
    ctx.close()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        f.write(json.dumps(out) + "\n")
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

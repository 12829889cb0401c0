"""Times detect + NMS over N images in one model call (mpn_model_detect_nms_batch_dev) against N per-image calls
(mpn_get_images_dev + mpn_model_detect_nms_dev per image, the same work) on one GPU, in one process, and writes one JSON
line per measurement.

  * detect + NMS, device-resident: VGG-16 Fast R-CNN (21 classes) and MultiPathNet (81 classes), raw 600 x 1000 images
    (getImages keeps 600 x 1000), R = 300, 500 and 1000 random ROIs per image, N = 1, 2, 4, 8. Each form runs on a model
    of its own, built and warmed up at every (R, N) first; then the two forms alternate --reps times, each timing --steps
    calls with CUDA events. Medians per image are reported.
  * fc6 / fc7 at M = R and M = 4R rows, as a model plans each layer (Context.linear_bench: CUDA events over --iters
    launches, split-K reduce included), per ROI.
  * validate (Tester_FRCNN:test + the device COCO evaluator) per image with images_per_batch 1 and 4, alternated, on
    --val-images synthetic COCO-like 480 x 640 images with 500 proposals each, MultiPathNet (81 classes, integral_k 6).
The GPU's name and power limit are read in the same process.
    python tools/detect_batch_time.py [--steps 5] [--warmup 2] [--reps 5] [--iters 30] [--out profiles/h100_detect_batch.json]"""
import argparse
import ctypes as C
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
from svd_time import gpu_info

H0, W0, SCALE, MAX_SIZE = 600, 1000, 600, 1000
RS, NS = (300, 500, 1000), (1, 2, 4, 8)
CONFIGS = {"vgg16_frcnn": ("vgg16_fast_rcnn", 21, {}), "multipathnet": ("vgg16_multipathnet", 81, {})}
LINEARS = [("fc6", 4096, 25088, True), ("fc7", 4096, 4096, True)]     # (name, N outputs, K inputs, w16 as VGG-16 plans it)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=30)
    ap.add_argument("--val-images", type=int, default=16)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_detect_batch.json"))
    args = ap.parse_args()
    if args.reps < 3:
        raise SystemExit("--reps must be at least 3")
    import torch
    import multipathnet_b200 as mpn
    from multipathnet_b200 import models, workloads as wl
    from multipathnet_b200._lib import CImageTransform
    ctx = mpn.Context(0)                 # the legacy default stream: the one torch's events below are recorded on
    lines = []

    def emit(line):
        line = {"tool": "detect_batch_time", **line, **gpu_info()}
        print(json.dumps(line), flush=True)
        lines.append(line)

    nmax, rmax = max(NS), max(RS)
    raws = [torch.from_numpy(wl.raw_image(H0, W0, 10 + i)).cuda() for i in range(nmax)]
    for name, (builder, ncls, kw) in CONFIGS.items():
        spec = getattr(models, builder)(ncls, seed=1234, **kw)
        tf = CImageTransform.of(spec.transformer)
        h, w = H0, W0
        scaled = [torch.empty((3, h, w), device="cuda") for _ in range(nmax)]
        boxes = torch.from_numpy(np.concatenate([wl.random_boxes(rmax, H0, W0, 20 + i) for i in range(nmax)], 0)).cuda()
        sc = torch.empty((nmax * rmax, ncls), device="cuda"); bb = torch.empty((nmax * rmax, 4 * ncls), device="cuda")
        kp = torch.empty((ncls - 1) * nmax * rmax, dtype=torch.int32, device="cuda")
        kc = torch.empty((nmax, ncls - 1), dtype=torch.int32, device="cuda")
        mb = mpn.Model(ctx, spec, max_rois=nmax * rmax, max_h=h, max_w=w)
        mp = mpn.Model(ctx, spec, max_rois=rmax, max_h=h, max_w=w)
        im_scale = float(SCALE) / min(H0, W0)
        for R in RS:
            for N in NS:
                def batched():
                    mb.detect_nms_batch_dev(raws[:N], [(H0, W0)] * N, spec.transformer, SCALE, MAX_SIZE, [R] * N, boxes[:N * R], -1.5, 0.3,
                                            sc, bb, kp, kc)

                def per_image():
                    for i in range(N):
                        ctx.check(ctx.lib.mpn_get_images_dev(ctx.h, raws[i].data_ptr(), H0, W0, C.addressof(tf), h, w, scaled[i].data_ptr()),
                                  "get_images_dev")
                        mp.detect_nms_dev(scaled[i], h, w, boxes[i * R:(i + 1) * R], R, im_scale, W0, H0, -1.5, 0.3, sc, bb, kp, kc)
                # the batched call's rows are image-major: image i's R proposals are rows [i R, (i + 1) R) of `boxes`
                forms = {"batched": batched, "per_image": per_image}
                for f in forms.values():
                    for _ in range(args.warmup):
                        f()
                torch.cuda.synchronize()
                runs = {k: [] for k in forms}
                for _ in range(args.reps):
                    for k, f in forms.items():
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        for _ in range(args.steps):
                            f()
                        b.record()
                        b.synchronize()
                        runs[k].append(a.elapsed_time(b) / args.steps / N)
                med = {k: float(np.median(v)) for k, v in runs.items()}
                emit({"what": "detect_nms_dev", "config": name, "classes": ncls, "H": h, "W": w, "R": R, "N": N, "steps": args.steps,
                      "reps": args.reps, "ms_per_image": runs, "median_ms_per_image": med,
                      "per_image_over_batched": med["per_image"] / med["batched"]})
        mb.close(); mp.close()
    # fc6 / fc7 per ROI at M = R and 4 R
    for R in RS:
        ms = {}
        for n, N, K, w16 in LINEARS:
            for M in (R, 4 * R):
                ctx.linear_bench(M, N, K, w16, False, iters=3)
                ms[(n, M)] = []
        for _ in range(args.reps):
            for n, N, K, w16 in LINEARS:
                for M in (R, 4 * R):
                    ms[(n, M)].append(ctx.linear_bench(M, N, K, w16, False, iters=args.iters)[0])
        layers = {}
        for n, N, K, _ in LINEARS:
            for M in (R, 4 * R):
                t = float(np.median(ms[(n, M)]))
                layers[f"{n}_M{M}"] = {"M": M, "N": N, "K": K, "median_ms": t, "us_per_roi": 1e3 * t / M,
                                       "tflops": 2.0 * M * K * N / (t * 1e-3) / 1e12}
        emit({"what": "fc_layers", "R": R, "iters": args.iters, "reps": args.reps, "layers": layers})
    # validate per image, images_per_batch 1 against 4
    spec = models.vgg16_multipathnet(81, seed=1234, integral_k=6)
    gt, _ = wl.coco_eval_set(args.val_images, 80, 6, 10, seed=3)
    ids = [im["id"] for im in gt["images"]]
    ims = [wl.raw_image(480, 640, 30 + i) for i in range(len(ids))]
    props = [wl.random_boxes(500, 480, 640, 40 + i) for i in range(len(ids))]
    m = mpn.Model(ctx, spec, max_rois=2000, max_h=600, max_w=800)
    val = {1: [], 4: []}
    stats = {}
    for b in val:
        stats[b] = mpn.validate(m, spec.transformer, ims[:4], props[:4], ids[:4], gt, images_per_batch=b)     # warm-up
    for _ in range(3):
        for b in val:
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            stats[b] = mpn.validate(m, spec.transformer, ims, props, ids, gt, images_per_batch=b)
            val[b].append(1e3 * (time.perf_counter() - t0) / len(ids))
    m.close()
    emit({"what": "validate", "model": "vgg16_multipathnet(81, integral_k=6)", "images": len(ids), "proposals": 500, "raw": [480, 640],
          "ms_per_image": {str(k): v for k, v in val.items()}, "median_ms_per_image": {str(k): float(np.median(v)) for k, v in val.items()},
          "same_stats": bool(np.array_equal(stats[1], stats[4]))})
    ctx.close()
    os.makedirs(os.path.dirname(args.out), exist_ok=True)
    with open(args.out, "w") as f:
        for line in lines:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

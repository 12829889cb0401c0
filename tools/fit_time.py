"""Times what train.lua's loop adds around the step (multipathnet_b200.fit), on the recipe's minibatch
(scripts/train_multipathnet_coco.sh: scale 800, max_size 1000, 4 images, 64 ROIs per image) and
vgg16_multipathnet(81, integral_k=6) trained with the integral loss, the batches sampled on the device from a synthetic
COCO-like dataset (80 categories, 1000 proposals per image):
  - fit's per-step overhead: fit over --epochs x --epoch-size steps (no snapshot inside) against a bare loop of
    `sample_integral(k)` + `step_batch`, the two alternating --rounds times, host clock around each run (both end with
    a synchronous step);
  - a checkpoint: save_checkpoint / load_checkpoint + Trainer.load_state_dict times, and the file size against the size
    counted from the shapes (a master and a momentum buffer per trained tensor, fp32);
  - validation: `validate` per image over --val-images test images with 500 proposals each (train.lua's
    test_best_proposals_number), after one warm-up image.
Writes profiles/h100_fit.json (or --out) with the GPU's name and power limit read in the same run.
    python tools/fit_time.py [--out FILE] [--rounds 3] [--epochs 2] [--epoch-size 10] [--val-images 8]"""
import argparse
import json
import os
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
import numpy as np
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from multipathnet_b200.batch_provider import integral_thresholds
from train_time import gpu_info

NCAT, K, SEED = 80, 6, 555


def dataset(n, seed, n_props):
    """n images of 480..640 x 640..800 pixels, 1..6 objects each, n_props proposals (a third jittered objects)"""
    rng = np.random.default_rng(seed)
    images, anns, boxes, sizes = [], [], [], []
    for i in range(n):
        H, W = int(rng.integers(480, 641)), int(rng.integers(640, 801))
        sizes.append((H, W))
        images.append({"id": i + 1, "file_name": f"{i}.jpg", "height": H, "width": W})
        objs = []
        for _ in range(int(rng.integers(1, 7))):
            w, h = float(rng.uniform(20, W / 2)), float(rng.uniform(20, H / 2))
            x, y = float(rng.uniform(0, W - w)), float(rng.uniform(0, H - h))
            objs.append((x, y, w, h))
            anns.append({"id": len(anns) + 1, "image_id": i + 1, "category_id": int(rng.integers(1, NCAT + 1)), "bbox": [x, y, w, h],
                         "area": w * h, "iscrowd": 0})
        b = np.empty((n_props, 4), np.float32)
        for p in range(n_props):
            if p % 3 == 0:
                x, y, w, h = objs[p % len(objs)]
                j = rng.normal(0, 0.15, 4) * [w, h, w, h]
                b[p] = (x + j[0], y + j[1], x + w + j[2], y + h + j[3])
            else:
                x1, y1 = rng.uniform(0, W - 16), rng.uniform(0, H - 16)
                b[p] = (x1, y1, rng.uniform(x1 + 8, W), rng.uniform(y1 + 8, H))
        boxes.append(np.clip(b, 0, [W - 1, H - 1, W - 1, H - 1]).astype(np.float32))
    gt = {"images": images, "annotations": anns, "categories": [{"id": c} for c in range(1, NCAT + 1)]}
    return gt, {"boxes": boxes, "images": [im["file_name"] for im in images]}, sizes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--epochs", type=int, default=2)
    ap.add_argument("--epoch-size", type=int, default=10)
    ap.add_argument("--val-images", type=int, default=8)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_fit.json"))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("no CUDA device: this tool measures the GPU only")
    info = gpu_info()
    ctx = mpn.Context(0)
    gt, props, sizes = dataset(40, 1, 1000)

    def image(i):
        H, W = sizes[i]
        return np.random.default_rng(100 + i).integers(0, 256, (H, W, 3), dtype=np.uint8)
    spec = models.vgg16_multipathnet(NCAT + 1, seed=1234, integral_k=K)
    db = mpn.RoiDB(ctx, gt, props, NCAT, integral_thresholds(K), best_number=1000)
    prov = mpn.BatchProviderROI(db, image, spec.transformer, imgs_per_batch=4, batch_size=64, scale=800, max_size=1000, seed=SEED)
    prov.setup_data()
    m = mpn.Model(ctx, spec, max_rois=1000, max_h=1000, max_w=1000)
    tr = mpn.Trainer(m, lr=1e-5, seed=SEED, integral=True)   # a small rate keeps the random model's detections finite
    n_steps = args.epochs * args.epoch_size

    def bare():
        for k in range(n_steps):
            tr.step_batch(prov.sample_integral(k))

    def loop():
        # the same sample indices as bare(): fit draws step k of epoch e at (e - 1) * epochSize + k
        mpn.fit(tr, prov, dict(nEpochs=args.epochs, epochSize=args.epoch_size, step=10 ** 6, snapshot=10 ** 6, integral=True),
                log=lambda s: None)
    for k in range(3):                                            # warm-up: plans, the image sizes of the first batches
        tr.step_batch(prov.sample_integral(k))
    rounds = []
    for _ in range(args.rounds):
        row = {}
        for name, fn in (("bare", bare), ("fit", loop)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            row[name] = (time.perf_counter() - t0) * 1e3 / n_steps
        rounds.append({k: round(v, 3) for k, v in row.items()})
    bare_ms = float(np.median([r["bare"] for r in rounds]))
    fit_ms = float(np.median([r["fit"] for r in rounds]))

    # a checkpoint of this training
    counted = sum(2 * 4 * int(np.prod(spec.weights[i].shape)) for i in tr.trained)
    with tempfile.TemporaryDirectory() as tmp:
        path = os.path.join(tmp, "checkpoint.npz")
        t0 = time.perf_counter()
        mpn.save_checkpoint(path, tr, epoch=args.epochs, step=10 ** 6, decay=0.1, bbox_mean=prov.bbox_regr[0], bbox_std=prov.bbox_regr[1])
        save_s = time.perf_counter() - t0
        size = os.path.getsize(path)
        t0 = time.perf_counter()
        d = mpn.load_checkpoint(path)
        read_s = time.perf_counter() - t0
        t0 = time.perf_counter()
        tr.load_state_dict(d)
        apply_s = time.perf_counter() - t0

    # validation on the training model's handle
    test = list(range(20, 20 + 1 + args.val_images))
    ims = [np.ascontiguousarray(image(i).transpose(2, 0, 1), np.float32) / np.float32(255) for i in test]
    tp = [props["boxes"][i][:500] for i in test]
    ids = [i + 1 for i in test]
    sub = dict(gt, images=[gt["images"][i] for i in test], annotations=[a for a in gt["annotations"] if a["image_id"] in set(ids)])
    mpn.validate(m, spec.transformer, ims[:1], tp[:1], ids[:1], sub, scale=800, max_size=1000)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    stats = mpn.validate(m, spec.transformer, ims[1:], tp[1:], ids[1:], sub, scale=800, max_size=1000)
    val_ms = (time.perf_counter() - t0) * 1e3 / args.val_images
    tr.step_batch(prov.sample_integral(0))                       # training goes on after validating

    res = {"tool": "fit_time", **info,
           "shape": f"vgg16_multipathnet(81, integral_k={K}); 4 images per step at scale 800 / max_size 1000, 64 ROIs each",
           "steps_per_run": n_steps, "rounds": args.rounds, "per_round_ms_per_step": rounds,
           "bare_ms_per_step": round(bare_ms, 3), "fit_ms_per_step": round(fit_ms, 3),
           "fit_overhead_ms_per_step": round(fit_ms - bare_ms, 3),
           "checkpoint": {"save_s": round(save_s, 3), "read_s": round(read_s, 3), "load_state_dict_s": round(apply_s, 3),
                          "file_bytes": size, "counted_bytes": counted, "trained_tensors": len(tr.trained)},
           "validate_ms_per_image": round(val_ms, 1), "validate_images": args.val_images, "validate_proposals_per_image": 500,
           "validate_stats_finite": bool(np.isfinite(stats).all()),
           "note": "host clock around runs that end in a synchronous step; counted_bytes is 2 x 4 bytes per trained element "
                   "(master + momentum buffer), the file adds the JSON metadata and the npz headers"}
    d = os.path.dirname(args.out)
    if d:
        os.makedirs(d, exist_ok=True)
    with open(args.out, "w") as f:
        f.write(json.dumps(res) + "\n")
    print(json.dumps(res))
    tr.close(); m.close(); db.close(); ctx.close()


if __name__ == "__main__":
    main()

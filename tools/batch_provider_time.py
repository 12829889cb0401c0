"""Time the training feed on one GPU and write profiles/h100_batch_provider.json (or --out):

- RoiDB construction at COCO trainval35k scale (synthetic, seeded: --images images, --props proposals and about --gt
  GT boxes per image), with one threshold set and with the six integral sets (fg = bg_hi = 0.5 + (i - 1) / 20): wall time,
  the matching pass's kernel time (CUDA events), the rest (host tables + upload), algorithmic bytes / kernel time, and
  the device memory the RoiDB holds (cudaMemGetInfo before / after);
- one step of 2 images scaled to 600 x 1000: plan + image upload + flipped getImages + sampler (BatchProviderROI.sample),
  beside the vgg16_fast_rcnn training step it feeds (Trainer.step_batch);
- the numpy restatement (tests/_batch_provider_ref.py) on a smaller set, for scale.

The card's name and power limit are read in the same run and stored beside the numbers."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

import multipathnet_b200 as mpn  # noqa: E402
from multipathnet_b200 import models  # noqa: E402


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return q.stdout.strip().splitlines()[0] if q.returncode == 0 and q.stdout.strip() else "not read"


def synthetic(n, props, gt_per_image, seed, H=480, W=640):
    rng = np.random.default_rng(seed)
    ng = rng.poisson(gt_per_image, n)
    ng[ng == 0] = 1
    anns = []
    aid = 1
    gx = rng.uniform(0, W - 60, ng.sum()); gy = rng.uniform(0, H - 60, ng.sum())
    gw = rng.uniform(8, 200, ng.sum()); gh = rng.uniform(8, 200, ng.sum())
    gc = rng.integers(1, 81, ng.sum())
    k = 0
    for i in range(n):
        for _ in range(ng[i]):
            anns.append({"id": aid, "image_id": i + 1, "category_id": int(gc[k]), "bbox": [float(gx[k]), float(gy[k]), float(gw[k]), float(gh[k])],
                         "area": float(gw[k] * gh[k]), "iscrowd": int(aid % 50 == 0)})
            aid += 1; k += 1
    gt = {"images": [{"id": i + 1, "file_name": f"{i + 1:012d}.jpg", "height": H, "width": W} for i in range(n)],
          "annotations": anns, "categories": [{"id": c, "name": str(c)} for c in range(1, 81)]}
    x1 = rng.uniform(0, W - 20, (n, props)).astype(np.float32); y1 = rng.uniform(0, H - 20, (n, props)).astype(np.float32)
    b = np.stack([x1, y1, x1 + rng.uniform(4, 300, (n, props)).astype(np.float32), y1 + rng.uniform(4, 300, (n, props)).astype(np.float32)], 2)
    s = rng.random((n, props), dtype=np.float32)
    return gt, {"boxes": list(b), "scores": list(s), "images": [im["file_name"] for im in gt["images"]]}


def build(ctx, gt, props, thr):
    import torch
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    ctx.profile_begin()
    t0 = time.perf_counter()
    db = mpn.RoiDB(ctx, gt, props, 80, thr)
    ctx.synchronize()
    wall = time.perf_counter() - t0
    prof = ctx.profile_end()
    kern = sum(ms for ms, _ in prof.values())
    free1 = torch.cuda.mem_get_info()[0]
    rows, lists = db.n_rows, int(db.counts.sum())
    nbytes = rows * (16 + 12) + 2 * len(thr) * rows * 4 + 4 * lists + 4 * 3 * db.counts.size
    return db, {"sets": len(thr), "images": db.n_images, "rows": rows, "list_entries": lists, "create_wall_ms": wall * 1e3,
                "kernel_ms": kern, "host_tables_and_upload_ms": wall * 1e3 - kern, "kernel_bytes": nbytes,
                "kernel_GB_per_s": nbytes / (kern * 1e-3) / 1e9 if kern > 0 else None, "device_bytes_held": int(free0 - free1)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--images", type=int, default=118287)
    ap.add_argument("--props", type=int, default=1000)
    ap.add_argument("--gt", type=float, default=7.3)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--ref-images", type=int, default=200)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_batch_provider.json"))
    a = ap.parse_args()
    out = {"card": card(), "args": vars(a)}
    ctx = mpn.Context(0)
    t0 = time.perf_counter()
    gt, props = synthetic(a.images, a.props, a.gt, 0)
    out["synthetic_data_s"] = time.perf_counter() - t0
    db1, out["match_one_set"] = build(ctx, gt, props, [(0.5, 0.1, 0.5)])
    db1.close()
    db6, out["match_six_integral_sets"] = build(ctx, gt, props, [(0.5 + i / 20, 0.1, 0.5 + i / 20) for i in range(6)])
    db6.close()
    del props

    # one step: 2 images 480 x 800 -> 600 x 1000, and the VGG16 Fast R-CNN step it feeds
    small_gt, small_props = synthetic(2000, 1000, a.gt, 1, H=480, W=800)
    db = mpn.RoiDB(ctx, small_gt, small_props, 80)
    raw = [np.random.default_rng(i).integers(0, 256, (480, 800, 3), dtype=np.uint8) for i in range(4)]
    prov = mpn.BatchProviderROI(db, lambda i: raw[i % 4], "ross")
    prov.setup_data()
    spec = models.vgg16_fast_rcnn(81, seed=0)
    m = mpn.Model(ctx, spec, max_rois=256, max_h=1000, max_w=1000)
    tr = mpn.Trainer(m)
    for s in range(3):
        tr.step_batch(prov.sample(s))
    ctx.synchronize()
    ts, tt = [], []
    for s in range(3, 3 + a.steps):
        t0 = time.perf_counter()
        b = prov.sample(s)
        ctx.synchronize()
        t1 = time.perf_counter()
        tr.step_batch(b)
        t2 = time.perf_counter()
        ts.append((t1 - t0) * 1e3); tt.append((t2 - t1) * 1e3)
    out["step"] = {"images": "2 x 480 x 800 uint8 -> 600 x 1000", "rows": int(b.R), "sample_ms_median": float(np.median(ts)),
                   "sample_ms_min": float(np.min(ts)), "train_step_ms_median": float(np.median(tt)), "train_step_ms_min": float(np.min(tt))}
    tr.close(); m.close(); db.close()

    import _batch_provider_ref as ref
    rg, rp = synthetic(a.ref_images, a.props, a.gt, 2)
    t0 = time.perf_counter()
    ref.restate_roidb(rg, rp, 80, [(0.5, 0.1, 0.5)])
    out["numpy_restatement_for_scale"] = {"images": a.ref_images, "props": a.props, "seconds": time.perf_counter() - t0,
                                          "note": "the test restatement on the host, one set; not a product path"}
    ctx.close()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    with open(a.out, "w") as f:
        json.dump(out, f, indent=1)
    print(json.dumps(out, indent=1))


if __name__ == "__main__":
    main()

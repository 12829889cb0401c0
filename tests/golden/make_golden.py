"""Generates tests/golden/*.npz. Needs the reference's source (oracle/Makefile REF=<reference checkout>, for the literal
nms.c build): `python tests/golden/make_golden.py`. The NMS goldens are outputs of the REFERENCE's own
nms.c; the others are outputs of the C restatement (parity unpinned, see DESIGN.md), committed so that
any later change to the oracle is caught.

Two more fixtures come from the reference and let the suite run without it:
  * nms_literal_golden.npz — the literal nms.c's output for every fixed input the suite feeds oracle.ref's ref_* functions
    (keyed by a hash of the inputs). Regenerate by running the tests that call them with the literal build present and
    MPN_LITERAL_RECORD=tests/golden/nms_literal_golden.npz (the GPU NMS tests' inputs do not depend on the GPU).
  * image_detect_methods.json — the method table (name -> arguments) of the reference's ImageDetect.lua."""
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import ref as O  # noqa: E402
from multipathnet_b200 import workloads as wl  # noqa: E402

O.build()
here = os.path.dirname(os.path.abspath(__file__))
d = {}
cases = [("n1", 1, 0.3, False), ("n64", 64, 0.3, False), ("n65", 65, 0.3, False), ("n300", 300, 0.3, False),
         ("n1000", 1000, 0.3, False), ("n1000_t5", 1000, 0.5, False), ("ties200", 200, 0.3, True), ("ties777", 777, 0.3, True)]
for i, (name, n, thr, ties) in enumerate(cases):
    sb = wl.nms_sweep_boxes(n, 1, 500 + i, ties=ties)[0]
    d[name + "_sb"] = sb
    d[name + "_rows"] = O.ref_nms_rows(sb, thr)          # literal reference nms.c
    d[name + "_thr"] = np.float32(thr)
np.savez_compressed(os.path.join(here, "nms_golden.npz"), **d)

rng = np.random.default_rng(42)
rois = np.concatenate([np.ones((48, 1), np.float32), wl.random_boxes(48, 600, 800, 42)], 1)
fmap = rng.standard_normal((1, 16, 38, 50)).astype(np.float32)
rois_neg = (rng.standard_normal((40, 5)) * 50).astype(np.float32)
rois_neg[:, 0] = 1
deltas = (rng.standard_normal((48, 12)) * 0.3).astype(np.float32)
boxes = rois[:, 1:].copy()
dense_sb = wl.nms_sweep_boxes(300, 1, 77)[0]
np.savez_compressed(os.path.join(here, "ops_golden.npz"), rois=rois, foveal=O.foveal(rois), fmap=fmap, rois_neg=rois_neg,
                    roi_v2=O.roi_pool(fmap, rois_neg, 7, 7, 1 / 16, 2), roi_v1=O.roi_pool(fmap, rois_neg, 7, 7, 1 / 16, 1),
                    deltas=deltas, boxes=boxes, decoded=O.convert_from(deltas, boxes), dense_sb=dense_sb,
                    dense_pick=O.nms_dense(dense_sb, 0.3))

# getImages (SURVEY 8f-1): raw image -> transformer -> image.scale, outputs of the two-pass C restatement (parity unpinned)
g = {}
for name, (H0, W0, scale, max_size, kind) in {"grow": (20, 30, 33, 1000, "ross"), "shrink": (40, 56, 17, 1000, "imagenet"),
                                               "capped": (16, 60, 32, 90, "ross"), "same": (24, 32, 24, 1000, "imagenet")}.items():
    im = wl.raw_image(H0, W0, 900 + H0)
    out, s = O.get_images(im, kind, scale, max_size)
    g[name + "_im"], g[name + "_out"], g[name + "_cfg"] = im, out, np.array([scale, max_size, s, kind == "imagenet"], np.float64)
np.savez_compressed(os.path.join(here, "getimages_golden.npz"), **g)
print("golden fixtures written")

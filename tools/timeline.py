"""In-kernel timeline of the tensor-core launches of the default workload (GPU): where the time between layers goes.
Per launch (us, relative to the first stamp): kernel entry (first CTA), dependency wait passed, first MMA, last MMA issued,
last epilogue finished, exit; `gap` = this launch's first MMA minus the previous launch's last epilogue."""
import ctypes as C, os, sys
import numpy as np, torch
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
ctx = mpn.Context(0)
Cn, H, W, R = 21, 600, 800, 1000
spec = models.vgg16_fast_rcnn(Cn, seed=1234)
m = mpn.Model(ctx, spec, max_rois=R, max_h=H, max_w=W)
dev = torch.device("cuda:0")
img = torch.from_numpy(wl.transform(wl.raw_image(H, W, 7), "ross")).to(dev)
boxes = torch.from_numpy(wl.random_boxes(R, H, W, 100)).to(dev)
sc = torch.empty((R, Cn), device=dev); bb = torch.empty((R, 4 * Cn), device=dev)
kp = torch.empty((Cn - 1, R), dtype=torch.int32, device=dev); ct = torch.empty((Cn - 1,), dtype=torch.int32, device=dev)
step = lambda: m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, sc, bb, kp, ct)
for _ in range(5): step()
ctx.synchronize()
ctx.check(ctx.lib.mpn_ctx_timeline_begin(ctx.h, 128), "timeline_begin")
for _ in range(3): step()
mn = (C.c_uint64 * 512)(); mx = (C.c_uint64 * 512)(); n = C.c_int32(0)
ctx.check(ctx.lib.mpn_ctx_timeline_end(ctx.h, mn, mx, C.byref(n)), "timeline_end")
n = n.value
per = n // 3
names = ["conv1_2", "conv2_1", "conv2_2", "conv3_1", "conv3_2", "conv3_3", "conv4_1", "conv4_2", "conv4_3", "conv5_1", "conv5_2", "conv5_3",
         "fc6", "fc7", "cls", "bbox"]
t0 = mn[4 * per]          # second step
prev_epi = None
print(f"{n} launches, {per} per step; second step:")
tot_gap = 0.0
for i in range(per, 2 * per):
    e, w_, f = mn[4 * i], mn[4 * i + 1], mn[4 * i + 2]
    lm, le, ex = mx[4 * i], mx[4 * i + 1], mx[4 * i + 2]
    us = lambda t: (t - t0) / 1e3
    gap = (f - prev_epi) / 1e3 if prev_epi else float('nan')
    if prev_epi: tot_gap += gap
    nm = names[i - per] if i - per < len(names) else "?"
    print(f"{nm:8s} entry {us(e):8.1f}  wait_ok {us(w_):8.1f}  first_mma {us(f):8.1f}  last_mma {us(lm):8.1f}  last_epi {us(le):8.1f}  exit {us(ex):8.1f} | "
          f"mma_span {(lm - f) / 1e3:6.1f}  epi_tail {(le - lm) / 1e3:5.1f}  gap_from_prev_epi {gap:6.1f}")
    prev_epi = le
print("sum of gaps between tensor-core launches (includes the non-TC kernels in between):", round(tot_gap, 1), "us")
print("step span (first entry -> next step's first entry):", (mn[4 * 2 * per] - mn[4 * per]) / 1e3, "us")

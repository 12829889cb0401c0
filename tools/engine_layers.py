"""Per-layer view of the wgmma engine on the default workload (vgg16_frcnn: VGG-16 Fast R-CNN, 600 x 800, 1000 ROIs).

Two measurements in one process, and the GPU's name, power limit and SM clock read right after them:
  - conv_bench: ms per launch of each trunk convolution (conv1_2 .. conv5_3) at its workload shape, CUDA events over
    --iters launches; with the plan (N tile, split-K, tiles) that gives the SM cycles per K block, i.e. the launch's
    time x SMs / (units x K blocks) at the SM clock read, against the tensor pipe's MMA time of one K block
    (3 products x 128 x BN x 64 MACs at 2048 bf16 MACs per clock: 3072 / 1536 / 768 clocks for BN = 256 / 128 / 64);
  - the in-kernel timeline (mpn_ctx_timeline_begin / end) of every engine launch of one detect + NMS step:
    mma_span = first MMA start .. last MMA end, epi_tail = last MMA end .. last epilogue store, epi_sum = the epilogue
    time of every tile summed over CTAs (0 for builds that do not record it).
One JSON line per run is appended to --out; --root runs the library of another checkout (e.g. the parent commit's).
    python tools/engine_layers.py [--label branch] [--root .] [--iters 50] [--out profiles/h100_engine_ring.json]"""
import argparse
import ctypes as C
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, HERE)
from bf16_time import gpu_info       # noqa: E402  (the read-only nvidia-smi query of the timing tools)

H, W, R, NCLS = 600, 800, 1000, 21
# (name, Cin, H, W, Cout) of the 3x3 / pad 1 trunk convolutions that run on the engine (conv1_1 has its own kernel)
TRUNK = [("conv1_2", 64, 600, 800, 64), ("conv2_1", 64, 300, 400, 128), ("conv2_2", 128, 300, 400, 128),
         ("conv3_1", 128, 150, 200, 256), ("conv3_2", 256, 150, 200, 256), ("conv3_3", 256, 150, 200, 256),
         ("conv4_1", 256, 75, 100, 512), ("conv4_2", 512, 75, 100, 512), ("conv4_3", 512, 75, 100, 512),
         ("conv5_1", 512, 38, 50, 512), ("conv5_2", 512, 38, 50, 512), ("conv5_3", 512, 38, 50, 512)]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--label", default="branch")
    ap.add_argument("--root", default=ROOT, help="checkout whose multipathnet_b200 (and built library) is measured")
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--out", default=os.path.join(ROOT, "profiles", "h100_engine_ring.json"))
    args = ap.parse_args()
    sys.path.insert(0, os.path.abspath(args.root))
    import torch
    import multipathnet_b200 as mpn
    from multipathnet_b200 import models, workloads as wl

    ctx = mpn.Context(0)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    layers = []
    for name, cin, h, w, cout in TRUNK:
        plan = (C.c_int32 * 8)()
        assert ctx.lib.mpn_debug_plan(1, cin, h, w, cout, 3, 1, 1, 0, sms, plan) == 0
        mode, bn, splitk, th, tw = plan[0], plan[2], plan[3], plan[6], plan[7]
        tiles_m = -(-w // tw) * -(-h // th)
        units = tiles_m * -(-cout // bn) * splitk
        kblocks = 9 * cin // 64 // splitk
        ms = ctx.conv_bench(1, cin, h, w, cout, 3, 1, 1, iters=args.iters)[0]
        layers.append({"layer": name, "bn": bn, "mode": mode, "splitk": splitk, "units": units, "kblocks_per_unit": kblocks,
                       "ms_per_launch": ms, "mma_bound_clk_per_kblock": 3 * 128 * bn * 64 // 2048})
    info = gpu_info()
    for l in layers:
        l["clk_per_kblock"] = l["ms_per_launch"] * 1e-3 * info["sm_mhz"] * 1e6 * sms / (l["units"] * l["kblocks_per_unit"]) if info["sm_mhz"] else None

    spec = models.vgg16_fast_rcnn(NCLS, seed=1234)
    m = mpn.Model(ctx, spec, max_rois=R + 48, max_h=H + 8, max_w=W)
    img = torch.from_numpy(wl.transform(wl.raw_image(H, W, 2), spec.transformer)).cuda()
    boxes = torch.from_numpy(wl.random_boxes(R, H, W, 2)).cuda()
    outs = (torch.empty((R, NCLS), dtype=torch.float32, device="cuda"), torch.empty((R, 4 * NCLS), dtype=torch.float32, device="cuda"),
            torch.empty((NCLS - 1, R), dtype=torch.int32, device="cuda"), torch.empty((NCLS - 1,), dtype=torch.int32, device="cuda"))
    for _ in range(5):
        m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, *outs)
    torch.cuda.synchronize()
    cap = 64
    ctx.check(ctx.lib.mpn_ctx_timeline_begin(ctx.h, cap), "timeline_begin")
    m.detect_nms_dev(img, H, W, boxes, R, 1.0, W, H, -1.5, 0.3, *outs)
    tmin, tmax, n = (C.c_uint64 * (4 * cap))(), (C.c_uint64 * (4 * cap))(), C.c_int32()
    ctx.check(ctx.lib.mpn_ctx_timeline_end(ctx.h, tmin, tmax, C.byref(n)), "timeline_end")
    names = [t[0] for t in TRUNK]
    timeline = []
    for i in range(n.value):
        lo, hi = tmin[4 * i:4 * i + 4], tmax[4 * i:4 * i + 4]
        timeline.append({"launch": i, "layer": names[i] if i < len(names) else f"head{i - len(names)}",
                         "span_us": (hi[1] - lo[0]) / 1e3, "mma_span_us": (hi[0] - lo[2]) / 1e3, "epi_tail_us": (hi[1] - hi[0]) / 1e3,
                         "epi_sum_us": hi[3] / 1e3})
    m.close(); ctx.close()
    line = {"tool": "engine_layers", "label": args.label, "workload": "vgg16_frcnn", "sms": sms, **info,
            "trunk_conv_bench": layers, "timeline_one_step": timeline}
    print(json.dumps(line), flush=True)
    with open(args.out, "a") as f:
        f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()

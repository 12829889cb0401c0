"""References of MultiPathNet's phase 2 (Trainer(phase2=True), set_phase2):

- the towers' ROI pooling backward as the device runs it (csrc/roi.cu): the foveal region of a ROI, the per-job argmax,
  the normalisation's (a, b) in double and the in-order fp32 gather, for the kernel-level tests;
- an fp64 oracle of one phase-2 step: torch autograd from each image's stored input of layer phase2_from through the
  trained convolutions and max pools, every tower's foveal, normalised ROI pooling of conv5 / conv4 / conv3, conv_mix,
  fc6, fc7 and the heads. As in _train_trunk_ref, the oracle takes from the device what decides a branch: every ReLU
  side, every max-pool and ROI argmax (the rules below, on the device's stored maps), the dropout masks and the per-ROI
  ReLU gates."""
import numpy as np

from _train_trunk_ref import _roundf, pool_argmax

FLT_MAX = np.float32(np.finfo(np.float32).max)
_OFF = {1: 0.25, 2: 0.5, 3: 1.5}
_MUL = {1: 1.5, 2: 2.0, 3: 4.0}


def region_box(box, region):
    """nn.Foveal's region of a ROI (x1, y1, x2, y2) in double, rounded once to fp32 (csrc/roi.cu roi_geometry)"""
    x1, y1, x2, y2 = (np.float32(v) for v in box)
    if region == 0:
        return x1, y1, x2, y2
    off, mul = _OFF[region], _MUL[region]
    w, h = float(x2) - float(x1), float(y2) - float(y1)
    rx, ry = float(x1) - w * off, float(y1) - h * off
    rw, rh = w * mul, h * mul
    return np.float32(rx), np.float32(ry), np.float32(rx + rw), np.float32(ry + rh)


def bin_windows(box, region, scale, variant, PW, PH, H, W):
    """roi_geometry / bin_window in fp32 for the job's region: [(hs, he, ws, we)] per bin, ph major"""
    f = np.float32
    x1, y1, x2, y2 = region_box(box, region)
    sc = f(scale)
    sw, sh = _roundf(f(x1 - f(1)) * sc), _roundf(f(y1 - f(1)) * sc)
    ew, eh = _roundf(f(x2 - f(1)) * sc), _roundf(f(y2 - f(1)) * sc)
    if variant == 2:
        ew, eh = ew - 1, eh - 1
    rw, rh = max(ew - sw + 1, 1), max(eh - sh + 1, 1)
    bw, bh = f(f(rw) / f(PW)), f(f(rh) / f(PH))
    out = []
    for ph in range(PH):
        for pw in range(PW):
            hs = int(np.floor(f(ph) * bh)) + sh
            he = int(np.ceil(f(ph + 1) * bh)) + sh
            ws = int(np.floor(f(pw) * bw)) + sw
            we = int(np.ceil(f(pw + 1) * bw)) + sw
            out.append((min(max(hs, 0), H), min(max(he, 0), H), min(max(ws, 0), W), min(max(we, 0), W)))
    return out


def roi_argmax(fmap, boxes, region, scale, variant, PW, PH):
    """per ROI, bin and channel the flat index h * W + w of the first cell in (h, w) scan order holding the window's
    maximum (the device's '> running max from -FLT_MAX' rule for finite maps); -1 for an empty bin -> R x PH*PW x C"""
    fmap = np.asarray(fmap, np.float32)
    C, H, W = fmap.shape
    out = np.full((len(boxes), PH * PW, C), -1, np.int64)
    for r, box in enumerate(boxes):
        for b, (hs, he, ws, we) in enumerate(bin_windows(box, region, scale, variant, PW, PH, H, W)):
            if he <= hs or we <= ws:
                continue
            k = np.argmax(fmap[:, hs:he, ws:we].reshape(C, -1), axis=1)
            out[r, b] = (hs + k // (we - ws)) * W + ws + k % (we - ws)
    return out


def norm_ab(x, g):
    """(a, b) of one ROI's normalised level: x, g its pooled values and their gradient (any shape), in double:
    n = sqrt(sum x^2 + 1e-10f), a = 1000 / n, b = 1000 (x . g) / n^3"""
    x, g = np.asarray(x, np.float64).ravel(), np.asarray(g, np.float64).ravel()
    n = np.sqrt(np.sum(x * x) + float(np.float32(1e-10)))
    return 1000.0 / n, 1000.0 * float(np.dot(x, g)) / (n * n * n)


def gather(fmap_hwc, jobs):
    """the device's gather for the jobs that pool one map (fmap_hwc H x W x C fp32, the cells' values). jobs: in order,
    dicts with argmax (R x bins x C, flat cell or -1), g (R x bins x C fp32: the job's slice of the pooled gradient) and
    ab (R x 2 doubles, or None). Per cell and channel the sum from +0 in job, r, bin order of g or fl(fl(a g) - fl(b x))
    in fp32 (np.add.at adds in index order) -> H x W x C"""
    H, W, C = fmap_hwc.shape
    x = np.asarray(fmap_hwc, np.float32).reshape(H * W, C)
    out = np.zeros((H * W, C), np.float32)
    for jb in jobs:
        am, g = np.asarray(jb["argmax"]), np.asarray(jb["g"], np.float32)
        sel = am >= 0
        cc = np.broadcast_to(np.arange(C), am.shape)
        v = g
        if jb.get("ab") is not None:
            ab = np.asarray(jb["ab"], np.float64)
            a = ab[:, 0].astype(np.float32)[:, None, None]
            b = ab[:, 1].astype(np.float32)[:, None, None]
            xv = x[np.maximum(am, 0), cc]
            v = (a * g).astype(np.float32) - (b * xv).astype(np.float32)
        np.add.at(out, (am[sel], cc[sel]), v[sel].astype(np.float32))
    return out.reshape(H, W, C)


def phase2_step_oracle(spec, k0, stored, rois_per_image, labels, targets, weights, gates, p, head=0, bbox_w=1.0, dev="cpu"):
    """fp64 losses and gradients {weight index: array} of one phase-2 step (trunk training from layer k0) of a
    multi-tower graph. stored[i]: {slot: C x H x W} of image i (the device's kept slots); gates: (tower, layer) ->
    R x cout, the device's backward gate through each per-ROI ReLU (inside its dropout mask); head: the trained class
    head of an integral model."""
    import torch
    dt = torch.float64
    params = {}

    def P(i):
        if i not in params:
            params[i] = torch.tensor(np.asarray(weights[i], np.float64), dtype=dt, device=dev, requires_grad=True)
        return params[i]

    layers = spec.trunk_layers
    maps = []                                                            # per image: slot -> 1 x C x H x W
    for i in range(len(rois_per_image)):
        s = {layers[k0].in_slot: torch.tensor(stored[i][layers[k0].in_slot], dtype=dt, device=dev)[None]}
        for L in layers[k0:]:
            x = s[L.in_slot]
            if L.kind == 1:
                z = torch.nn.functional.conv2d(x, P(L.weight), P(L.bias), padding=1)
                s[L.out_slot] = z * torch.tensor(stored[i][L.out_slot] > 0, dtype=dt, device=dev)[None]
            else:
                idx = torch.tensor(pool_argmax(stored[i][L.in_slot]), device=dev)
                Cc = x.shape[1]
                s[L.out_slot] = x.reshape(1, Cc, -1).gather(2, idx.reshape(1, Cc, -1)).reshape(1, Cc, idx.shape[1], idx.shape[2])
        maps.append(s)
    outs = []
    for t, T in enumerate(spec.towers):
        PW, PH = T.pooled_w, T.pooled_h
        levels = []
        for slot, scale in T.levels:
            per = []
            for i, boxes in enumerate(rois_per_image):
                fm = stored[i][slot]
                Cc, H, W = fm.shape
                am = roi_argmax(fm, boxes, T.region, scale, spec.roi_variant, PW, PH)
                flat = maps[i][slot].reshape(Cc, H * W)
                ok = torch.tensor(am >= 0, device=dev)
                g = flat[torch.arange(Cc, device=dev)[None, None, :].expand(am.shape), torch.tensor(np.maximum(am, 0), device=dev)]
                per.append(g * ok)                                       # R_i x bins x C
            v = torch.cat(per, 0)
            if T.normalize:
                R = v.shape[0]
                n = torch.sqrt((v.reshape(R, -1) ** 2).sum(1) + float(np.float32(1e-10)))
                v = v / n[:, None, None] * 1000.0
            levels.append(v)
        x = torch.cat(levels, 2)                                         # R x bins x Ctot, (h, w, c)
        R = x.shape[0]
        slots = {0: x.reshape(R, PH, PW, -1).permute(0, 3, 1, 2)}        # R x Ctot x PH x PW
        for li, L in enumerate(T.layers):
            x = slots[L.in_slot]
            if L.kind == 4:
                y = x.reshape(R, -1)
            elif x.dim() == 4:                                           # conv_mix, 1x1 on the pooled map
                y = torch.nn.functional.conv2d(x, P(L.weight), P(L.bias))
                if L.relu:
                    raise NotImplementedError("a ReLU on a per-ROI map")
            else:
                y = x @ P(L.weight).reshape(L.cout, -1).T + P(L.bias)
                if L.relu:
                    y = y * torch.tensor(gates[(t, li)], dtype=dt, device=dev) / (1.0 - p)
            slots[L.out_slot] = y
        outs.append(slots[T.out_slot])
    cat = torch.cat(outs, 1)
    R = cat.shape[0]
    hc, hb = spec.cls_heads[head], spec.bbox_head
    logits = cat[:, hc.col_begin:hc.col_begin + hc.col_len] @ P(hc.weight).T + P(hc.bias)
    deltas = cat[:, hb.col_begin:hb.col_begin + hb.col_len] @ P(hb.weight).T + P(hb.bias)
    lab = torch.tensor(np.asarray(labels, np.int64) - 1, device=dev)
    ce = torch.nn.functional.cross_entropy(logits, lab)
    sel = torch.zeros_like(deltas)
    rows = torch.nonzero(lab > 0)[:, 0]
    for k in range(4):
        sel[rows, 4 * lab[rows] + k] = 1.0
    masked = deltas * sel + (deltas - deltas.detach()) * (1.0 - sel)
    diff = masked - torch.tensor(targets, dtype=dt, device=dev)
    ad = diff.abs()
    sl1 = torch.where(ad < 1, 0.5 * diff * diff, ad - 0.5).sum() / R
    loss = ce + bbox_w * sl1
    loss.backward()
    grads = {i: t.grad.detach().cpu().numpy() for i, t in params.items()}
    return (loss.item(), ce.item(), sl1.item()), grads

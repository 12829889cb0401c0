"""fp64 oracle of the trunk-training step (Trainer(train_trunk=True)): torch autograd from each image's stored input of
the first trained trunk layer through the trained convolutions, max pools, ROI pooling, the tower and the heads. The
oracle takes from the device what decides a branch: every ReLU side (the stored output > 0), every max-pool and ROI
argmax (the rules below, applied to the device's stored planes), the dropout masks and the per-ROI ReLU gates. A
reordered fp32 sum can flip a near-tie; taking the device's side keeps the oracle's derivative the device's."""
import numpy as np

FLT_MAX = np.float32(np.finfo(np.float32).max)


def pool_argmax(y):
    """2x2 / stride 2 ceil-mode max pool of y (C x H x W fp32): flat index h * W + w of each window's first maximum in
    row-major order (> against the running max from -FLT_MAX), windows clipped at odd sizes -> C x ceil(H/2) x ceil(W/2)"""
    y = np.asarray(y, np.float32)
    C, H, W = y.shape
    Ho, Wo = (H + 1) // 2, (W + 1) // 2
    best = np.full((C, Ho, Wo), -FLT_MAX, np.float32)
    idx = np.full((C, Ho, Wo), -1, np.int64)
    oh, ow = np.meshgrid(np.arange(Ho), np.arange(Wo), indexing="ij")
    for dy in (0, 1):
        for dx in (0, 1):
            hh, ww = 2 * oh + dy, 2 * ow + dx
            ok = (hh < H) & (ww < W)
            v = np.where(ok[None], y[:, np.minimum(hh, H - 1), np.minimum(ww, W - 1)], -np.inf)
            upd = v > best
            best = np.where(upd, v, best)
            idx = np.where(upd, (hh * W + ww)[None], idx)
    return idx


def _roundf(x):
    x = float(x)
    return int(np.floor(abs(x) + 0.5)) * (1 if x >= 0 else -1)       # roundf: half away from zero


def roi_bin_windows(box, scale, variant, PW, PH, H, W):
    """csrc/roi.cu roi_geometry / bin_window (region 0) in fp32: [(hs, he, ws, we)] for the bins of one ROI, ph major"""
    f = np.float32
    x1, y1, x2, y2 = (f(v) for v in box)
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


def roi_argmax(fmap, boxes, scale, variant, PW, PH):
    """roi_pool_nchw_kernel's rule on fmap (C x H x W fp32): per ROI, bin and channel the flat index of the first cell
    in (h, w) scan order whose value is > the running max (from -FLT_MAX); -1 for an empty bin -> R x PH*PW x C"""
    fmap = np.asarray(fmap, np.float32)
    C, H, W = fmap.shape
    out = np.full((len(boxes), PH * PW, C), -1, np.int64)
    for r, box in enumerate(boxes):
        for b, (hs, he, ws, we) in enumerate(roi_bin_windows(box, scale, variant, PW, PH, H, W)):
            if he <= hs or we <= ws:
                continue
            win = fmap[:, hs:he, ws:we].reshape(C, -1)                   # (h, w) scan order
            m = np.full(C, -FLT_MAX, np.float32)
            mi = np.full(C, -1, np.int64)
            for k in range(win.shape[1]):
                upd = win[:, k] > m
                m = np.where(upd, win[:, k], m)
                mi = np.where(upd, (hs + k // (we - ws)) * W + ws + k % (we - ws), mi)
            out[r, b] = mi
    return out


def roi_backward(grad_out, argmax, H, W):
    """the gather the device runs, restated as a scatter in (r, bin) order: grad_out / argmax R x bins x C -> C x H x W
    (np.add.at adds one by one in index order, in fp32: the device's summation order per cell)"""
    g = np.asarray(grad_out, np.float32)
    R, B, C = g.shape
    out = np.zeros((H * W, C), np.float32)
    sel = argmax >= 0
    cc = np.broadcast_to(np.arange(C), argmax.shape)
    np.add.at(out, (argmax[sel], cc[sel]), g[sel])
    return out.T.reshape(C, H, W)


def trunk_step_oracle(spec, k0, stored, rois_per_image, labels, targets, weights, gates, p, bbox_w=1.0, dev="cpu"):
    """fp64 losses and gradients {weight index: array} of one step with the trunk training from layer k0.
    stored[i]: {slot: C x H x W} of image i (the device's kept slots); gates: (tower, layer) -> R x cout, the device's
    backward gate through each per-ROI ReLU (inside its dropout mask)."""
    import torch
    dt = torch.float64
    params = {}

    def P(i):
        if i not in params:
            params[i] = torch.tensor(np.asarray(weights[i], np.float64), dtype=dt, device=dev, requires_grad=True)
        return params[i]

    T = spec.towers[0]
    slot, scale = T.levels[0]
    pooled = []
    for i, boxes in enumerate(rois_per_image):
        layers = spec.trunk_layers
        x = torch.tensor(stored[i][layers[k0].in_slot], dtype=dt, device=dev)[None]
        for L in layers[k0:]:
            if L.kind == 1:                                              # conv 3x3, ReLU at the device's side
                z = torch.nn.functional.conv2d(x, P(L.weight), P(L.bias), padding=1)
                x = z * torch.tensor(stored[i][L.out_slot] > 0, dtype=dt, device=dev)[None]
            else:                                                        # max pool at the device-derived argmax
                idx = torch.tensor(pool_argmax(stored[i][L.in_slot]), device=dev)
                Cc = x.shape[1]
                x = x.reshape(1, Cc, -1).gather(2, idx.reshape(1, Cc, -1)).reshape(1, Cc, idx.shape[1], idx.shape[2])
        fm = stored[i][slot]
        Cc, H, W = fm.shape
        am = roi_argmax(fm, boxes, scale, spec.roi_variant, T.pooled_w, T.pooled_h)   # R x bins x C
        flat = x.reshape(Cc, H * W)
        ok = torch.tensor(am >= 0, device=dev)
        g = flat[torch.arange(Cc, device=dev)[None, None, :].expand(am.shape), torch.tensor(np.maximum(am, 0), device=dev)]
        pooled.append(g * ok)                                            # R x bins x C, (h, w, c)
    x = torch.cat(pooled, 0)
    R = x.shape[0]
    x = x.reshape(R, T.pooled_h, T.pooled_w, -1).permute(0, 3, 1, 2)
    slots = {0: x}
    for li, L in enumerate(T.layers):
        x = slots[L.in_slot]
        if L.kind == 4:
            y = x.reshape(R, -1)
        else:
            y = x @ P(L.weight).reshape(L.cout, -1).T + P(L.bias)
            if L.relu:
                y = y * torch.tensor(gates[(0, li)], dtype=dt, device=dev) / (1.0 - p)
        slots[L.out_slot] = y
    cat = slots[T.out_slot]
    hc, hb = spec.cls_heads[0], spec.bbox_head
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

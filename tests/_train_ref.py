"""fp64 restatements for the training tests: the per-ROI graph with torch autograd, the criteria and optim.sgd in numpy,
Philox4x32-10 in numpy."""
import numpy as np

M0, M1, W0, W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85


def philox4x32_10(ctr, key):
    """ctr: 4 x n uint64 arrays of 32-bit words, key: 2 words -> 4 x n output words"""
    c = [np.asarray(x, np.uint64) & 0xFFFFFFFF for x in ctr]
    k0, k1 = np.uint64(key[0]), np.uint64(key[1])
    mask = np.uint64(0xFFFFFFFF)
    for i in range(10):
        if i > 0:
            k0 = (k0 + np.uint64(W0)) & mask
            k1 = (k1 + np.uint64(W1)) & mask
        p0 = np.uint64(M0) * c[0]
        p1 = np.uint64(M1) * c[2]
        hi0, lo0 = p0 >> np.uint64(32), p0 & mask
        hi1, lo1 = p1 >> np.uint64(32), p1 & mask
        c = [hi1 ^ c[1] ^ k0, lo1, hi0 ^ c[3] ^ k1, lo0]
    return c


def dropout_keep(seed, step, tower, layer, elems, p):
    """csrc/train_rule.cuh: counter (element / 4, step, tower << 16 | layer, 0), key (seed lo, seed hi), word element % 4,
    keep iff word >> 8 >= floor(p * 2^24)"""
    e = np.asarray(elems, np.uint64)
    q = e >> np.uint64(2)
    n = e.shape[0]
    out = philox4x32_10([q & np.uint64(0xFFFFFFFF), q >> np.uint64(32), np.full(n, step, np.uint64),
                         np.full(n, (tower << 16) | layer, np.uint64)], (seed & 0xFFFFFFFF, seed >> 32))
    words = np.stack(out)[(e & np.uint64(3)).astype(np.int64), np.arange(n)]
    return (words >> np.uint64(8)) >= np.uint64(int(float(p) * 16777216.0))


def criteria(x, d, labels, t, bbox_w=1.0):
    """nn.ParallelCriterion{CrossEntropy, BBoxRegression x bbox_w} in fp64 -> (total, ce, bbox, d/dx, d/dd)"""
    x, d, t = (np.asarray(a, np.float64) for a in (x, d, t))
    R, C = x.shape
    lab = np.asarray(labels) - 1
    m = x.max(1, keepdims=True)
    e = np.exp(x - m)
    s = e.sum(1, keepdims=True)
    ce = float(np.mean((m + np.log(s))[:, 0] - x[np.arange(R), lab]))
    gx = e / s
    gx[np.arange(R), lab] -= 1.0
    gx /= R
    masked = np.zeros_like(d)
    for r in range(R):
        if lab[r] > 0:
            masked[r, 4 * lab[r]:4 * lab[r] + 4] = d[r, 4 * lab[r]:4 * lab[r] + 4]
    diff = masked - t
    ad = np.abs(diff)
    sl1 = float(np.where(ad < 1, 0.5 * diff * diff, ad - 0.5).sum() / R)
    gd = np.clip(diff, -1.0, 1.0) / R * bbox_w
    return ce + bbox_w * sl1, ce, sl1, gx, gd


def sgd(w, g, buf, lr, momentum, dampening, wd, first):
    """optim.sgd as recalled (one explicit fma per multiply-add, computed exactly in long double)"""
    L = np.longdouble
    f = lambda a, b, c: (L(a) * L(b) + L(c)).astype(np.float32)   # noqa: E731
    w, g, buf = (np.asarray(a, np.float32) for a in (w, g, buf))
    gg = f(np.float32(wd), w, g) if wd != 0 else g
    if momentum != 0:
        buf = gg.copy() if first else f(np.float32(momentum), buf, np.float32(1.0 - np.float32(dampening)) * gg)
        gg = buf
    return f(np.float32(-lr), gg, w), buf


def per_roi_forward(spec, pooled, masks, p, weights, dev="cpu", gates=None):
    """the towers and heads of `spec` in fp64 on the given pooled rows (tower -> R x bins x Ctot, channels last) and
    dropout masks ((tower, layer) -> R x cout) -> (logits, deltas, params{index: leaf tensor}).
    gates ((tower, layer) -> R x cout, optional): the device's ReLU (+ dropout) gate of a per-ROI Linear (2-D output; a
    convolution on a map keeps relu), used in place of
    relu(z) * mask, so that a pre-activation within rounding of 0 takes the device's side of the kink: the value differs
    from the exact one by that rounding only, the derivative is the device's."""
    import torch
    dt = torch.float64
    params = {}

    def P(i):
        if i not in params:
            params[i] = torch.tensor(np.asarray(weights[i], np.float64), dtype=dt, device=dev, requires_grad=True)
        return params[i]

    outs = []
    for t, T in enumerate(spec.towers):
        R = pooled[t].shape[0]
        x0 = torch.tensor(pooled[t], dtype=dt, device=dev).reshape(R, T.pooled_h, T.pooled_w, -1).permute(0, 3, 1, 2)
        slots = {0: x0}
        for li, L in enumerate(T.layers):
            x = slots[L.in_slot]
            if L.kind == 4:                                          # FLATTEN: Torch (c, h, w) order
                y = x.reshape(R, -1)
            else:
                W = P(L.weight)
                b = P(L.bias) if L.bias >= 0 else None
                if x.dim() == 4:
                    y = torch.nn.functional.conv2d(x, W.reshape(L.cout, -1, 1, 1), b)
                else:
                    y = x @ W.reshape(L.cout, -1).T + (b if b is not None else 0)
                if L.relu and y.dim() == 2 and gates is not None and (t, li) in gates:
                    y = y * torch.tensor(gates[(t, li)], dtype=dt, device=dev) / (1.0 - p)
                elif L.relu:
                    y = torch.relu(y)
                    if p > 0 and y.dim() == 2:
                        y = y * torch.tensor(masks[(t, li)], dtype=dt, device=dev) / (1.0 - p)
            slots[L.out_slot] = y
        outs.append(slots[T.out_slot])
    cat = torch.cat(outs, 1)
    hc, hb = spec.cls_heads[0], spec.bbox_head
    logits = cat[:, hc.col_begin:hc.col_begin + hc.col_len] @ P(hc.weight).T + P(hc.bias)
    deltas = cat[:, hb.col_begin:hb.col_begin + hb.col_len] @ P(hb.weight).T + P(hb.bias)
    return logits, deltas, params


def step_oracle(spec, pooled, masks, p, weights, labels, targets, bbox_w=1.0, dev="cpu", gates=None):
    """fp64 losses and gradients {weight index: array} of one step"""
    import torch
    logits, deltas, params = per_roi_forward(spec, pooled, masks, p, weights, dev, gates)
    R = logits.shape[0]
    lab = torch.tensor(np.asarray(labels, np.int64) - 1, device=dev)
    ce = torch.nn.functional.cross_entropy(logits, lab)
    sel = torch.zeros_like(deltas)
    rows = torch.nonzero(lab > 0)[:, 0]
    for k in range(4):
        sel[rows, 4 * lab[rows] + k] = 1.0
    # the value is the masked buffer; its gradient reaches every delta unmasked (BBoxRegressionCriterion.lua:38-41)
    masked = deltas * sel + (deltas - deltas.detach()) * (1.0 - sel)
    diff = masked - torch.tensor(targets, dtype=torch.float64, device=dev)
    ad = diff.abs()
    sl1 = torch.where(ad < 1, 0.5 * diff * diff, ad - 0.5).sum() / R
    loss = ce + bbox_w * sl1
    loss.backward()
    grads = {i: t.grad.detach().cpu().numpy() for i, t in params.items()}
    return (loss.item(), ce.item(), sl1.item()), grads, (logits.detach().cpu().numpy(), deltas.detach().cpu().numpy())

"""fp64 oracle of a fixed-batch-norm Inception-v3 training step (Trainer on models.inception_v3_fast_rcnn(fixed_bn=True):
the tower Mixed_7a .. 7c and the heads, the trunk frozen): torch autograd on the UNFOLDED tower, every recorded
convolution as conv2d(x, W, padding=(ph, pw)) * a + b with W = W' / a the leaf and a, b constants (inceptionv3.lua's
BNtoFixed), from the device's pooled map through the branches, their concatenations, the windowed and max pools, the
average pool and the heads. As _train_resnet_ref does, the oracle takes from the device what decides a branch: every
ReLU side (the device's gates). Gradients come back in the device's parameterisation: dL/dW' = dL/dW / a per output
channel for a recorded weight."""
import numpy as np

from _train_resnet_ref import unfolded

CONV, MAXPOOL, AVGPOOL, AVGPOOL_WIN = 1, 2, 3, 6


def joined(planes):
    """the fp64 value hi + lo of split planes (uint16 bf16 bits)"""
    f = lambda p: (p.astype(np.uint32) << 16).view(np.float32).astype(np.float64)
    return f(planes["hi"]) + f(planes["lo"])


def inception_step_oracle(spec, pooled, labels, targets, weights, gates, head=0, bbox_w=1.0, dev="cpu"):
    """fp64 losses and gradients {weight index: dL/d(stored parameter)} of one step. pooled: R x PH x PW x C, the device's
    pooled map (a constant: the trunk is frozen); weights: the spec's folded arrays (W'); gates: tower layer index ->
    (R * pixels) x cout, the device's backward gate of each per-ROI ReLU."""
    import torch
    F = torch.nn.functional                        # looked up at each call: _train_bf16_ref.bf16_operands swaps conv2d
    dt = torch.float64
    W = unfolded(spec, weights)
    params = {}

    def P(i):
        if i not in params:
            params[i] = torch.tensor(W[i], dtype=dt, device=dev, requires_grad=True)
        return params[i]

    def const(x):
        return torch.tensor(np.asarray(x, np.float64), dtype=dt, device=dev)

    T = spec.towers[0]
    R = pooled.shape[0]
    parts = {0: [(0, const(pooled).permute(0, 3, 1, 2))]}     # slot -> [(channel offset, R x c x h x w)]

    def read(s):
        return torch.cat([t for _, t in sorted(parts[s], key=lambda p: p[0])], 1)

    for li, L in enumerate(T.layers):
        x = read(L.in_slot)
        if L.kind == AVGPOOL:
            y = x.mean(dim=(2, 3))
        elif L.kind == MAXPOOL:
            y = F.max_pool2d(x, L.kh, L.stride, L.pad, ceil_mode=bool(L.ceil_mode))
        elif L.kind == AVGPOOL_WIN:
            y = F.avg_pool2d(x, L.kh, L.stride, L.pad, ceil_mode=bool(L.ceil_mode), count_include_pad=not L.exclude_pad)
        else:
            pad = (L.pad, L.padw)
            if L.weight in spec.fixed_bn:              # ConstAffine after a bias-free convolution
                a = const(spec.fixed_bn[L.weight])[None, :, None, None]
                y = F.conv2d(x, P(L.weight), None, stride=L.stride, padding=pad) * a + const(weights[L.bias])[None, :, None, None]
            else:
                y = F.conv2d(x, P(L.weight), P(L.bias), stride=L.stride, padding=pad)
            if L.relu:
                gt = np.asarray(gates[li]).reshape(R, y.shape[2], y.shape[3], -1).transpose(0, 3, 1, 2)
                y = y * const(gt)
        parts.setdefault(L.out_slot, []).append((L.out_c_off, y))
    cat = read(T.out_slot)
    hc, hb = spec.cls_heads[head], spec.bbox_head
    logits = cat[:, hc.col_begin:hc.col_begin + hc.col_len] @ P(hc.weight).T + P(hc.bias)
    deltas = cat[:, hb.col_begin:hb.col_begin + hb.col_len] @ P(hb.weight).T + P(hb.bias)
    lab = torch.tensor(np.asarray(labels, np.int64) - 1, device=dev)
    ce = F.cross_entropy(logits, lab)
    sel = torch.zeros_like(deltas)
    rows = torch.nonzero(lab > 0)[:, 0]
    for k in range(4):
        sel[rows, 4 * lab[rows] + k] = 1.0
    masked = deltas * sel + (deltas - deltas.detach()) * (1.0 - sel)
    diff = masked - const(targets)
    ad = diff.abs()
    sl1 = torch.where(ad < 1, 0.5 * diff * diff, ad - 0.5).sum() / R
    loss = ce + bbox_w * sl1
    loss.backward()
    grads = {}
    for i, t in params.items():
        g = t.grad.detach().cpu().numpy()
        if i in spec.fixed_bn:
            g = g / np.asarray(spec.fixed_bn[i], np.float64)[:, None, None, None]
        grads[i] = g
    return (loss.item(), ce.item(), sl1.item()), grads


def avgpool_win_backward_np(g, H, W, k, s, p, exclude_pad):
    """numpy restatement of the device's windowed average pool backward, in its fp32 summation order: g n x Ho x Wo x C
    (fp32) -> n x H x W x C, per cell the sum from +0 over (ky, kx) of g / count of the window that holds the cell at tap
    (ky, kx)"""
    n, Ho, Wo, C = g.shape
    g = g.astype(np.float32)
    out = np.zeros((n, H, W, C), np.float32)
    cnt = np.zeros((Ho, Wo), np.float32)
    for ho in range(Ho):
        for wo in range(Wo):
            h0, w0 = ho * s - p, wo * s - p
            h1, w1 = min(h0 + k, H + p), min(w0 + k, W + p)
            c = (h1 - h0) * (w1 - w0)
            if exclude_pad:
                c = (min(h1, H) - max(h0, 0)) * (min(w1, W) - max(w0, 0))
            cnt[ho, wo] = max(c, 1)
    q = g / cnt[None, :, :, None]                     # fp32 division, as the kernel's g / (float)count
    for h in range(H):
        for w in range(W):
            acc = np.zeros((n, C), np.float32)
            for ky in range(k):
                th = h + p - ky
                if th < 0 or th % s or th // s >= Ho:
                    continue
                for kx in range(k):
                    tw = w + p - kx
                    if tw < 0 or tw % s or tw // s >= Wo:
                        continue
                    acc = acc + q[:, th // s, tw // s, :]
            out[:, h, w, :] = acc
    return out

"""fp64 oracle of a fixed-batch-norm ResNet training step (Trainer on models.resnet{18,50}_fast_rcnn(fixed_bn=True) with
the trunk training): torch autograd on the UNFOLDED graph, every recorded convolution as conv2d(x, W) * a + b with
W = W' / a the leaf and a, b constants (resnet.lua's BNtoFixed), from each image's stored input of the first trained
trunk layer through the trunk blocks, ROI pooling, layer4, the average pool and the heads. As _train_trunk_ref does,
the oracle takes from the device what decides a branch: every ReLU side (the stored output > 0, per ROI the device's
gates) and every ROI argmax. Gradients come back in the device's parameterisation: dL/dW' = dL/dW / a per output
channel for a recorded weight."""
import numpy as np

from _train_trunk_ref import roi_argmax

CONV, AVGPOOL = 1, 3


def unfolded(spec, weights):
    """{weight index: W = W' / a (fp64)} for the recorded convolutions, the other entries as given (fp64)"""
    out = {}
    for i, w in enumerate(weights):
        w = np.asarray(w, np.float64)
        if i in spec.fixed_bn:
            w = w / np.asarray(spec.fixed_bn[i], np.float64)[:, None, None, None]
        out[i] = w
    return out


def resnet_step_oracle(spec, stored, rois_per_image, labels, targets, weights, gates, head=0, bbox_w=1.0, dev="cpu"):
    """fp64 losses and gradients {weight index: dL/d(stored parameter)} of one step, the trunk training from
    spec.trunk_train_from. weights: the spec's folded arrays (W'); stored[i]: {slot: C x H x W} of image i; gates:
    tower layer index -> (R * pixels) x cout, the device's backward gate of each per-ROI ReLU."""
    import torch
    import torch.nn.functional as F
    dt = torch.float64
    k0 = spec.trunk_train_from
    W = unfolded(spec, weights)
    params = {}

    def P(i):
        if i not in params:
            params[i] = torch.tensor(W[i], dtype=dt, device=dev, requires_grad=True)
        return params[i]

    def const(x):
        return torch.tensor(np.asarray(x, np.float64), dtype=dt, device=dev)

    def conv(L, x):
        if L.weight in spec.fixed_bn:                  # ConstAffine after a bias-free convolution
            a = const(spec.fixed_bn[L.weight])[None, :, None, None]
            return F.conv2d(x, P(L.weight), None, stride=L.stride, padding=L.pad) * a + const(weights[L.bias])[None, :, None, None]
        return F.conv2d(x, P(L.weight), P(L.bias), stride=L.stride, padding=L.pad)

    T = spec.towers[0]
    top, scale = T.levels[0]
    pooled = []
    for i, boxes in enumerate(rois_per_image):
        slots = {spec.trunk_layers[k0].in_slot: const(stored[i][spec.trunk_layers[k0].in_slot])[None]}
        for L in spec.trunk_layers[k0:]:
            z = conv(L, slots[L.in_slot])
            if L.residual_slot >= 0:
                z = z + slots[L.residual_slot]
            if L.relu:
                z = z * const(stored[i][L.out_slot] > 0)[None]
            slots[L.out_slot] = z
        fm = stored[i][top]
        Cc, H, Wd = fm.shape
        am = roi_argmax(fm, boxes, scale, spec.roi_variant, T.pooled_w, T.pooled_h)     # R x bins x C
        flat = slots[top].reshape(Cc, H * Wd)
        ok = torch.tensor(am >= 0, device=dev)
        g = flat[torch.arange(Cc, device=dev)[None, None, :].expand(am.shape), torch.tensor(np.maximum(am, 0), device=dev)]
        pooled.append(g * ok)
    x = torch.cat(pooled, 0)
    R = x.shape[0]
    slots = {0: x.reshape(R, T.pooled_h, T.pooled_w, -1).permute(0, 3, 1, 2)}
    for li, L in enumerate(T.layers):
        x = slots[L.in_slot]
        if L.kind == AVGPOOL:
            y = x.mean(dim=(2, 3))
        else:
            y = conv(L, x)
            if L.residual_slot >= 0:
                y = y + slots[L.residual_slot]
            if L.relu:
                gt = np.asarray(gates[li]).reshape(R, y.shape[2], y.shape[3], -1).transpose(0, 3, 1, 2)
                y = y * const(gt)
        slots[L.out_slot] = y
    cat = slots[T.out_slot]
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


def sgd_unfolded(spec, w, buf, grads_folded, lr, mom, wd, first, biases):
    """one optim.sgd step on the UNFOLDED parameters (fp64, in place): w / buf {index: W or folded entry}, grads in the
    device's parameterisation (dL/dW' for a recorded weight: dL/dW = a * dL/dW')"""
    for i, g in grads_folded.items():
        if i in spec.fixed_bn:
            g = g * np.asarray(spec.fixed_bn[i], np.float64)[:, None, None, None]
        g = g + (0.0 if i in biases else wd) * w[i]
        buf[i] = g if first else mom * buf[i] + g
        w[i] = w[i] - lr * buf[i]


def fold(spec, w):
    """W' = a * W of the recorded entries of an unfolded dict"""
    return {i: (v * np.asarray(spec.fixed_bn[i], np.float64)[:, None, None, None] if i in spec.fixed_bn else v) for i, v in w.items()}

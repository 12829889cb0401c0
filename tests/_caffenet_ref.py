"""Restatements for CaffeNet's device layers (tests/test_caffenet_{cpu,gpu}.py).

lrn_rule: csrc/lrn_rule.cuh's arithmetic in numpy fp32, one rounded operation per step, so it pins the host build and
lrn_split_kernel bit for bit. lrn64 / grouped_conv64: the same layers in fp64 (torch), the bars' reference."""
import numpy as np
import torch
import torch.nn.functional as F

A = np.float32(1e-4 / 5)          # (float)(1e-4 / 5)


def lrn_rule(x):
    """x (..., C) fp32 -> y (..., C) fp32: q_j = x_j^2; S_c = q_{c-2} + .. + q_{c+2} inside [0, C), ascending from the first
    term; s = 1 + a S; d = sqrt(s) sqrt(sqrt(s)); y = x_c / d"""
    x = np.asarray(x, np.float32)
    C = x.shape[-1]
    q = x * x
    S = np.zeros_like(x)
    with np.errstate(over="ignore", invalid="ignore"):
        for c in range(C):
            j0, j1 = max(c - 2, 0), min(c + 2, C - 1)
            s = q[..., j0].copy()
            for j in range(j0 + 1, j1 + 1):
                s = s + q[..., j]
            S[..., c] = s
        s = np.float32(1) + A * S
        r = np.sqrt(s)
        return x / (r * np.sqrt(r))


def lrn64(x):
    """fp64 y_c = x_c / (1 + 1e-4 / 5 * S_c)^0.75 of x (..., C)"""
    x = torch.as_tensor(np.asarray(x), dtype=torch.float64)
    q = F.pad((x * x).unsqueeze(0), (2, 2)).squeeze(0)
    S = sum(q[..., k:k + x.shape[-1]] for k in range(5))
    return (x / (1.0 + 1e-4 / 5 * S) ** 0.75).numpy()


def alpha_s(x):
    """a * S_c in fp64 for x (..., C): how far the LRN is from the identity"""
    x = torch.as_tensor(np.asarray(x), dtype=torch.float64)
    q = F.pad((x * x).unsqueeze(0), (2, 2)).squeeze(0)
    return (1e-4 / 5 * sum(q[..., k:k + x.shape[-1]] for k in range(5))).numpy()


def split_planes(y):
    """the split store: hi = rn_bf16(y), lo = rn_bf16(y - hi); returns hi + lo in fp32"""
    t = torch.as_tensor(np.ascontiguousarray(y, np.float32))
    hi = t.to(torch.bfloat16).float()
    lo = (t - hi).to(torch.bfloat16).float()
    return (hi + lo).numpy()


def lrn_inputs(rng, C, n=3, h=5, w=7):
    """NHWC inputs whose a * S spans 1e-3 .. 1e3 across pixels, with zeros, both signs and the edge channels exercised"""
    x = rng.standard_normal((n, h, w, C)).astype(np.float32)
    # per pixel scale 10^u, u in [0.5, 3.5]: a * S ~ 1e-4 * x^2 from ~1e-3 to ~1e3
    u = rng.uniform(0.5, 3.5, (n, h, w, 1)).astype(np.float32)
    x = x * np.power(np.float32(10), u)
    x[0, 0, 0, :] = 0                                  # a zero pixel
    x[0, 0, 1, ::3] = 0                                # zeros inside a window
    x[0, 1, 0, 0] = -x[0, 1, 0, 0]                     # signs at the edge channels
    x[0, 1, 0, -1] = -abs(x[0, 1, 0, -1])
    return x.astype(np.float32)


def grouped_conv64(x_nchw, w, b, groups, stride, pad, relu=True):
    xd = torch.as_tensor(np.asarray(x_nchw), dtype=torch.float64)
    y = F.conv2d(xd, torch.as_tensor(np.asarray(w), dtype=torch.float64),
                 None if b is None else torch.as_tensor(np.asarray(b), dtype=torch.float64), stride=stride, padding=pad, groups=groups)
    return (torch.relu(y) if relu else y).numpy()


LRN_TYPES = ("SpatialCrossMapLRN", "SpatialCrossResponseNormalization")


def evaluate_nn(m, x):
    """a torch nn graph (T7Object tree) evaluated module by module in eval mode, fp32 on the CPU: tests/_nn_interp.py plus
    what CaffeNet adds (grouped cudnn.SpatialConvolution, the cross-map LRN modules, as torch's local_response_norm)"""
    from multipathnet_b200.t7 import _base, _children
    import _nn_interp as NI
    b, kids = _base(m.typename), _children(m)
    if b == "Sequential":
        for c in kids:
            x = evaluate_nn(c, x)
        return x
    if b == "ConcatTable":
        return [evaluate_nn(c, x) for c in kids]
    if b == "ParallelTable":
        return [evaluate_nn(c, xi) for c, xi in zip(kids, x)]
    if b in ("SpatialConvolution", "SpatialConvolutionMM"):
        g = int(m.get("groups", 1) or 1)
        return F.conv2d(x, NI._t(m.weight), NI._t(m.bias), stride=int(m.dW), padding=int(m.get("padW", 0)), groups=g)
    if b in LRN_TYPES:
        return F.local_response_norm(x, int(m.size), alpha=float(m.alpha), beta=float(m.beta), k=float(m.k))
    return NI.evaluate(m, x)

"""Oracle of the bf16 training step (Trainer(bf16=True)): the fp64 oracles of _train_ref, _train_trunk_ref,
_train_resnet_ref and _train_phase2_ref, unchanged, run inside `bf16_operands`, which makes every convolution
(torch.nn.functional.conv2d) and every Linear (the `@` of the per-ROI layers and heads) round its forward operands
(x, W) and its backward operands (grad_out, x, W) to bf16, round to nearest even, as the device's BF16X1 GEMMs read
them. acc=torch.float32 sums the same products in fp32: the distance between the two is the oracle's own order
sensitivity (DESIGN 4, the bf16 inference mode's methodology)."""
import contextlib
import dataclasses

import numpy as np


def rn_bf16(x):
    """fp32 -> the nearest bf16 (ties to even), as fp32"""
    b = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((b + 0x7FFF + ((b >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32)


def split_planes(x):
    """fp32 -> (hi, lo) uint16 planes with hi = rn_bf16(x), lo = rn_bf16(x - hi): the device's split_bf16"""
    x = np.ascontiguousarray(x, np.float32)
    hi = rn_bf16(x)
    lo = rn_bf16(x - hi)
    return (hi.view(np.uint32) >> 16).astype(np.uint16), (lo.view(np.uint32) >> 16).astype(np.uint16)


def planes_value(p):
    return (p.astype(np.uint32) << 16).view(np.float32)


@contextlib.contextmanager
def bf16_operands(acc=None):
    """within: conv2d and Tensor.__matmul__ take rn_bf16 operands forward and a rn_bf16 output gradient backward (so dX
    and dW are products of bf16 operands), summed in `acc` (default fp64) and returned in the input's dtype"""
    import torch
    F = torch.nn.functional
    acc = torch.float64 if acc is None else acc

    def rn(t):
        return t.to(torch.float32).to(torch.bfloat16).to(t.dtype)

    class RoundIn(torch.autograd.Function):          # an operand: rounded forward, its gradient passed through
        @staticmethod
        def forward(ctx, x):
            return rn(x)

        @staticmethod
        def backward(ctx, g):
            return g

    class RoundGrad(torch.autograd.Function):        # an output: as is forward, its gradient rounded backward
        @staticmethod
        def forward(ctx, y):
            return y.clone()

        @staticmethod
        def backward(ctx, g):
            return rn(g)

    conv0, mm0 = F.conv2d, torch.Tensor.__matmul__

    def conv2d(x, w, bias=None, stride=1, padding=0, dilation=1, groups=1):
        y = conv0(RoundIn.apply(x).to(acc), RoundIn.apply(w).to(acc), None, stride, padding, dilation, groups).to(x.dtype)
        y = RoundGrad.apply(y)
        return y if bias is None else y + bias[None, :, None, None]

    def matmul(a, b):
        return RoundGrad.apply(mm0(RoundIn.apply(a).to(acc), RoundIn.apply(b).to(acc)).to(a.dtype))

    F.conv2d, torch.Tensor.__matmul__ = conv2d, matmul
    try:
        yield
    finally:
        F.conv2d, torch.Tensor.__matmul__ = conv0, mm0


def unit_scales(spec):
    """a fixed-batch-norm spec whose recorded scales are all 1: _train_resnet_ref then runs conv2d(x, W') + b on the
    folded weights the device rounds, and its gradients are dL/dW' as they stand"""
    return dataclasses.replace(spec, fixed_bn={i: np.ones_like(np.asarray(a, np.float32)) for i, a in spec.fixed_bn.items()})


def three_oracles(run):
    """run(): (losses, grads) of a wrapped oracle -> (plain fp64, bf16 operands in fp64, bf16 operands summed in fp32)"""
    import torch
    plain = run()
    with bf16_operands():
        b64 = run()
    with bf16_operands(torch.float32):
        b32 = run()
    return plain, b64, b32


def rel(a, b):
    a = np.asarray(a, np.float64); b = np.asarray(b, np.float64)
    return float(np.max(np.abs(a - b)) / max(np.max(np.abs(b)), 1e-30))


def bars(dev_losses, dev_grads, plain, b64, b32):
    """per quantity (the three losses, every gradient): (device vs bf16 oracle, its bar max(1e-3, 3 x sensitivity), device
    vs plain fp64, its sanity bar max(5e-2, 3 x |bf16 oracle - plain|))"""
    out = {}
    names = [("loss", k) for k in range(3)] + [("grad", i) for i in b64[1]]
    for kind, k in names:
        if kind == "loss":
            d, p, o, s = dev_losses[k], plain[0][k], b64[0][k], b32[0][k]
        else:
            d, p, o, s = dev_grads[k], plain[1][k], b64[1][k], b32[1][k]
        out[(kind, k)] = (rel(d, o), max(1e-3, 3 * rel(s, o)), rel(d, p), max(5e-2, 3 * rel(o, p)))
    return out

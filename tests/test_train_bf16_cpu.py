"""CPU: the bf16 training oracle (_train_bf16_ref): rn_bf16 and the split planes against torch's conversion, and
bf16_operands' conv2d / Linear against the products of explicitly rounded operands, forward and backward; the header
documents the "train_bf16" option."""
import os

import numpy as np
import torch

from _train_bf16_ref import bf16_operands, planes_value, rn_bf16, split_planes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _rn(t):
    return t.to(torch.float32).to(torch.bfloat16).to(t.dtype)


def test_rn_bf16_is_round_to_nearest_even():
    rng = np.random.default_rng(0)
    x = np.concatenate([rng.standard_normal(100000).astype(np.float32) * 10.0 ** rng.integers(-30, 30, 100000),
                        np.array([1 + 2 ** -8, 1 + 3 * 2 ** -8, -(1 + 2 ** -8), 0.0, -0.0], np.float32)])
    want = torch.from_numpy(x).to(torch.bfloat16).to(torch.float32).numpy()
    assert np.array_equal(rn_bf16(x).view(np.uint32), want.view(np.uint32))
    assert rn_bf16(np.float32(1 + 2 ** -8)) == 1.0 and rn_bf16(np.float32(1 + 3 * 2 ** -8)) == np.float32(1 + 2 ** -6)
    hi, lo = split_planes(x[:1000])
    assert np.array_equal(planes_value(hi), rn_bf16(x[:1000]))
    assert np.all(np.abs(planes_value(hi).astype(np.float64) + planes_value(lo) - x[:1000]) <= np.abs(x[:1000]) * 2.0 ** -16)


def test_bf16_operands_round_forward_and_backward_operands():
    g = torch.Generator().manual_seed(1)
    x = torch.randn(2, 8, 5, 6, dtype=torch.float64, generator=g, requires_grad=True)
    w = torch.randn(4, 8, 3, 3, dtype=torch.float64, generator=g, requires_grad=True)
    b = torch.randn(4, dtype=torch.float64, generator=g, requires_grad=True)
    go = torch.randn(2, 4, 5, 6, dtype=torch.float64, generator=g)
    a = torch.randn(7, 16, dtype=torch.float64, generator=g, requires_grad=True)
    m = torch.randn(16, 3, dtype=torch.float64, generator=g, requires_grad=True)
    gm = torch.randn(7, 3, dtype=torch.float64, generator=g)
    with bf16_operands():
        y = torch.nn.functional.conv2d(x, w, b, padding=1)
        z = a @ m
    (y * go).sum().backward()
    (z * gm).sum().backward()
    # by hand: operands rounded, the output gradient rounded, products in fp64
    xr, wr = _rn(x.detach()).requires_grad_(), _rn(w.detach()).requires_grad_()
    yr = torch.nn.functional.conv2d(xr, wr, None, padding=1) + b.detach()[None, :, None, None]
    assert torch.equal(y.detach(), yr.detach())
    yr.backward(_rn(go))
    assert torch.allclose(x.grad, xr.grad, rtol=0, atol=1e-12) and torch.allclose(w.grad, wr.grad, rtol=0, atol=1e-12)
    assert torch.allclose(b.grad, go.sum((0, 2, 3)), rtol=0, atol=1e-12)            # the bias takes the unrounded gradient
    ar, mr = _rn(a.detach()).requires_grad_(), _rn(m.detach()).requires_grad_()
    zr = ar @ mr
    assert torch.equal(z.detach(), zr.detach())
    zr.backward(_rn(gm))
    assert torch.allclose(a.grad, ar.grad, rtol=0, atol=1e-12) and torch.allclose(m.grad, mr.grad, rtol=0, atol=1e-12)
    # restored afterwards
    assert torch.equal(a.detach() @ m.detach(), torch.matmul(a.detach(), m.detach()))


def test_the_header_documents_the_option():
    with open(os.path.join(ROOT, "include", "mpn_abi.h")) as f:
        h = f.read()
    assert '"train_bf16"' in h

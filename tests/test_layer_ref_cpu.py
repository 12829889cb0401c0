"""The per-layer references of tests/_layer_ref.py on the CPU: row-sampled convolutions and pools equal the full Torch ops
on those rows, the operand rules reuse the oracles' rounding, and the FLATTEN permutation matches nn.View's order."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import _layer_ref as LR
from _bf16_oracle import rn_bf16
import _fp8_oracle as F8


def _getter(x):
    return lambda a, b: x[:, :, a:b]


@pytest.mark.parametrize("N,C,H,W,Co,k,s,p", [(1, 8, 17, 13, 5, 3, 1, 1), (2, 4, 16, 11, 3, 3, 2, 1), (1, 3, 23, 19, 4, 7, 2, 3),
                                              (3, 6, 9, 10, 7, 1, 1, 0), (1, 5, 14, 15, 6, 1, 2, 0), (1, 4, 12, 12, 4, 3, 1, 0)])
def test_conv_rows_equal_full_conv(N, C, H, W, Co, k, s, p):
    g = torch.Generator().manual_seed(N * 100 + H)
    x = torch.randn(N, C, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(Co, C, k, k, generator=g, dtype=torch.float64)
    b = torch.randn(Co, generator=g, dtype=torch.float64)
    full = F.conv2d(x, w, b, stride=s, padding=p)
    Ho = full.shape[2]
    rows = sorted({0, 1, Ho // 2, Ho - 2, Ho - 1} & set(range(Ho)))
    got = LR.conv_rows(_getter(x), H, w, b, s, p, rows)
    assert got.shape == full[:, :, rows].shape
    assert float((got - full[:, :, rows]).abs().max()) <= 1e-12 * float(full.abs().max())
    every = LR.conv_rows(_getter(x), H, w, b, s, p, list(range(Ho)))
    assert every.shape == full.shape and float((every - full).abs().max()) <= 1e-12 * float(full.abs().max())


@pytest.mark.parametrize("H,W,k,s,p,ceil", [(15, 13, 2, 2, 0, 1), (16, 12, 2, 2, 0, 1), (15, 13, 2, 2, 0, 0), (17, 21, 3, 2, 1, 0),
                                            (18, 20, 3, 2, 1, 1), (11, 9, 3, 2, 1, 0)])
def test_maxpool_rows_equal_full_pool(H, W, k, s, p, ceil):
    g = torch.Generator().manual_seed(H * W)
    x = torch.randn(2, 3, H, W, generator=g, dtype=torch.float64)
    full = F.max_pool2d(x, k, s, p, ceil_mode=bool(ceil))
    rows = list(range(full.shape[2]))
    got = LR.maxpool_rows(_getter(x), H, k, s, p, ceil, rows)
    assert got.shape == full.shape and torch.equal(got, full)


@pytest.mark.parametrize("H,W", [(15, 13), (16, 12), (9, 20)])
def test_conv_pool_rows_equal_full(H, W):
    g = torch.Generator().manual_seed(H + W)
    x = torch.randn(1, 4, H, W, generator=g, dtype=torch.float64)
    w = torch.randn(6, 4, 3, 3, generator=g, dtype=torch.float64)
    b = torch.randn(6, generator=g, dtype=torch.float64)
    full = F.max_pool2d(F.relu(F.conv2d(x, w, b, padding=1)), 2, 2, ceil_mode=True)
    Hp = full.shape[2]
    rows = sorted({0, 1, Hp // 2, Hp - 1})
    got = LR.conv_pool_rows(_getter(x), H, w, b, 1, True, rows)
    assert float((got - full[:, :, rows]).abs().max()) <= 1e-12 * float(full.abs().max())


def test_w16_reference_equals_the_engine_emulation():
    """the w16 operands restate test_engine_gpu's former _w16_emulation arithmetic, term by term"""
    rng = np.random.default_rng(4)
    A = np.maximum(rng.standard_normal((37, 256)), 0).astype(np.float32)
    B = (rng.standard_normal((70, 256)) / 16).astype(np.float32)
    B[0, :3] = [3.0, 1e-9, -2.5]
    bias = rng.standard_normal(70).astype(np.float32)
    a = torch.from_numpy(A)
    hi = a.to(torch.float16).float()
    a2 = (hi + (a - hi).to(torch.float16).float()).double()
    e = 14 - int(np.frexp(float(np.abs(B).max()))[1])
    b16 = (torch.from_numpy(B) * float(2.0 ** e)).to(torch.float16).double() / float(2.0 ** e)
    want = F.relu(a2 @ b16.t() + torch.from_numpy(bias).double()).float().numpy()
    assert np.array_equal(LR.w16_emulation(A, B, bias, True), want)
    assert torch.equal(LR.act_operand("w16", hi, (a - hi).to(torch.float16).float()), a2)
    assert torch.equal(LR.weight_operand("w16", torch.from_numpy(B)), b16)


def test_bf16_rule_on_a_2x2_case():
    """A = hi alone (the lo plane is ignored), W = rn_bf16(w) with ties to even"""
    hi = torch.tensor([[1.0, -2.0], [0.5, 3.0]])
    lo = torch.tensor([[2.0 ** -10, 0.0], [-2.0 ** -12, 2.0 ** -8]])
    w = torch.tensor([[1.0 + 2.0 ** -8, 1.0 + 3 * 2.0 ** -8], [-0.75, 2.0 ** -20]])      # ties: down to 1, up to 1 + 2^-6
    assert torch.equal(LR.act_operand("bf16", hi, lo), hi.double())
    wo = LR.weight_operand("bf16", w)
    assert wo.tolist() == [[1.0, 1.0 + 2.0 ** -6], [-0.75, 2.0 ** -20]]
    assert torch.equal(wo, rn_bf16(w).double())
    assert torch.equal(LR.act_operand("exact", hi, lo), hi.double() + lo.double())


def test_fp8_rule_on_a_2x2_case():
    """per-sample exponents of the hi plane and e4m3 rounding, as _fp8_oracle.quantize gives them"""
    hi = torch.tensor([[1.0, -3.0], [100.0, 0.0078125]])
    e = LR.act_exponents("fp8", hi)
    assert e.tolist() == [7, 2]                                       # 3 * 2^7 = 384 <= 448; 100 * 2^2 = 400 <= 448
    got = LR.act_operand("fp8", hi, torch.zeros(2, 2), e)
    q, eq = F8.quantize(hi)
    assert torch.equal(eq, e)
    assert torch.equal(got, q.double() * torch.ldexp(torch.ones(2, 1, dtype=torch.float64), -eq.double().reshape(2, 1)))
    assert got.tolist() == [[1.0, -3.0], [96.0, 0.0078125]]           # 400 -> e4m3 384 (3 mantissa bits)
    assert LR.act_exponents("fp8_per_tensor", hi).tolist() == [2, 2]
    w = torch.tensor([[0.3, -0.1], [5.0, 1e-3]])
    h = rn_bf16(w)
    qw, ew = F8.quantize(w)
    want = qw.double() * torch.ldexp(torch.ones(2, 1, dtype=torch.float64), -ew.double().reshape(2, 1))
    assert torch.equal(LR.weight_operand("fp8", w), want)
    assert torch.equal(LR.fp8_dequant(h, ew), want)


def test_flatten_permutation():
    """device FLATTEN rows are (h, w, c); Torch's nn.View of an N x C x H x W map is (c, h, w)"""
    x = torch.arange(2 * 3 * 4 * 5).reshape(2, 3, 4, 5)                # Torch N x C x H x W
    nhwc = x.permute(0, 2, 3, 1).contiguous()
    assert torch.equal(LR.flatten_nhwc_to_torch(nhwc), x.reshape(2, -1))
    assert LR.flatten_nhwc_to_torch(nhwc)[1, :6].tolist() == [60, 61, 62, 63, 64, 65]


def test_planes_decode():
    assert LR.bf16_values(np.array([0x3f80, 0xc000, 0x0000], np.uint16)).tolist() == [1.0, -2.0, 0.0]
    assert LR.plane_values(np.array([0x3c00, 0xc000], np.uint16), 1).tolist() == [1.0, -2.0]
    assert LR.e4m3_values(np.array([0x38, 0xb8, 0x7e], np.uint8)).tolist() == [1.0, -1.0, 448.0]


def test_row_sets():
    assert LR.trunk_rows(38) == [0, 1, 15, 16, 17, 18, 19, 21, 22, 36, 37]
    assert LR.trunk_rows(10) == [0, 1, 4, 5, 8, 9]
    assert LR.roi_rows(1000)[:5] == [0, 1, 127, 128, 129] and LR.roi_rows(1000)[-1] == 999
    r = LR.roi_rows(2000, np.random.default_rng(0))
    assert len(r) == 32 and r == sorted(set(r))

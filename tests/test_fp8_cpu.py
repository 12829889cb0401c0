"""The fp8 operand rule of csrc/fp8_e4m3.cuh, the code the device quantizers run, built into the library's host view
mpn_debug_fp8: scale exponents and e4m3 codes bit-exact against torch.float8_e4m3fn and the rule restated in Python
(tests/_fp8_oracle.py). No GPU needed."""
import os

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
import _fp8_oracle as F8

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def debug_fp8(h):
    """(exponents, codes) of h (n_samples x elems) from the product's host view; None if a sample has no scale"""
    h = np.ascontiguousarray(h, np.float32)
    e = np.zeros(h.shape[0], np.int32)
    q = np.zeros(h.shape, np.uint8)
    rc = mpn.load_library().mpn_debug_fp8(h.ctypes.data, h.shape[0], h[0].size, e.ctypes.data, q.ctypes.data)
    return None if rc != 0 else (e, q)


def torch_rule(h):
    t = torch.from_numpy(np.ascontiguousarray(h, np.float32))
    e = F8.scale_exponents(t)
    sc = torch.ldexp(torch.ones(len(e)), e.float()).reshape(-1, *([1] * (t.dim() - 1)))
    return e.numpy().astype(np.int32), (t * sc).to(torch.float8_e4m3fn).view(torch.uint8).numpy()


def bf16(a):
    return torch.from_numpy(np.ascontiguousarray(a, np.float32)).to(torch.bfloat16).float().numpy()


def check(h):
    got = debug_fp8(h)
    assert got is not None
    e, q = torch_rule(h)
    assert np.array_equal(got[0], e), (got[0], e)
    assert np.array_equal(got[1], q), np.argwhere(got[1] != q)[:8]
    return got


def test_every_code_round_trips():
    """the 254 finite e4m3 values (and -0) at scale 0: a sample whose max is 448 keeps e = 0, every value is its own code"""
    codes = np.array([c for c in range(256) if c & 0x7f != 0x7f], np.uint8)
    vals = torch.from_numpy(codes).view(torch.float8_e4m3fn).float().numpy()
    e, q = check(vals[None])
    assert e[0] == 0 and np.array_equal(q[0], codes)


def test_ties_subnormals_zero_and_448():
    # e = 0 throughout (max 448): midpoints between neighbours round to even, in the normal and the subnormal range
    mid_normal = [1.0625, 1.1875, 3.5 + 0.125, 240.0 - 8.0, 0.015625 * 1.0625, 0.015625 * 1.1875]
    mid_sub = [k * 2.0 ** -10 for k in range(1, 16, 2)]          # halfway points of the 2^-9 grid, down to 2^-10
    sub = [2.0 ** -9, 2.0 ** -8, 3 * 2.0 ** -9, 7 * 2.0 ** -9, 2.0 ** -6 - 2.0 ** -10, 2.0 ** -11, 2.0 ** -12]
    row = np.array([448.0, 0.0, -0.0, -448.0, 447.0, 440.0, 432.0] + mid_normal + mid_sub + sub, np.float32)
    row = np.concatenate([row, -row])
    e, q = check(row[None])
    assert e[0] == 0
    assert q[0, 0] == 0x7e and q[0, 1] == 0x00 and q[0, 2] == 0x80


@pytest.mark.parametrize("amax", [448.0, 449.0, 1.0, 0.875 * 2 ** -3, 0.876 * 2 ** -3, 1e-3, 3e4, 2.0 ** -140, 1e-38, 5e20])
def test_scale_rule(amax):
    rng = np.random.default_rng(int(np.log2(amax) * 7) % 1000)
    h = bf16(rng.uniform(-1, 1, (3, 97)) * amax)
    h[:, 5] = np.float32(bf16(np.float32(amax)))          # the group max itself
    e, q = check(h)
    for i in range(3):
        a = float(np.abs(h[i]).max())
        want = 0 if a == 0 else max(-60, min(60, max(k for k in range(-200, 201) if a * 2.0 ** k <= 448)))
        assert e[i] == want


def test_clamp_and_zero_groups():
    h = np.zeros((4, 64), np.float32)
    h[1, 3] = 1e-30                                       # e would be 105: clamped to 60
    h[2, :] = bf16(np.linspace(-3e20, 4e20, 64))          # e = -60 exactly fits
    h[3, 0] = 2.0 ** -133                                 # a bf16 subnormal: clamped, flushes to code 0
    e, q = check(h)
    assert list(e) == [0, 60, -60, 60]
    assert not q[0].any() and not q[3].any()


def test_random_groups_bit_exact():
    rng = np.random.default_rng(0)
    h = bf16(rng.standard_normal((64, 1000)) * np.exp(rng.uniform(-20, 20, (64, 1))))
    h[7] = 0.0
    h[9, 17] = 1e6                                        # one outlier: the other values of its group fall to subnormals / 0
    check(h)


def test_no_scale_for_non_finite_or_huge_groups():
    for bad in (np.inf, -np.inf, np.nan, 1e30):
        h = np.ones((2, 8), np.float32)
        h[1, 2] = bad
        assert debug_fp8(h) is None


def test_lua_flag():
    src = open(os.path.join(ROOT, "lua", "mpn_ffi.lua")).read()
    assert "os.getenv('mpn_fp8') == '1'" in src and "C.mpn_ctx_set_option(out[0], 'fp8', 1)" in src

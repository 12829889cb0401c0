"""Per-layer fp64 references for teacher-forced checks of a model's plan (tests/test_layers_gpu.py).

A layer is recomputed in fp64 from the planes it read on the device (mpn_model_get_slot_planes), with the operand rule of
the numerics in force, so the error of a layer does not depend on its depth. The rules (DESIGN 3, plan_trunk /
plan_heads in csrc/model.cu):

  rule        A operand                          W operand
  "exact"     hi + lo                            the fp32 weight             (default; the heads in every mode but bf16)
  "w16"       hi + lo of the fp16 planes         fp16(w * 2^e) / 2^e         (fc6 / fc7 of single-tower graphs)
  "bf16"      hi                                 rn_bf16(w)
  "fp8"       e4m3(2^e_s * hi) / 2^e_s           e4m3(2^e_c * rn_bf16(w)) / 2^e_c   (per sample s / output channel c)

Bias, residual (read back as hi + lo) and ReLU are applied in fp64. The first trunk convolution reads the fp32 image and
is computed in fp64 on it under every rule. "Wrong" rules for negative controls: "bf16_of_exact" (A = rn_bf16(hi + lo),
W = rn_bf16(w)), "w16_bf16w" (the w16 A operand with an rn_bf16 weight), "fp8_per_tensor" (one exponent for all samples).

Full-size maps are row-sampled: a convolution or pool is evaluated on chosen output rows from the input strip that feeds
them, zero-padded (or -inf-padded for a max) only at the true map border."""
import numpy as np
import torch
import torch.nn.functional as F

from _bf16_oracle import rn_bf16
import _fp8_oracle as F8


# ---------------------------------------------------------------- raw planes
def bf16_values(u16):
    """raw bf16 bits (uint16) -> fp32 values"""
    return (np.asarray(u16, np.uint16).astype(np.uint32) << 16).view(np.float32)


def plane_values(u16, fmt):
    """raw 16-bit plane -> fp32 values; fmt 0 = bf16, 1 = fp16"""
    return bf16_values(u16) if fmt == 0 else np.asarray(u16, np.uint16).view(np.float16).astype(np.float32)


def e4m3_values(u8):
    """raw e4m3 codes (uint8) -> fp32 values"""
    return torch.from_numpy(np.ascontiguousarray(u8, np.uint8)).view(torch.float8_e4m3fn).float()


def nhwc_to_nchw(a):
    """numpy N x H x W x C -> torch N x C x H x W (fp32)"""
    return torch.from_numpy(np.ascontiguousarray(a)).permute(0, 3, 1, 2).contiguous()


def flatten_nhwc_to_torch(x):
    """rows of a device FLATTEN, (h, w, c) order, -> Torch's nn.View order (c, h, w). x: N x H x W x C"""
    x = torch.as_tensor(x)
    return x.permute(0, 3, 1, 2).reshape(x.shape[0], -1)


# ---------------------------------------------------------------- operand rules
def _pow2(e, like):
    return torch.ldexp(torch.ones_like(like, dtype=torch.float64), e.double())


def fp8_dequant(h, e):
    """e4m3(2^e * h) / 2^e in fp64, h fp32 values already on the bf16 grid, e one exponent per dim-0 group (int tensor)"""
    sh = (-1,) + (1,) * (h.dim() - 1)
    sc = torch.ldexp(torch.ones(h.shape[0], dtype=torch.float32), e.float()).reshape(sh)
    q = (h.float() * sc).to(torch.float8_e4m3fn).double()
    return q * torch.ldexp(torch.ones(h.shape[0], dtype=torch.float64), -e.double()).reshape(sh)


def fp16_planes(a):
    """fp32 values -> the fp16 hi / lo planes the w16 layers store, as one fp64 value hi + lo"""
    a = torch.as_tensor(a, dtype=torch.float32)
    hi = a.to(torch.float16).float()
    return (hi + (a - hi).to(torch.float16).float()).double()


def w16_weight(w):
    """the w16 weight operand: fp16(w * 2^e) / 2^e in fp64, 2^e putting max|w| into [8192, 16384) (prepare_conv_weight_w16)"""
    w = torch.as_tensor(w, dtype=torch.float32)
    e = 14 - int(np.frexp(float(w.abs().max()))[1])
    return (w * float(2.0 ** e)).to(torch.float16).double() / float(2.0 ** e)


def w16_emulation(A, B, bias, relu):
    """what the w16 kernels compute, in fp64: (A_hi + A_lo) @ fp16(B * 2^e)^T / 2^e (+ bias)(ReLU) with A_hi / A_lo the fp16
    planes of A; the only difference left to the GPU is its fp32 accumulation"""
    y = fp16_planes(torch.from_numpy(A)) @ w16_weight(torch.from_numpy(B)).t()
    if bias is not None:
        y = y + torch.from_numpy(bias).double()
    return (F.relu(y) if relu else y).float().numpy()


def weight_operand(rule, w):
    """w: fp32 Torch-layout weight [Cout][...] -> fp64 operand"""
    w = torch.as_tensor(w, dtype=torch.float32)
    if rule == "exact":
        return w.double()
    if rule == "w16":
        return w16_weight(w)
    if rule in ("bf16", "bf16_of_exact", "w16_bf16w"):
        return rn_bf16(w).double()
    if rule in ("fp8", "fp8_per_tensor"):
        h = rn_bf16(w.reshape(w.shape[0], -1))
        return fp8_dequant(h, F8.scale_exponents(h)).reshape(w.shape)
    raise ValueError(rule)


def act_exponents(rule, hi):
    """per-sample fp8 exponents of an activation's hi plane (fp32, samples along dim 0); one shared exponent (the largest
    sample's) for "fp8_per_tensor"; None for the other rules"""
    if rule == "fp8":
        return F8.scale_exponents(hi)
    if rule == "fp8_per_tensor":
        e = F8.scale_exponents(hi)
        return torch.full_like(e, int(e.min()))
    return None


def act_operand(rule, hi, lo, e=None):
    """elementwise A operand (fp64) from the read-back planes' values (fp32 tensors); e: act_exponents for the fp8 rules"""
    if rule in ("exact", "w16", "w16_bf16w"):
        return hi.double() + lo.double()
    if rule == "bf16":
        return hi.double()
    if rule == "bf16_of_exact":
        return rn_bf16(hi + lo).double()
    if rule in ("fp8", "fp8_per_tensor"):
        return fp8_dequant(hi, e)
    raise ValueError(rule)


# ---------------------------------------------------------------- row sampling
def trunk_rows(H, rng=None, n_random=4):
    """output rows of a trunk map checked at full size: the borders, the 16-row patch edges, the middle, + seeded rows"""
    s = {0, 1, 15, 16, 17, H // 2 - 1, H // 2, H - 17, H - 16, H - 2, H - 1}
    if rng is not None:
        s |= set(int(r) for r in rng.integers(0, H, n_random))
    return sorted(r for r in s if 0 <= r < H)


def roi_rows(R, rng=None, n_random=26):
    """ROI rows of a per-ROI layer checked at full size: the first, the 128-row tile edges, the last, + seeded rows"""
    s = {0, 1, 127, 128, 129, R - 1}
    if rng is not None:
        s |= set(int(r) for r in rng.choice(R, min(n_random, R), replace=False))
    return sorted(r for r in s if 0 <= r < R)


def _strips(get, rows, k, stride, pad, H, fill):
    """N*len(rows) x C x k x W: the k input rows under each output row; rows beyond the map are `fill`"""
    out = []
    for r in rows:
        top = r * stride - pad
        a, b = max(top, 0), min(top + k, H)
        s = get(a, b)
        if a - top or top + k - b:
            s = F.pad(s, (0, 0, a - top, top + k - b), value=fill)
        out.append(s)
    return torch.stack(out, 0)                                  # len(rows) x N x C x k x W


def conv_rows(get, H, w, b, stride, pad, rows):
    """fp64 conv2d(x, w, b, stride, pad) on output rows `rows`: N x Cout x len(rows) x Wo. get(a, b) returns the fp64
    operand rows [a, b) of x (N x C x (b - a) x W)."""
    k = w.shape[2]
    S = _strips(get, rows, k, stride, pad, H, 0.0)
    n, N = S.shape[0], S.shape[1]
    y = F.conv2d(S.reshape(n * N, *S.shape[2:]), w, b, stride=(1, stride), padding=(0, pad))
    return y.reshape(n, N, y.shape[1], y.shape[3]).permute(1, 2, 0, 3)


def maxpool_rows(get, H, k, stride, pad, ceil_mode, rows):
    """max_pool2d on output rows `rows` from the input strips (-inf beyond the map): N x C x len(rows) x Wo"""
    S = _strips(get, rows, k, stride, pad, H, float("-inf"))
    n, N = S.shape[0], S.shape[1]
    y = F.max_pool2d(S.reshape(n * N, *S.shape[2:]), (k, k), stride=(stride, stride), padding=(0, pad), ceil_mode=bool(ceil_mode))
    return y.reshape(n, N, y.shape[1], y.shape[3]).permute(1, 2, 0, 3)


def conv_pool_rows(get, H, w, b, pad, relu, rows):
    """a 3x3 / stride 1 conv (+ ReLU) and the 2x2 / stride 2 ceil-mode max pool of its fp64 output, on pool rows `rows`"""
    Hc = H + 2 * pad - w.shape[2] + 1
    crow = sorted({c for r in rows for c in (2 * r, 2 * r + 1) if c < Hc})
    y = conv_rows(get, H, w, b, 1, pad, crow)
    if relu:
        y = F.relu(y)
    pos = {c: i for i, c in enumerate(crow)}
    return maxpool_rows(lambda a, z: y[:, :, [pos[c] for c in range(a, z)]], Hc, 2, 2, 0, 1, rows)

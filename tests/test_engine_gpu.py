"""GPU parity: the wgmma bf16x3 conv/GEMM engine vs fp32 PyTorch-CPU math (the oracle for dense layers).
Tolerance: 1e-4 normwise per layer (the engine carries ~16 mantissa bits; the path's bar is 1e-3 end to end)."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from conftest import rel_err, record_parity

pytestmark = pytest.mark.gpu
TOL = 1e-4


def _ref_gemm(A, B, bias, relu):
    y = torch.from_numpy(A).double() @ torch.from_numpy(B).double().t()
    if bias is not None:
        y = y + torch.from_numpy(bias).double()
    return (F.relu(y) if relu else y).float().numpy()


@pytest.mark.parametrize("impl", [1, 0])     # 1 = plain fp32 check kernel first: separates data-prep bugs from engine bugs
@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (128, 128, 128), (128, 256, 192), (1, 64, 64), (100, 21, 256),
                                   (300, 84, 4096), (257, 320, 512), (1000, 4096, 1024), (500, 512, 25088)])
def test_gemm(ctx, impl, M, N, K):
    rng = np.random.default_rng(M + N + K)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    got = ctx.gemm_check(A, B, bias, relu=True, impl=impl)
    assert rel_err(got, _ref_gemm(A, B, bias, True)) < TOL


def test_gemm_row_chunk_invariance(ctx):
    """reference modules/test.lua:85-98 (SequentialSplitBatch_Tensor): chunked rows == unchunked, EXACTLY"""
    rng = np.random.default_rng(3)
    A = rng.standard_normal((40, 512)).astype(np.float32)
    B = (rng.standard_normal((9, 512)) / 22).astype(np.float32)
    b = rng.standard_normal(9).astype(np.float32)
    full = ctx.gemm_check(A, B, b)
    parts = np.concatenate([ctx.gemm_check(A[:25], B, b), ctx.gemm_check(A[25:], B, b)])
    assert np.array_equal(full, parts)


@pytest.mark.parametrize("M,N,K,cuts", [(1000, 4096, 1024, (300,)), (1000, 4096, 1024, (128, 129, 700)), (900, 84, 4096, (77, 500)),
                                        (700, 21, 4096, (1, 699)), (640, 512, 2048, (100, 356))])
def test_gemm_row_chunk_invariance_head_shapes(ctx, M, N, K, cuts):
    """Per-ROI GEMMs at head sizes: the plan may depend on the row count (grid size) but nothing that changes rounding may
    (the N tile and split-K are functions of (N, K) only), so any chunking of the
    rows gives the same bits as the full call (ImageDetect.lua:126-133 forwards ROIs in chunks)."""
    rng = np.random.default_rng(M + N)
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    full = ctx.gemm_check(A, B, b)
    edges = [0, *cuts, M]
    parts = np.concatenate([ctx.gemm_check(A[a:z], B, b) for a, z in zip(edges[:-1], edges[1:])])
    assert np.array_equal(full, parts)


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("N,Cin,H,W,Cout,k,s,p", [
    (1, 64, 16, 16, 64, 3, 1, 1), (1, 64, 37, 53, 128, 3, 1, 1), (1, 128, 75, 100, 256, 3, 1, 1), (1, 512, 38, 50, 512, 3, 1, 1),
    (3, 64, 7, 7, 64, 3, 1, 1), (5, 128, 14, 14, 64, 1, 1, 0), (2, 256, 9, 11, 512, 1, 1, 0), (1, 64, 33, 47, 64, 7, 1, 3),
    (2, 64, 15, 15, 64, 7, 1, 0)])
def test_conv_stride1(ctx, impl, N, Cin, H, W, Cout, k, s, p):
    rng = np.random.default_rng(Cin + H + W + Cout)
    x = rng.standard_normal((N, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    ref = F.relu(F.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), torch.from_numpy(b).double(), stride=s, padding=p)).float().numpy()
    got = ctx.conv_check(x, w, b, stride=s, pad=p, relu=True, impl=impl)
    assert rel_err(got, ref) < TOL


@pytest.mark.parametrize("impl", [1, 0])
@pytest.mark.parametrize("N,Cin,H,W,Cout,k,s,p", [(2, 64, 14, 14, 128, 3, 2, 1), (1, 128, 28, 36, 256, 1, 2, 0), (3, 64, 15, 17, 64, 3, 2, 1)])
def test_conv_stride2(ctx, impl, N, Cin, H, W, Cout, k, s, p):
    """ResNet stride-2 convs: TMA elementStrides"""
    rng = np.random.default_rng(7 + Cin + H)
    x = rng.standard_normal((N, Cin, H, W)).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32)
    ref = F.conv2d(torch.from_numpy(x).double(), torch.from_numpy(w).double(), None, stride=s, padding=p).float().numpy()
    got = ctx.conv_check(x, w, None, stride=s, pad=p, relu=False, impl=impl)
    assert rel_err(got, ref) < TOL


@pytest.mark.parametrize("Cin,Cout,k,s,p,H,W", [(3, 64, 3, 1, 1, 40, 56), (3, 64, 7, 2, 3, 65, 81)])
def test_first_layer_direct_conv(ctx, Cin, Cout, k, s, p, H, W):
    rng = np.random.default_rng(11)
    x = (rng.random((1, Cin, H, W)) * 255 - 110).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k, k)) / 64).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    ref = F.relu(F.conv2d(torch.from_numpy(x), torch.from_numpy(w), torch.from_numpy(b), stride=s, padding=p)).numpy()
    got = ctx.conv_check(x, w, b, stride=s, pad=p, relu=True, impl=2)
    assert rel_err(got, ref) < TOL


# ---- "w16" numerics of fc6 / fc7 (round 2): weight = ONE fp16 plane scaled by a power of two, two products per MAC ------
def _w16_emulation(A, B, bias, relu):
    """what the w16 kernels compute, in fp64: (A_hi + A_lo) @ fp16(B * 2^e)^T / 2^e (+ bias)(ReLU) with A_hi / A_lo the fp16
    planes of A; the only difference left to the GPU is its fp32 accumulation"""
    a = torch.from_numpy(A)
    hi = a.to(torch.float16).float()
    a2 = (hi + (a - hi).to(torch.float16).float()).double()
    amax = float(np.abs(B).max())
    e = 14 - int(np.frexp(amax)[1])
    b16 = (torch.from_numpy(B) * float(2.0 ** e)).to(torch.float16).double() / float(2.0 ** e)
    y = a2 @ b16.t()
    if bias is not None:
        y = y + torch.from_numpy(bias).double()
    return (F.relu(y) if relu else y).float().numpy()


@pytest.mark.parametrize("M,N,K", [(128, 256, 64), (200, 512, 128), (300, 1024, 2048), (100, 1024, 2048), (1000, 4096, 4096), (257, 2000, 2112), (500, 4096, 25088)])
def test_gemm_w16(ctx, M, N, K):
    """the fp16 x fp16 kernels (A as fp16 hi / lo planes, B as one scaled fp16 plane) do what the numerics note says: equal to
    the fp64 emulation of that arithmetic to fp32-accumulation accuracy, and within the weight plane's 2^-12 of the exact
    product. (wgmma wants A and B in one 16-bit format, so the activation planes are fp16 too.)"""
    rng = np.random.default_rng(M + N + K)
    A = np.maximum(rng.standard_normal((M, K)), 0).astype(np.float32)              # post-ReLU activations, like fc6 / fc7 inputs
    B = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    B[0, :8] = [3.0, -2.5, 1e-9, -1e-9, 0.0, 1e-4, -7e-5, 2.0]                      # a wide dynamic range inside one tensor
    bias = rng.standard_normal(N).astype(np.float32)
    got = ctx.gemm_check(A, B, bias, relu=True, impl=2)
    # vs the fp64 emulation of the same operand planes. What is left is the tensor pipe's fp32 accumulation: one rounding
    # TOWARDS ZERO per k16 MMA step (every output below the emulation with these all-positive activations), i.e. a drift of ~2 * K/16 * 2^-25 of the running sum; at K <= 128 (<= 8 steps) it vanishes
    # and the bar pins the operand formats themselves (a bf16 `lo` plane instead of fp16 would already show 1e-5 there)
    tol_acc = 3e-6 if K <= 128 else (3e-5 if K <= 4096 else 2e-4)
    e_emu, e_ref = rel_err(got, _w16_emulation(A, B, bias, True)), rel_err(got, _ref_gemm(A, B, bias, True))
    record_parity("gemm_w16", M=M, N=N, K=K, vs_emulation=e_emu, vs_fp64=e_ref)
    assert e_emu < tol_acc
    assert e_ref < 3e-4


def test_gemm_w16_row_chunk_invariance(ctx):
    """chunked rows == unchunked, bit for bit, whatever the grid size (ImageDetect.lua:126-133)"""
    rng = np.random.default_rng(5)
    M, N, K = 1000, 4096, 2048
    A = rng.standard_normal((M, K)).astype(np.float32)
    B = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    full = ctx.gemm_check(A, B, b, impl=2)
    edges = [0, 100, 228, 229, 700, M]
    parts = np.concatenate([ctx.gemm_check(A[a:z], B, b, impl=2) for a, z in zip(edges[:-1], edges[1:])])
    assert np.array_equal(full, parts)


def test_w16_activation_overflow_is_loud(ctx):
    """an activation beyond fp16's range saturates and the call FAILS (no silent garbage): the flag is raised by the plane
    conversion, tested at the synchronising entry point, and re-armed"""
    import multipathnet_b200 as mpn
    rng = np.random.default_rng(9)
    A = rng.standard_normal((64, 2048)).astype(np.float32); A[3, 7] = 1.0e5
    B = (rng.standard_normal((1024, 2048)) / 45).astype(np.float32)
    ctx.gemm_check(A, B, None, impl=2)                 # the check entry itself does not test the flag...
    with pytest.raises(mpn.MpnError, match="fp16"):
        ctx.synchronize()                              # ...the next synchronising call does
    ctx.synchronize()                                  # re-armed
    A[3, 7] = 1.0
    ctx.gemm_check(A, B, None, impl=2); ctx.synchronize()

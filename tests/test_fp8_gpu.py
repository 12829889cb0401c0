"""The opt-in fp8 inference numerics (mpn_ctx_set_option "fp8" = 1): every layer on the wgmma engine except the cls / bbox
heads runs its FP8X1 kernels, one e4m3 product per MAC, on e4m3 planes of the hi planes scaled by a power of two per
sample (activations) and per output channel (weights); the rule is csrc/fp8_e4m3.cuh, restated in tests/_fp8_oracle.py.

Bars:
  * engine: impl 1 (the fp32 check kernel reading the same e4m3 planes and exponents) within 1e-5 normwise of an fp64
    product of the same scaled e4m3 operands; impl 0 (wgmma) within 1e-4 of it and of impl 1. The tensor pipe's e4m3
    product keeps fewer bits than fp32 even inside one k32 instruction: measured on an H100, 3-7e-5 with the engine's
    promotion of every k32 product into fp32 registers (1.5e-4 when two k32 steps share a fragment), independent of K up
    to 25088, so the bf16 mode's 1e-5 is out of reach of any e4m3 wgmma. Conv outputs are stored as split planes
    (+ 2^-17, as in the bf16 mode);
  * the quantizer: bit-exact against the host rule (read back through an identity weight, which makes the engine's
    output exactly the dequantized operand); a non-finite input fails the call;
  * per-ROI Linears: chunked rows == the full call, two runs and fc_w16 0 / 1 bit-exact;
  * whole graphs: scores and boxes against the fp8-operand oracle within max(1e-3, 3 x the oracle's own sensitivity),
    the larger of its fp32-vs-fp64 order sensitivity and its distance to itself with noise of the engine's precision
    (1e-5 x max|sum|, tests/_fp8_oracle.py) in every fp8 layer's sum; the distance to the plain fp32 oracle recorded and
    checked against max(5e-2, 3 x the fp8 oracle's own distance to it);
  * NMS keep lists bit-exact vs nms.c on the device's own outputs; the pooled tensor as in the default mode.
Every test sets the option in try / finally and restores -1, so the rest of the suite sees the default numerics."""
import contextlib

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from oracle import graphs as G, ref as O
from conftest import rel_err, record_parity
from test_model_gpu import _inputs, assert_nms_every_class
from test_roi_product_gpu import check_tower, run_detect
import _fp8_oracle as F8

pytestmark = pytest.mark.gpu
TOL_ENGINE = 1e-5           # the fp32 check kernel
TOL_WGMMA = 1e-4            # the e4m3 wgmma (docstring)
TOL = 1e-3
SANITY = 5e-2


@contextlib.contextmanager
def option(ctx, name, value):
    ctx.set_option(name, value)
    try:
        yield
    finally:
        ctx.set_option(name, -1)


def _deq(a):
    """the fp8 operand of a (groups along dim 0) as fp64 values q * 2^-e"""
    q, e = F8.quantize(torch.from_numpy(np.ascontiguousarray(a, np.float32)))
    return q.double() * torch.ldexp(torch.ones(1, dtype=torch.float64), -e.double()).reshape(-1, *([1] * (q.dim() - 1)))


# ---------------------------------------------------------------- 1. engine
@pytest.mark.parametrize("M,N,K", [(128, 64, 64), (128, 128, 128), (128, 256, 192), (1, 64, 64), (100, 21, 256),
                                   (300, 84, 4096), (257, 320, 512), (1000, 4096, 1024), (500, 512, 25088)])
def test_gemm_fp8(ctx, M, N, K):
    rng = np.random.default_rng(M + N + K)
    A = rng.standard_normal((M, K)).astype(np.float32)
    Bm = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    bias = rng.standard_normal(N).astype(np.float32)
    with option(ctx, "fp8", 1):
        got0 = ctx.gemm_check(A, Bm, bias, relu=True, impl=0)
        got1 = ctx.gemm_check(A, Bm, bias, relu=True, impl=1)
    ref = torch.relu(_deq(A) @ _deq(Bm).t() + torch.from_numpy(bias).double()).numpy()
    e01, e0, e1 = rel_err(got0, got1), rel_err(got0, ref), rel_err(got1, ref)
    record_parity("gemm_fp8", M=M, N=N, K=K, engine_vs_check=e01, engine_vs_fp64=e0, check_vs_fp64=e1)
    assert e01 <= TOL_WGMMA and e0 <= TOL_WGMMA and e1 <= TOL_ENGINE, (e01, e0, e1)
    assert not np.array_equal(got0, ctx.gemm_check(A, Bm, bias, relu=True, impl=0))     # the option is really off again


@pytest.mark.parametrize("N,Cin,H,W,Cout,k,s,p", [
    (1, 64, 16, 16, 64, 3, 1, 1), (1, 64, 37, 53, 128, 3, 1, 1), (1, 128, 75, 100, 256, 3, 1, 1), (1, 512, 38, 50, 512, 3, 1, 1),
    (3, 64, 7, 7, 64, 3, 1, 1), (5, 128, 14, 14, 64, 1, 1, 0), (2, 256, 9, 11, 512, 1, 1, 0), (1, 64, 33, 47, 64, 7, 1, 3),
    (2, 64, 15, 15, 64, 7, 1, 0), (2, 64, 14, 14, 128, 3, 2, 1), (1, 128, 28, 36, 256, 1, 2, 0), (3, 64, 15, 17, 64, 3, 2, 1),
    (4, 1024, 14, 14, 256, 1, 1, 0), (4, 256, 14, 14, 256, 3, 2, 1)])
def test_conv_fp8(ctx, N, Cin, H, W, Cout, k, s, p):
    """Cin = 64 (64-byte rows), stride 1 (16 x 8 patches for 3x3, flat 1x1, generic 7x7) and stride 2, several samples
    (one exponent each: the per-ROI layer4 shapes at the end); the output is stored as split planes"""
    rng = np.random.default_rng(Cin + H + W + Cout + s)
    x = (rng.standard_normal((N, Cin, H, W)) * np.exp(rng.uniform(-3, 3, (N, 1, 1, 1)))).astype(np.float32)
    w = (rng.standard_normal((Cout, Cin, k, k)) / np.sqrt(Cin * k * k)).astype(np.float32)
    b = rng.standard_normal(Cout).astype(np.float32)
    with option(ctx, "fp8", 1):
        got0 = ctx.conv_check(x, w, b, stride=s, pad=p, relu=True, impl=0)
        got1 = ctx.conv_check(x, w, b, stride=s, pad=p, relu=True, impl=1)
    ref = torch.relu(torch.nn.functional.conv2d(_deq(x), _deq(w), torch.from_numpy(b).double(), stride=s, padding=p)).numpy()
    e01, e0, e1 = rel_err(got0, got1), rel_err(got0, ref), rel_err(got1, ref)
    record_parity("conv_fp8", shape=[N, Cin, H, W, Cout, k, s, p], engine_vs_check=e01, engine_vs_fp64=e0, check_vs_fp64=e1)
    assert e0 <= TOL_WGMMA and e1 <= TOL_ENGINE and e01 <= TOL_WGMMA + 2.0 ** -17, (e01, e0, e1)


# ---------------------------------------------------------------- 2. the quantizer
def test_quantizer_bit_exact(ctx):
    """A @ I: the weight rows are one-hot, so e_w = 8 and q_w = 256 exactly, and the output is q_a * 2^-e_a, the
    dequantized operand, exactly (one exact product per output). Rows = samples: spread scales, an all-zero row, a row
    with a huge outlier whose other values fall to subnormals and zeros, a row at the clamp."""
    rng = np.random.default_rng(1)
    K = 256
    A = (rng.standard_normal((40, K)) * np.exp(rng.uniform(-25, 25, (40, 1)))).astype(np.float32)
    A[3] = 0.0
    A[5, 7] = 3e8
    A[6] = A[6] * np.float32(1e-30)                      # e would be above 60: clamped
    eye = np.eye(K, dtype=np.float32)
    want = _deq(A).float().numpy()
    with option(ctx, "fp8", 1):
        for impl in (0, 1):
            got = ctx.gemm_check(A, eye, None, relu=False, impl=impl)
            assert np.array_equal(got, want), (impl, np.argwhere(got != want)[:8])


def test_quantizer_non_finite_fails(ctx):
    A = np.ones((8, 64), np.float32)
    A[3, 5] = np.inf
    Bm = np.ones((64, 64), np.float32)
    with option(ctx, "fp8", 1):
        with pytest.raises(mpn.MpnError):
            ctx.gemm_check(A, Bm, None, impl=0)
        A[3, 5] = np.nan
        with pytest.raises(mpn.MpnError):
            ctx.gemm_check(A, Bm, None, impl=0)
        ctx.gemm_check(np.ones((8, 64), np.float32), Bm, None, impl=0)          # the flag is re-armed


# ---------------------------------------------------------------- 3. row-chunk invariance
@pytest.mark.parametrize("M,N,K,cuts", [(1000, 4096, 1024, (300,)), (1000, 4096, 1024, (128, 129, 700)), (900, 84, 4096, (77, 500)),
                                        (700, 21, 4096, (1, 699)), (640, 512, 25088, (100, 356))])
def test_gemm_fp8_row_chunk_invariance(ctx, M, N, K, cuts):
    rng = np.random.default_rng(M + N)
    A = (rng.standard_normal((M, K)) * np.exp(rng.uniform(-4, 4, (M, 1)))).astype(np.float32)
    Bm = (rng.standard_normal((N, K)) / np.sqrt(K)).astype(np.float32)
    b = rng.standard_normal(N).astype(np.float32)
    edges = [0, *cuts, M]
    with option(ctx, "fp8", 1):
        full = ctx.gemm_check(A, Bm, b)
        parts = np.concatenate([ctx.gemm_check(A[a:z], Bm, b) for a, z in zip(edges[:-1], edges[1:])])
    assert np.array_equal(full, parts)


# ---------------------------------------------------------------- 4. whole graphs (+ NMS)
def _graph_check(name, got, spec, img, boxes, W, H):
    (s, b) = got
    rs, rb = F8.test_one(spec, img, boxes, 1.0, W, H)
    os_, ob = F8.test_one(spec, img, boxes, 1.0, W, H, fp64_sums=True)
    ns, nb = F8.test_one(spec, img, boxes, 1.0, W, H, sum_noise=1e-5)
    fs, fb = G.test_one(spec, img, boxes, 1.0, W, H, nms_fn=lambda sb, thr: np.zeros(0, np.int64))[:2]
    e = dict(scores=rel_err(s, rs), boxes=rel_err(b, rb), order_scores=rel_err(os_, rs), order_boxes=rel_err(ob, rb),
             scores_vs_fp32=rel_err(s, fs), boxes_vs_fp32=rel_err(b, fb), oracle_scores_vs_fp32=rel_err(rs, fs),
             oracle_boxes_vs_fp32=rel_err(rb, fb), noise_scores=rel_err(ns, rs), noise_boxes=rel_err(nb, rb))
    record_parity(name, **e)
    print(name, e)
    sens_s, sens_b = max(e["order_scores"], e["noise_scores"]), max(e["order_boxes"], e["noise_boxes"])
    assert e["scores"] < max(TOL, 3 * sens_s) and e["boxes"] < max(TOL, 3 * sens_b), e
    assert e["scores_vs_fp32"] < max(SANITY, 3 * e["oracle_scores_vs_fp32"]), e
    assert e["boxes_vs_fp32"] < max(SANITY, 3 * e["oracle_boxes_vs_fp32"]), e


@pytest.mark.parametrize("graph", ["vgg", "multipathnet", "resnet_integral"])
def test_small_graphs_fp8(ctx, graph):
    if graph == "vgg":
        spec = models.vgg16_fast_rcnn(21, seed=7, width_div=4, fc_dim=256)
        H, W, R, seed, sharp = 150, 203, 200, 2, False
    elif graph == "multipathnet":
        spec = models.vgg16_multipathnet(21, seed=11, width_div=4, fc_dim=256)
        H, W, R, seed, sharp = 160, 208, 128, 6, True
    else:
        spec = models.resnet50_fast_rcnn(21, seed=5, integral_k=3)
        H, W, R, seed, sharp = 160, 224, 48, 8, True
    img, boxes = _inputs(spec, H, W, R, seed, sharp=sharp)
    with option(ctx, "fp8", 1):
        m = mpn.Model(ctx, spec, max_rois=256, max_h=256, max_w=320)
        try:
            got = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        finally:
            m.close()
    scores, bboxes, keeps = got
    _graph_check(f"fp8_small_{graph}", (scores, bboxes), spec, img, boxes, W, H)
    assert_nms_every_class(scores, bboxes, keeps)


@pytest.mark.parametrize("cfg", [2, 3, 4])
def test_full_size_fp8(ctx, cfg):
    """cfg 2: VGG-16 Fast R-CNN 600x800, R = 1000, C = 21; cfg 3: MultiPathNet (5 towers) 600x800, R = 1000, C = 81;
    cfg 4: ResNet-50 integral K = 6, 800x1000, R = 2000, C = 81"""
    if cfg == 2:
        spec = models.vgg16_fast_rcnn(21, seed=1234)
        H, W, R, seed, sharp, mh = 600, 800, 1000, 2, False, 608
    elif cfg == 3:
        spec = models.vgg16_multipathnet(81, seed=1234)
        H, W, R, seed, sharp, mh = 600, 800, 1000, 3, True, 608
    else:
        spec = models.resnet50_fast_rcnn(81, seed=1234, integral_k=6)
        H, W, R, seed, sharp, mh = 800, 1000, 2000, 4, True, 808
    img, boxes = _inputs(spec, H, W, R, seed, sharp=sharp)
    with option(ctx, "fp8", 1):
        m = mpn.Model(ctx, spec, max_rois=R + 48, max_h=mh, max_w=W)
        try:
            scores, bboxes, keeps = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        finally:
            m.close()
    assert_nms_every_class(scores, bboxes, keeps)
    _graph_check(f"fp8_full_size_cfg{cfg}", (scores, bboxes), spec, img, boxes, W, H)


# ---------------------------------------------------------------- 5. pooled tensor
@pytest.mark.parametrize("graph", ["multipathnet_small", "cfg2"])
def test_pooled_tensor_fp8(ctx, graph):
    """the product ROI kernel under the fp8 numerics: the towers read trunk slots written by FP8X1 convs (stored as
    split-bf16 planes as always), and the pooled tensor equals the module op on the read-back slots"""
    if graph == "cfg2":
        spec = models.vgg16_fast_rcnn(21, seed=1234)
        H, W, R, seed, sharp, mr, mh, mw = 600, 800, 1000, 2, False, 1024, 608, 800
    else:
        spec = models.vgg16_multipathnet(21, seed=11, width_div=4, fc_dim=256)
        H, W, R, seed, sharp, mr, mh, mw = 160, 208, 128, 6, True, 256, 256, 320
    with option(ctx, "fp8", 1):
        m = mpn.Model(ctx, spec, max_rois=mr, max_h=mh, max_w=mw)
        try:
            rois = run_detect(m, spec, H, W, R, seed, sharp)
            for t in range(len(spec.towers)):
                check_tower(spec, m, rois, t, slice(0, R))
        finally:
            m.close()


# ---------------------------------------------------------------- 6. the switch
def test_switch(ctx):
    spec = models.vgg16_fast_rcnn(21, seed=7, width_div=4, fc_dim=256)
    H, W = 150, 203
    img, boxes = _inputs(spec, H, W, 300, 3)
    rois = O.project_rois(boxes, 1.0)

    def run():
        m = mpn.Model(ctx, spec, max_rois=512, max_h=256, max_w=320)
        try:
            return m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        finally:
            m.close()

    def same(a, b):
        return np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and all(np.array_equal(x, y) for x, y in zip(a[2], b[2]))

    before = run()                                                   # default numerics (the suite resets the option)
    with option(ctx, "fp8", 1):
        on = run()
        on2 = run()
        with option(ctx, "fc_w16", 1):
            w16_on = run()
        with option(ctx, "fc_w16", 0):
            w16_off = run()
        m = mpn.Model(ctx, spec, max_rois=512, max_h=256, max_w=320)
        try:
            m.trunk(img)
            cf, bf = m.heads(rois)
            c1, b1 = m.heads(rois[:130]); c2, b2 = m.heads(rois[130:])
        finally:
            m.close()
        with option(ctx, "bf16", 1):                                 # both on: the plan fails
            m = mpn.Model(ctx, spec, max_rois=512, max_h=256, max_w=320)
            try:
                with pytest.raises(mpn.MpnError):
                    m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
            finally:
                m.close()
            with pytest.raises(mpn.MpnError):
                ctx.gemm_check(np.ones((4, 64), np.float32), np.ones((8, 64), np.float32), None)
    ctx.set_option("fp8", 0)                                         # 0 means the default too
    after0 = run()
    after = run()
    assert not np.array_equal(on[0], before[0])                      # the option changes the numerics
    assert same(on, on2)                                             # fp8 runs are deterministic
    assert same(w16_on, on) and same(w16_off, on)                    # fc_w16 is ignored under fp8
    assert np.array_equal(np.concatenate([c1, c2]), cf) and np.array_equal(np.concatenate([b1, b2]), bf)
    assert same(after, before) and same(after0, before)              # reset: bit-identical to never having set it
    with pytest.raises(mpn.MpnError):
        ctx.set_option("fp9", 1)


def test_model_built_without_the_option_switches(ctx):
    """weights prepared in the default numerics (fp32 copy freed) re-plan into fp8 from their hi planes"""
    spec = models.vgg16_fast_rcnn(21, seed=7, width_div=4, fc_dim=256)
    H, W = 150, 203
    img, boxes = _inputs(spec, H, W, 200, 2)
    img2, boxes2 = np.ascontiguousarray(img[:, :H - 16, :W - 16]), np.ascontiguousarray(boxes[:150])
    m = mpn.Model(ctx, spec, max_rois=512, max_h=256, max_w=320)
    try:
        with option(ctx, "fc_w16", 0):
            m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
            with option(ctx, "fp8", 1):          # a new image size and ROI count: trunk and heads plan again
                got = m.detect_nms(img2, boxes2, 1.0, W - 16, H - 16, -1.5, 0.3)
    finally:
        m.close()
    with option(ctx, "fp8", 1):
        m = mpn.Model(ctx, spec, max_rois=512, max_h=256, max_w=320)
        try:
            want = m.detect_nms(img2, boxes2, 1.0, W - 16, H - 16, -1.5, 0.3)
        finally:
            m.close()
    assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])

"""Plain references of the detect tail after the network (ImageDetect.lua:183-191, Tester_FRCNN.lua:75-78,106-117): the
softmax / integral mean in fp64, BBoxNorm + convertFrom + clamp restated in fp32 op for op, the per-class gather and
nms.c (through oracle.ref.nms) on the gathered rows. Used by tests/test_detect_tail_{cpu,gpu}.py.

Bars (asserted by the GPU tests, derived here):
  softmax  |got - ref| <= 1e-6 ref + 2^-126 + 2^-24 mean_k(p_k |x_k - m_k|) elementwise. The last term is the fp32
           rounding of the shifted logit x - m that every fp32 softmax (nn.SoftMax included) performs before exp: its
           absolute error is at most 2^-24 |x - m|, which exp turns into a relative error of the same size; the fp64
           reference takes the exact difference. It matters only for the small probabilities of rows whose logits
           spread over more than 16 (randn * 3 at C = 201 reaches |x - m| ~ 18: up to 1.1e-6 relative; an H100 run
           measured 1.3e-6 relative at C = 81, 0.66 of this bar: profiles/h100_detect_tail.json).
  row sum  |sum_c p_c - 1| <= (C + K - 1) 2^-23: C - 1 roundings of the sum of exps and one of each quotient, each at
           most 2^-24 relative, and the K - 1 additions of the integral mean (K = 1: C 2^-23).
  decode   bit-exact where exp is exact (y.z = y.w = 0 after BBoxNorm); elsewhere |got - ref| <= 2^-21 |wt| (x) or
           2^-21 |ht| (y) + 1 ulp of ref: CUDA's expf is within 2 ulp, the restatement's exp within 1/2 ulp, the product
           with w / h adds one rounding each, hw = wt / 2 halves it, and the final add / sub rounds once more. The clamp
           is 1-Lipschitz and keeps the bound."""
import numpy as np

from oracle import ref as O

F32 = np.float32
TINY = 2.0 ** -126


# ---- class values: softmax of each head, mean over the K heads (model_utils.lua:296-313) ----------------------------
def softmax_mean(logits):
    """K x R x C fp32 logits -> fp64 R x C: the mean over K of the fp64 softmax of each head"""
    x = np.asarray(logits, np.float64)
    if x.ndim == 2:
        x = x[None]
    m = x.max(axis=2, keepdims=True)
    e = np.exp(x - m)
    return (e / e.sum(axis=2, keepdims=True)).mean(axis=0)


def softmax_bar(logits):
    """the elementwise bar of a device softmax / integral mean of these logits (module docstring)"""
    x = np.asarray(logits, np.float64)
    if x.ndim == 2:
        x = x[None]
    m = x.max(axis=2, keepdims=True)
    e = np.exp(x - m)
    p = e / e.sum(axis=2, keepdims=True)
    shift = np.where(p > 0, p * np.abs(x - m), 0.0).mean(axis=0)
    return 1e-6 * p.mean(axis=0) + TINY + 2.0 ** -24 * shift


def row_sum_bar(C, K):
    return (C + K - 1) * 2.0 ** -23


# ---- nn.BBoxNorm + utils.convertFrom per class block + clamp (bbox_decode_body, orc_convert_from) ---------------------
def exp32(y):
    """exp correctly rounded to fp32 (through fp64)"""
    with np.errstate(over="ignore"):
        return np.exp(np.asarray(y, np.float64)).astype(F32)


def decode(deltas, boxes, do_clamp=False, W0=0.0, H0=0.0, mean=None, std=None):
    """deltas R x 4C, boxes R x 4 -> (bboxes R x 4C, wt R x C, ht R x C), every step one fp32 rounding in the device's
    order: BBoxNorm y * std + mean (no FMA), xc = (x1 + x2) * 0.5, w = x2 - x1, xtc = xc + y.x * w, wt = exp(y.z) * w,
    hw = wt * 0.5, out = xtc -/+ hw; then x clamped to [1, W0], y to [1, H0]"""
    R = boxes.shape[0]
    y = np.asarray(deltas, F32).reshape(R, -1, 4)
    b = np.asarray(boxes, F32).reshape(R, 1, 4)
    with np.errstate(over="ignore", invalid="ignore"):
        if mean is not None:
            y = y * np.asarray(std, F32).reshape(4) + np.asarray(mean, F32).reshape(4)      # two fp32 roundings
        half = F32(0.5)
        xc, yc = (b[..., 0] + b[..., 2]) * half, (b[..., 1] + b[..., 3]) * half
        w, h = b[..., 2] - b[..., 0], b[..., 3] - b[..., 1]
        xtc, ytc = xc + y[..., 0] * w, yc + y[..., 1] * h
        wt, ht = exp32(y[..., 2]) * w, exp32(y[..., 3]) * h
        hw, hh = wt * half, ht * half
        out = np.stack([xtc - hw, ytc - hh, xtc + hw, ytc + hh], axis=-1).astype(F32)
    if do_clamp:
        lim = np.array([W0, H0, W0, H0], F32)
        out = np.where(out < F32(1), F32(1), np.where(out > lim, lim, out)).astype(F32)
    return out.reshape(R, -1), wt, ht


def decode_ratio(got, ref, wt, ht):
    """over the finite reference entries: the largest |got - ref| / bar (<= 1: inside the decode bar; NaN if the device
    gave NaN there) and the largest |got - ref| in ulps of ref"""
    R = ref.shape[0]
    g, r = got.reshape(R, -1, 4).astype(np.float64), ref.reshape(R, -1, 4).astype(np.float64)
    scale = np.stack([np.abs(wt), np.abs(ht), np.abs(wt), np.abs(ht)], axis=-1).astype(np.float64)
    ulp = np.spacing(np.abs(ref.reshape(R, -1, 4))).astype(np.float64)
    fin = np.isfinite(r)
    if not fin.any():
        return 0.0, 0.0
    err = np.abs(g[fin] - r[fin])
    bar = 2.0 ** -21 * np.where(np.isfinite(scale), scale, 0.0)[fin] + ulp[fin]
    return float(np.max(err / bar)), float(np.max(err / ulp[fin]))


def same_nonfinite(got, ref):
    """NaN where the reference is NaN, the same infinity where it is infinite"""
    nan_ok = np.array_equal(np.isnan(got), np.isnan(ref))
    inf = np.isinf(ref)
    return nan_ok and np.array_equal(np.isinf(got), inf) and np.array_equal(got[inf], ref[inf])


# ---- Tester_FRCNN.lua:106-117: gather + NMS per foreground class ----------------------------------------------------
def gather(scores, j, thresh):
    """rows with scores[:, j] > thresh (strict, fp32), in row order"""
    return np.nonzero(np.asarray(scores, F32)[:, j] > F32(thresh))[0].astype(np.int32)


def class_keeps(scores, bboxes, thresh, nms_thr, c_begin, c_end):
    """for every class j in [c_begin, c_end): the proposal rows nms.c keeps of the gathered [box, score] rows, in emission
    order (oracle.ref.nms on the gathered rows, mapped back through the gather)"""
    s, bb = np.asarray(scores, F32), np.asarray(bboxes, F32)
    out = []
    for j in range(c_begin, c_end):
        idx = gather(s, j, thresh)
        sb = np.concatenate([bb[idx, 4 * j:4 * j + 4], s[idx, j:j + 1]], 1).astype(F32)
        out.append(idx[O.nms(sb, nms_thr)] if len(idx) else idx)
    return out


def rank_ranges(n_classes, world):
    """the per-rank foreground class ranges [c0, c1) of bench.py's NMS sweep: c0 = 1 + n * rank // world"""
    return [(1 + (n_classes * r) // world, 1 + (n_classes * (r + 1)) // world) for r in range(world)]

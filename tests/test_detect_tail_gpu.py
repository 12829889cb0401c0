"""GPU parity of the detect tail after the network against tests/_detect_tail_ref.py (bars derived there):
(a) detect_tail_kernel (softmax / integral mean | BBoxNorm + decode + clamp, one grid split in two) through
    mpn_debug_detect_tail, at class counts around the 32-wide softmax chunks and row counts that split the grid unevenly;
(b) mpn_post_detect_dev, the class-range tail of the NMS sweep (BBoxNorm + decode + clamp, gather of a class range, NMS),
    on torch device buffers as bench.py calls it: keep lists bit-exact against nms.c on the device's own boxes, and the
    full class range equal to every per-rank split;
(c) mpn_pack_detections_dev on (b)'s outputs == utils.keep_top_k;
(d) the integral mean of softmaxes on the product path (detect of K = 2 / 3 head models);
(e) the other device forms of the ABI: mpn_nms_batched_dev, mpn_select_boxes_dev, mpn_get_images*_dev."""
import ctypes as C

import numpy as np
import pytest
import torch

import multipathnet_b200 as mpn
from multipathnet_b200 import dist as mdist, models, utils as U, workloads as wl
from multipathnet_b200._lib import CImageTransform, _ptr
from oracle import ref as O

import _detect_tail_ref as T
from conftest import record_parity

pytestmark = pytest.mark.gpu
F32 = np.float32
FLT_MAX = np.finfo(np.float32).max
MEAN, STD = F32([0.03, -0.02, 0.0, 0.0]), F32([0.1, 0.1, 0.2, 0.2])      # mean[2:4] = 0: y.z = y.w = 0 stays exact


def debug_tail(ctx, logits, deltas, boxes, do_softmax=1, do_clamp=0, W0=0.0, H0=0.0, norm=False):
    x, d, b = (np.ascontiguousarray(a, F32) for a in (logits, deltas, boxes))
    K, R, Cc = x.shape
    scores, bboxes = np.empty((R, Cc), F32), np.empty((R, 4 * Cc), F32)
    ctx.check(ctx.lib.mpn_debug_detect_tail(ctx.h, _ptr(x), K, R, Cc, int(do_softmax), _ptr(d), _ptr(b), int(do_clamp), float(W0), float(H0),
                                            int(norm), _ptr(MEAN) if norm else None, _ptr(STD) if norm else None, _ptr(scores),
                                            _ptr(bboxes)), "mpn_debug_detect_tail")
    return scores, bboxes


def make_logits(K, R, Cc, seed):
    """randn * 3, with every fifth row scaled to +-1e4 (probabilities exactly 1 and 0), all equal (1 / C) or holding
    -FLT_MAX in every third class"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((K, R, Cc)) * 3
    r = np.arange(R)
    big = r % 5 == 1
    x[:, big] *= 1e4 / np.abs(x[:, big]).max(axis=2, keepdims=True)
    x[:, r % 5 == 2] = 0.75
    x[:, (r % 5 == 3)[:, None] & (np.arange(Cc) % 3 == 1)[None, :]] = -FLT_MAX
    return x.astype(F32)


def make_deltas(R, Cc, seed):
    """randn * 0.5, every fourth row with y.z = y.w = 0 (exp exact)"""
    rng = np.random.default_rng(seed)
    d = (rng.standard_normal((R, Cc, 4)) * 0.5).astype(F32)
    d[::4, :, 2:] = 0
    return d.reshape(R, 4 * Cc)


# ---- (a) detect_tail_kernel --------------------------------------------------------------------------------------------
@pytest.mark.parametrize("R", [1, 7, 9, 1000, 5000])
@pytest.mark.parametrize("K", [1, 2, 3, 6])
@pytest.mark.parametrize("Cc", [2, 21, 31, 32, 33, 81, 201])
def test_detect_tail_kernel(ctx, Cc, K, R):
    seed = 1000 * Cc + 10 * K + R
    norm, clamp = seed % 2 == 1, (seed // 2) % 2 == 1
    H0, W0 = 480.0, 640.0
    x, d = make_logits(K, R, Cc, seed), make_deltas(R, Cc, seed + 1)
    boxes = wl.random_boxes(R, 400, 700, seed).astype(F32)
    boxes[::6] -= F32(60)                                                   # partly outside the image: the clamp bites
    scores, bboxes = debug_tail(ctx, x, d, boxes, 1, clamp, W0, H0, norm)
    # softmax / integral mean
    ref = T.softmax_mean(x)
    err = np.abs(scores.astype(np.float64) - ref)
    bar = T.softmax_bar(x)
    assert np.all(err <= bar), f"softmax: worst {float(np.max(err / bar)):.3g} of the bar"
    sums = np.abs(scores.astype(np.float64).sum(1) - 1.0)
    assert sums.max() <= T.row_sum_bar(Cc, K)
    if Cc in (2, 32):                                                       # equal logits: 1 / C, exact for powers of two
        assert np.all(scores[np.arange(R) % 5 == 2] == F32(1.0 / Cc))
    # decode
    want, wt, ht = T.decode(d, boxes, clamp, W0, H0, MEAN if norm else None, STD if norm else None)
    exact = np.arange(R) % 4 == 0
    assert np.array_equal(bboxes[exact], want[exact])
    dec, ulps = T.decode_ratio(bboxes, want, wt, ht)
    assert dec <= 1 and T.same_nonfinite(bboxes, want)
    record_parity("detect_tail_kernel", C=Cc, K=K, R=R, norm=int(norm), clamp=int(clamp),
                  softmax_of_bar=float(np.max(err / bar)), softmax_rel_max=float(np.max(err / (ref + T.TINY))),
                  row_sum_of_bar=float(sums.max() / T.row_sum_bar(Cc, K)), decode_of_bar=dec, decode_ulps=ulps)


@pytest.mark.parametrize("Cc,R", [(2, 9), (33, 1000), (201, 7)])
def test_detect_tail_no_softmax_copies_head_zero(ctx, Cc, R):
    x = make_logits(1, R, Cc, Cc + R)
    x[0, ::2] = np.abs(x[0, ::2]) / 1e4                                      # probabilities already
    scores, _ = debug_tail(ctx, x, make_deltas(R, Cc, 1), wl.random_boxes(R, 100, 100, 1))
    assert not np.array_equal(scores, x[0])
    scores, _ = debug_tail(ctx, x, make_deltas(R, Cc, 1), wl.random_boxes(R, 100, 100, 1), do_softmax=0)
    assert np.array_equal(scores.view(np.uint32), x[0].view(np.uint32))
    with pytest.raises(mpn.MpnError):
        debug_tail(ctx, np.stack([x[0], x[0]]), make_deltas(R, Cc, 1), wl.random_boxes(R, 100, 100, 1), do_softmax=0)


@pytest.mark.parametrize("norm", [False, True])
def test_detect_tail_clamp_and_overflow_edges(ctx, norm):
    """coordinates exactly at 1 and W0 / H0 and beyond them, exp overflowing to inf (y.z >= 89) and underflowing to 0:
    the device equals the restatement bit for bit, NaN (w = 0 times inf) in the same places"""
    W0, H0 = 640.0, 480.0
    boxes = F32([[1, 1, W0, H0], [-50, -20, W0 + 30, H0 + 10], [10, 10, 10, 50], [10, 10, 60, 10], [100, 100, 300, 200],
                 [1, 1, 1, 1], [W0, H0, W0 + 5, H0 + 5], [0.5, 0.75, W0 + 0.5, H0 + 0.25], [2, 3, 40, 90]])
    R, Cc = boxes.shape[0], 6
    raw = np.zeros((R, Cc, 4), F32)                                          # class 0: zero deltas
    raw[:, 1, 2:] = (89.0, -200.0)                                           # exp overflows / underflows
    raw[:, 2, 2:] = (100.0, 100.0)
    raw[:, 3, 2:] = (np.inf, -np.inf)
    raw[:, 4, :2] = (1e6, -1e6)                                              # centres far outside the image
    raw[:, 5, 2:] = (-np.inf, 1e4)
    if norm:
        raw[..., 2:] = raw[..., 2:] / STD[2:]                                # the same exp arguments after y * std + mean
    d = raw.reshape(R, 4 * Cc)
    x = make_logits(1, R, Cc, 5)
    for clamp in (0, 1):
        _, got = debug_tail(ctx, x, d, boxes, 1, clamp, W0, H0, norm)
        want, _, _ = T.decode(d, boxes, clamp, W0, H0, MEAN if norm else None, STD if norm else None)
        assert T.same_nonfinite(got, want)
        fin = np.isfinite(want)
        assert np.array_equal(got[fin], want[fin])
        assert np.isnan(want).any()
        if clamp and not norm:
            assert want[0, 0] == 1.0 and want[0, 2] == W0 and want[0, 3] == H0 and (want[1, :4] == (1, 1, W0, H0)).all()


# ---- (b) mpn_post_detect_dev -------------------------------------------------------------------------------------------
NC = 81
H0, W0 = 600.0, 800.0


def post_inputs(R, thresh, seed):
    """bench.py's shapes with crafted classes: 1 empty, 2 every row passes, 3 half the rows exactly at the threshold,
    4 tied scores, 5 duplicate rows (box, deltas and score); the others with per-class pass rates"""
    rng = np.random.default_rng(seed)
    boxes = wl.random_boxes(R, int(H0), int(W0), seed, wmax=0.4 * W0, hmax=0.4 * H0).astype(F32)
    deltas = (rng.standard_normal((R, 4 * NC)) * 0.5).astype(F32)
    deltas.reshape(R, NC, 4)[::4, :, 2:] = 0
    scores = (rng.random((R, NC)) ** rng.uniform(0.3, 4.0, NC)).astype(F32)
    scores[:, 1] = -2.0
    scores[:, 2] = F32(0.9) + F32(0.09) * rng.random(R).astype(F32)
    scores[::2, 3] = F32(thresh)
    scores[1::2, 3] = F32(0.7) + F32(0.2) * rng.random(R // 2).astype(F32)
    scores[:, 4] = np.floor(scores[:, 4] * 16) / 16
    n = 8                                                        # a multiple of 4: the exact rows stay exact
    boxes[n:2 * n] = boxes[2 * n:3 * n]
    deltas[n:2 * n] = deltas[2 * n:3 * n]
    scores[n:2 * n, 5] = scores[2 * n:3 * n, 5]
    return scores, deltas, boxes


class PostDetect:
    def __init__(self, ctx, scores, deltas, boxes, norm):
        self.ctx, self.R = ctx, scores.shape[0]
        self.sc, self.dl, self.bx = (torch.from_numpy(a).cuda() for a in (scores, deltas, boxes))
        self.bb = torch.full((self.R, 4 * NC), float("nan"), dtype=torch.float32, device="cuda")
        self.norm = norm

    def __call__(self, c0, c1, thresh, nms_thr=0.3, mean=MEAN, std=STD):
        n = max(c1 - c0, 1)                                      # refused ranges still get valid buffers
        keep = torch.full((n, self.R), -7, dtype=torch.int32, device="cuda")
        cnt = torch.full((n,), -7, dtype=torch.int32, device="cuda")
        m, s = (mean, std) if self.norm else (None, None)
        self.ctx.check(self.ctx.lib.mpn_post_detect_dev(self.ctx.h, _ptr(self.sc), _ptr(self.dl), _ptr(self.bx), self.R, NC, _ptr(m), _ptr(s),
                                                        W0, H0, float(thresh), float(nms_thr), int(c0), int(c1), _ptr(self.bb), _ptr(keep),
                                                        _ptr(cnt)), "mpn_post_detect_dev")
        torch.cuda.synchronize()
        return keep, cnt

    @staticmethod
    def lists(keep, cnt):
        k, c = keep.cpu().numpy(), cnt.cpu().numpy()
        return [k[s, :c[s]].copy() for s in range(len(c))]


POST_CASES = [(300, "bench", False), (300, "real", True), (4096, "bench", True), (4096, "real", False), (4097, "bench", False),
              (4097, "real", True), (6000, "real", True), (6000, "bench", False), (20000, "real", True), (20000, "bench", False)]


@pytest.mark.parametrize("R,th,norm", POST_CASES)
def test_post_detect_dev(ctx, R, th, norm):
    thresh = -1.5 if th == "bench" else 0.6
    scores, deltas, boxes = post_inputs(R, thresh, R + (th == "real"))
    pd = PostDetect(ctx, scores, deltas, boxes, norm)
    c0, c1 = (1, NC) if R <= 6000 else (1, 9)                   # 20000 rows: NMS scratch nseg * R * R / 8 bytes, 8 classes
    keep, cnt = pd(c0, c1, thresh)
    bb = pd.bb.cpu().numpy()
    # decode: the restatement's bars on every class block, bit-exact where exp is exact
    want, wt, ht = T.decode(deltas, boxes, True, W0, H0, MEAN if norm else None, STD if norm else None)
    assert np.array_equal(bb[::4], want[::4])
    dec, ulps = T.decode_ratio(bb, want, wt, ht)
    assert dec <= 1 and T.same_nonfinite(bb, want)
    # keeps: nms.c on the device's own boxes
    got = PostDetect.lists(keep, cnt)
    ref = T.class_keeps(scores, bb, thresh, 0.3, c0, c1)
    for j, (a, b) in enumerate(zip(got, ref), start=c0):
        assert np.array_equal(a, b), f"class {j}: {len(a)} vs {len(b)} kept"
    n_in = [len(T.gather(scores, j, thresh)) for j in range(c0, c1)]
    assert n_in[0] == 0 and got[0].size == 0 and n_in[1] == R and n_in[2] == R // 2
    if th == "real":
        assert 0 < min(n_in[5:]) and max(n_in[5:]) < R and len(set(n_in[5:])) > 1        # ragged, below cap = R
    # sharding: the bench's per-rank ranges, concatenated, equal the full range; the decode is the same bits every call
    n = c1 - c0
    for world in (2, 3, 4, 7, 8):
        parts = []
        for a, b in T.rank_ranges(n, world):
            parts += PostDetect.lists(*pd(c0 - 1 + a, c0 - 1 + b, thresh))
            assert np.array_equal(pd.bb.cpu().numpy().view(np.uint32), bb.view(np.uint32))
        assert len(parts) == n and all(np.array_equal(x, y) for x, y in zip(parts, got)), world
    record_parity("post_detect_dev", R=R, thresh=thresh, norm=int(norm), classes=n, kept=int(sum(len(k) for k in got)),
                  decode_of_bar=dec, decode_ulps=ulps)
    # (c) the record of the full range == utils.keep_top_k of the host tables
    if (c0, c1) == (1, NC):
        rec_d = torch.zeros(mpn.MPN_REC_FLOATS, dtype=torch.float32, device="cuda")
        ctx.check(ctx.lib.mpn_pack_detections_dev(ctx.h, _ptr(pd.sc), _ptr(pd.bb), R, NC, _ptr(keep), _ptr(cnt), R, 100, _ptr(rec_d)),
                  "mpn_pack_detections_dev")
        rec = rec_d.cpu().numpy()
        tables = [np.concatenate([bb[k, 4 * j:4 * j + 4], scores[k, j:j + 1]], 1).astype(F32) for j, k in enumerate(got, start=1)]
        kept, _ = U.keep_top_k([t.copy() for t in tables], 100)
        dets = mdist.tables_to_dets(kept)
        assert int(rec[0]) == dets.shape[0]
        if dets.shape[0] <= mpn.MPN_MAX_DET:
            assert np.array_equal(mdist.unpack_record(rec), dets)
            assert np.all(rec[1 + 6 * dets.shape[0]:] == 0)
        else:
            assert np.array_equal(rec[1:1 + 6 * mpn.MPN_MAX_DET].reshape(-1, 6), dets[:mpn.MPN_MAX_DET])


def test_post_detect_dev_refusals(ctx):
    scores, deltas, boxes = post_inputs(64, 0.5, 1)
    pd = PostDetect(ctx, scores, deltas, boxes, True)
    for c0, c1 in ((0, 5), (3, 3), (5, 4), (70, NC + 1)):
        with pytest.raises(mpn.MpnError, match="class range"):
            pd(c0, c1, 0.5)
    with pytest.raises(mpn.MpnError, match="go together"):
        pd(1, 5, 0.5, std=None)
    with pytest.raises(mpn.MpnError, match="go together"):
        pd(1, 5, 0.5, mean=None)
    keep, cnt = pd(1, NC, 0.5)                                   # the context still works
    assert int(cnt[0]) == 0


# ---- (d) the integral mean on the product path ---------------------------------------------------------------------
@pytest.mark.parametrize("name", ["mpn_small_integral", "resnet_small"])
def test_integral_scores_are_the_mean_of_softmaxes(ctx, name):
    build, H, W, R, K = {
        "mpn_small_integral": (lambda: models.vgg16_multipathnet(21, seed=11, width_div=4, fc_dim=256, integral_k=2), 160, 208, 128, 2),
        "resnet_small": (lambda: models.resnet50_fast_rcnn(21, seed=5, integral_k=3), 160, 224, 48, 3)}[name]
    spec = build()
    img = wl.transform(wl.raw_image(H, W, 6), spec.transformer)
    boxes = wl.sharpmask_boxes(R, H, W, 6)
    m = mpn.Model(ctx, spec, max_rois=256, max_h=256, max_w=320)
    try:
        scores, bboxes = m.detect(img, boxes, 1.0)
        cls, raw = m.head_outputs()
    finally:
        m.close()
    assert cls.shape == (K, R, spec.num_classes)
    ref = T.softmax_mean(cls)
    err = np.abs(scores.astype(np.float64) - ref)
    bar = T.softmax_bar(cls)
    assert np.all(err <= bar), float(np.max(err / bar))
    assert not np.all(np.abs(scores - T.softmax_mean(cls[:1])) <= bar)                      # the heads differ: the mean matters
    norm = bool(spec.has_bbox_norm)
    want, wt, ht = T.decode(raw, boxes, False, mean=F32(spec.bbox_mean) if norm else None, std=F32(spec.bbox_std) if norm else None)
    dec, ulps = T.decode_ratio(bboxes, want, wt, ht)
    assert dec <= 1
    record_parity("integral_scores", graph=name, K=K, softmax_of_bar=float(np.max(err / bar)), decode_of_bar=dec, decode_ulps=ulps)


# ---- (e) the other device forms ----------------------------------------------------------------------------------------
def nms_batched_dev(ctx, sb, thr):
    nseg, cap = sb.shape[:2]
    offs = (np.arange(nseg + 1) * cap).astype(np.int64)
    sb_d = torch.from_numpy(np.ascontiguousarray(sb, F32)).cuda()
    keep = torch.full((max(nseg * cap, 1),), -7, dtype=torch.int32, device="cuda")
    cnt = torch.full((nseg,), 0x5a5a5a5a, dtype=torch.int32, device="cuda")
    ctx.check(ctx.lib.mpn_nms_batched_dev(ctx.h, _ptr(sb_d), offs.ctypes.data_as(C.POINTER(C.c_int64)), nseg, float(thr), _ptr(keep),
                                          _ptr(cnt)), "mpn_nms_batched_dev")
    k, c = keep.cpu().numpy(), cnt.cpu().numpy()
    return [k[s * cap:s * cap + c[s]].copy() for s in range(nseg)]


@pytest.mark.parametrize("ties", [False, True])
@pytest.mark.parametrize("cap", [1, 63, 64, 65, 1024, 1025, 4096, 4097, 6000])
def test_nms_batched_dev_uniform_segments(ctx, cap, ties):
    sb = wl.nms_sweep_boxes(cap, 3, 7000 + cap, ties=ties)
    if cap >= 8:
        sb[1, cap // 2:cap // 2 + 4] = sb[1, :4]                 # duplicate rows
    got = nms_batched_dev(ctx, sb, 0.3)
    for s in range(3):
        assert np.array_equal(got[s], O.nms(sb[s], 0.3)), s


def test_nms_batched_dev_refusals_and_empty_segments(ctx):
    sb_d = torch.zeros((40, 5), dtype=torch.float32, device="cuda")
    keep = torch.zeros(40, dtype=torch.int32, device="cuda")
    cnt = torch.full((3,), 0x5a5a5a5a, dtype=torch.int32, device="cuda")
    i64 = C.POINTER(C.c_int64)
    for offs in ([0, 10, 30, 40], [0, 10, 20, 40], [5, 15, 25, 35]):
        o = np.int64(offs)
        with pytest.raises(mpn.MpnError, match="uniform"):
            ctx.check(ctx.lib.mpn_nms_batched_dev(ctx.h, _ptr(sb_d), o.ctypes.data_as(i64), 3, 0.3, _ptr(keep), _ptr(cnt)), "nms_batched_dev")
    o = np.zeros(4, np.int64)
    ctx.check(ctx.lib.mpn_nms_batched_dev(ctx.h, _ptr(sb_d), o.ctypes.data_as(i64), 3, 0.3, _ptr(keep), _ptr(cnt)), "nms_batched_dev")
    assert cnt.cpu().numpy().tolist() == [0, 0, 0]


@pytest.mark.parametrize("R,Cc", [(0, 21), (1, 2), (999, 81)])
def test_select_boxes_dev_equals_host(ctx, R, Cc):
    rng = np.random.default_rng(R + Cc)
    classes = rng.random((R, Cc)).astype(F32)
    classes[::5] = np.round(classes[::5], 1)
    ys = rng.standard_normal((R, 4 * Cc)).astype(F32)
    cl_d, ys_d = torch.from_numpy(classes).cuda(), torch.from_numpy(ys).cuda()
    for mean, std in ((None, None), (MEAN, STD)):
        out_d = torch.full((max(R, 1), 4), float("nan"), dtype=torch.float32, device="cuda")
        ctx.check(ctx.lib.mpn_select_boxes_dev(ctx.h, _ptr(cl_d) if R else None, _ptr(ys_d) if R else None, R, Cc, _ptr(mean), _ptr(std),
                                               _ptr(out_d) if R else None), "mpn_select_boxes_dev")
        got = out_d.cpu().numpy()[:R]
        assert np.array_equal(got, ctx.select_boxes(classes, ys, mean, std))
    with pytest.raises(mpn.MpnError, match="go together"):
        ctx.check(ctx.lib.mpn_select_boxes_dev(ctx.h, _ptr(cl_d), _ptr(ys_d), R, Cc, _ptr(MEAN), None, _ptr(out_d)), "mpn_select_boxes_dev")


@pytest.mark.parametrize("kind,H0,W0,scale", [("ross", 97, 131, 150), ("imagenet", 120, 90, 200), ("ross", 64, 64, 64)])
def test_get_images_dev_forms_equal_host_forms(ctx, kind, H0, W0, scale):
    h, w, _ = O.get_images_size(H0, W0, scale, 1000)
    tf = CImageTransform.of(kind)
    lib = ctx.lib
    im = wl.raw_image(H0, W0, H0 + W0)
    u8 = np.random.default_rng(W0).integers(0, 256, (H0, W0, 3), dtype=np.uint8)
    host = np.empty((3, h, w), F32)
    ctx.check(lib.mpn_get_images(ctx.h, _ptr(im), H0, W0, C.addressof(tf), h, w, _ptr(host)), "mpn_get_images")
    im_d, u8_d = torch.from_numpy(im).cuda(), torch.from_numpy(u8).cuda()
    out_d = torch.full((3, h, w), float("nan"), dtype=torch.float32, device="cuda")
    ctx.check(lib.mpn_get_images_dev(ctx.h, _ptr(im_d), H0, W0, C.addressof(tf), h, w, _ptr(out_d)), "mpn_get_images_dev")
    ctx.synchronize()
    assert np.array_equal(out_d.cpu().numpy().view(np.uint32), host.view(np.uint32))
    ctx.check(lib.mpn_get_images_u8(ctx.h, _ptr(u8), H0, W0, C.addressof(tf), h, w, _ptr(host)), "mpn_get_images_u8")
    out_d.fill_(float("nan"))
    ctx.check(lib.mpn_get_images_u8_dev(ctx.h, _ptr(u8_d), H0, W0, C.addressof(tf), h, w, _ptr(out_d)), "mpn_get_images_u8_dev")
    ctx.synchronize()
    assert np.array_equal(out_d.cpu().numpy().view(np.uint32), host.view(np.uint32))
    for flip in (0, 1):
        ctx.check(lib.mpn_get_images_u8_flip(ctx.h, _ptr(u8), H0, W0, C.addressof(tf), h, w, flip, _ptr(host)), "mpn_get_images_u8_flip")
        out_d.fill_(float("nan"))
        ctx.check(lib.mpn_get_images_u8_flip_dev(ctx.h, _ptr(u8_d), H0, W0, C.addressof(tf), h, w, flip, _ptr(out_d)),
                  "mpn_get_images_u8_flip_dev")
        ctx.synchronize()
        assert np.array_equal(out_d.cpu().numpy().view(np.uint32), host.view(np.uint32)), flip
        if flip == 0:
            first = host.copy()
    assert not np.array_equal(first, host)                      # the flip changed the image

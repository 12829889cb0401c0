"""GPU: one live model through a scripted sequence of calls whose image size, ROI count and entry point change from call
to call, as Tester_FRCNN / ImageDetect run a dataset (every COCO image scales to its own H x W and brings its own
proposals). Every call is compared bit for bit with a fresh model of the same spec and numerics that makes only that
call, and in the default numerics also with the fp64 oracle pipeline within 1e-3 normwise, so a fresh model that is
wrong in the same way still fails.

What the sequence crosses (tests/test_shape_sequence_cpu.py checks that it still does when the planner changes):
  * the first call is at the largest size of its descending prefix and at max_rois, on an image scaled up so that every
    buffer holds large non-zero values past any later extent; the prefix then shrinks in H and W (no buffer grows);
  * sizes shrink, grow back past an earlier size, repeat (A, B, A), include a portrait image and odd sizes; the
    pipelined pair's second submission is at the model limits and grows every trunk buffer while the first is in flight;
  * MultiPathNet: the pooled conv3 slot crosses the one-launch max-pyramid limit in both directions, and small images
    follow large ones, so its pyramid has more levels than a fresh model would build (maxima are exact and every pooled
    zero is +0, so the extra levels change no bit);
  * ResNet-50 / NIN: generic-mode patches (tn, th, tw) change between consecutive trunk plans;
  * R takes 1, 63, 64, 65, 129 and max_rois; heads run in chunks with boundaries at 1 and 129;
  * entry points detect_nms, detect(recompute_features=False) right after a call on another size, trunk + chunked
    heads, test_one (num_iter 2, rbox scores, voting), trunk_image, and detect_nms_submit / _submit_u8 / _wait."""
import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200.image_detect import _get_images_size
from oracle import graphs as G, ref as O
from conftest import rel_err, record_parity
from test_model_gpu import assert_nms_every_class
from test_layers_gpu import NUMERICS, options

pytestmark = pytest.mark.gpu
TOL = 1e-3
MAX_ROIS, MAX_H, MAX_W = 512, 320, 416

# one call per entry: (kind, H, W, R, seed). For "pipelined" H, W, R describe the second submission and the first is
# PIPE_FIRST; "trunk_image" / "submit_u8" take a raw H x W image that the device scales (scale, max_size) = TRUNK_SCALE.
SEQUENCE = [
    ("detect_nms", 304, 400, 512, 0),       # largest of the prefix, max_rois, scaled-up image
    ("detect_nms", 240, 320, 129, 1),       # MultiPathNet's conv3 pyramid drops below the one-launch limit
    ("detect_cached", 240, 320, 64, 2),     # the features of the call before, which was on another size
    ("heads_chunks", 161, 227, 300, 3),     # odd sizes; chunks of 1, 128 and 171 ROIs
    ("detect_nms", 128, 176, 63, 4),        # smallest: the end of the descending prefix
    ("test_one", 200, 150, 65, 5),          # portrait
    ("detect_nms", 240, 320, 64, 6),        # A
    ("detect_nms", 128, 176, 1, 7),         # B: small after large
    ("detect_nms", 240, 320, 65, 8),        # A again
    ("trunk_image", 300, 380, 129, 9),      # raw 300 x 380 scaled on the device to 256 x 324
    ("pipelined", 320, 416, 512, 10),       # at the limits: grows buffers while PIPE_FIRST is in flight
    ("submit_u8", 250, 330, 90, 12),        # raw uint8, scaled on the device to 200 x 264
]
DESCENDING = 5                              # SEQUENCE[:DESCENDING] never grows a buffer
PIPE_FIRST = (144, 200, 100, 11)
TRUNK_SCALE = {"trunk_image": (256, 352), "submit_u8": (200, 300)}
CHUNKS = (1, 129)                           # heads_chunks boundaries


def scaled_size(H0, W0, scale, max_size):
    """getImages' size: shorter side to `scale`, longer side capped at `max_size`"""
    h, w, _ = _get_images_size(H0, W0, scale, max_size)
    return h, w


def trunk_sizes(seq=SEQUENCE):
    """the (H, W) of every trunk plan the sequence makes, in call order"""
    out = []
    for kind, H, W, R, seed in seq:
        if kind == "detect_cached":
            continue
        if kind == "pipelined":
            out.append(PIPE_FIRST[:2])
        if kind in TRUNK_SCALE:
            H, W = scaled_size(H, W, *TRUNK_SCALE[kind])
        out.append((H, W))
    return out


def roi_counts(seq=SEQUENCE):
    """every R a heads pass runs with"""
    out = []
    for kind, H, W, R, seed in seq:
        if kind == "heads_chunks":
            cuts = (0,) + CHUNKS + (R,)
            out += [b - a for a, b in zip(cuts[:-1], cuts[1:])]
        elif kind == "test_one":
            out += [R, R]                              # num_iter = 2: the second pass re-pools the regressed boxes
        else:
            if kind == "pipelined":
                out.append(PIPE_FIRST[2])
            out.append(R)
    return out


GRAPHS = {
    "vgg": lambda: models.vgg16_fast_rcnn(21, seed=7, width_div=4, fc_dim=256),
    "mpn": lambda: models.vgg16_multipathnet(21, seed=11, width_div=4, fc_dim=256),
    "resnet50": lambda: models.resnet50_fast_rcnn(21, seed=5, integral_k=3, blocks=(1, 1, 1, 1)),
    "nin": lambda: models.nin_fast_rcnn(21, seed=9),
}
CASES = [(g, n) for g in GRAPHS for n in ("default", "bf16", "fp8") if not (g == "nin" and n == "fp8")]   # fp8 refuses NIN's tails


def _image(spec, H, W, seed, first=False):
    raw = wl.raw_image(H, W, seed)
    if first:                                  # bright, then scaled: large activations in every buffer
        return 4.0 * wl.transform(0.5 + 0.5 * raw, spec.transformer)
    return wl.transform(raw, spec.transformer)


def _boxes(spec, R, H, W, seed):
    return (wl.sharpmask_boxes if len(spec.towers) > 1 or spec.transformer == "imagenet" else wl.random_boxes)(R, H, W, seed)


def _u8(H, W, seed):
    return np.ascontiguousarray((wl.raw_image(H, W, seed).transpose(1, 2, 0) * 255).astype(np.uint8))


def _same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    if a.dtype == np.float32:
        a, b = a.view(np.uint32), np.asarray(b, np.float32).view(np.uint32)
    return a.shape == b.shape and np.array_equal(a, b)


def _assert_same(got, want, what):
    """nested tuples / lists of arrays, bit for bit"""
    if isinstance(want, (tuple, list)):
        assert len(got) == len(want), what
        for k, (g, w) in enumerate(zip(got, want)):
            _assert_same(g, w, f"{what}[{k}]")
    elif want is None:
        assert got is None, what
    else:
        assert _same(got, want), what


class Call:
    """one call of the sequence: run(model) makes it (and, for detect_cached, needs the previous call's image on a fresh
    model), oracle() gives the fp64 comparison or None"""

    def __init__(self, spec, kind, H, W, R, seed, prev=None):
        self.spec, self.kind, self.H, self.W, self.R, self.seed, self.prev = spec, kind, H, W, R, seed, prev
        if kind in TRUNK_SCALE:
            self.raw = _u8(H, W, seed) if kind == "submit_u8" else wl.raw_image(H, W, seed)
            h, w = scaled_size(H, W, *TRUNK_SCALE[kind])
            self.boxes = _boxes(spec, R, H, W, seed)              # raw-image coordinates
            self.rois = O.project_rois(_boxes(spec, R, h, w, seed), 1.0)
        else:
            self.img = prev.img if kind == "detect_cached" else _image(spec, H, W, seed, first=seed == 0)
            self.boxes = _boxes(spec, R, H, W, seed)
        if kind == "pipelined":
            h, w, r, s = PIPE_FIRST
            self.first = (_image(spec, h, w, s), _boxes(spec, r, h, w, s), h, w)

    def run(self, m, fresh=False):
        spec, H, W = self.spec, self.H, self.W
        if self.kind == "detect_nms":
            return m.detect_nms(self.img, self.boxes, 1.0, W, H, -1.5, 0.3)
        if self.kind == "detect_cached":
            if fresh:
                return m.detect(self.img, self.boxes, 1.0, True)
            return m.detect(None, self.boxes, 1.0, False)
        if self.kind == "heads_chunks":
            m.trunk(self.img)
            rois = O.project_rois(self.boxes, 1.0)
            cuts = (0,) + CHUNKS + (self.R,)
            return [m.heads(rois[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
        if self.kind == "test_one":
            return m.test_one(self.img, self.boxes, 1.0, W, H, num_iter=2, use_rbox_scores=True, bbox_voting=True)
        if self.kind == "trunk_image":
            got = m.trunk_image(self.raw, spec.transformer, *TRUNK_SCALE["trunk_image"])
            return got, m.heads(self.rois)
        if self.kind == "pipelined":
            im1, bx1, h1, w1 = self.first
            if fresh:                        # each submission against the blocking call on a fresh model of its own
                return None
            t1 = m.detect_nms_submit(im1, bx1, 1.0, w1, h1, -1.5, 0.3)
            t2 = m.detect_nms_submit(self.img, self.boxes, 1.0, W, H, -1.5, 0.3)
            return m.detect_nms_wait(t1), m.detect_nms_wait(t2)
        if self.kind == "submit_u8":
            t = m.detect_nms_submit_u8(self.raw, self.boxes, spec.transformer, *TRUNK_SCALE["submit_u8"])
            return m.detect_nms_wait(t)
        raise AssertionError(self.kind)

    def fresh(self, ctx):
        """the same call on a model that makes only it"""
        def one(fn):
            f = mpn.Model(ctx, self.spec, max_rois=MAX_ROIS, max_h=MAX_H, max_w=MAX_W)
            try:
                return fn(f)
            finally:
                f.close()
        if self.kind == "pipelined":
            im1, bx1, h1, w1 = self.first
            return (one(lambda f: f.detect_nms(im1, bx1, 1.0, w1, h1, -1.5, 0.3)),
                    one(lambda f: f.detect_nms(self.img, self.boxes, 1.0, self.W, self.H, -1.5, 0.3)))
        return one(lambda f: self.run(f, fresh=True))

    def check_oracle(self, got, name):
        """default numerics: within 1e-3 normwise of the fp64 pipeline, keep lists equal to nms.c on the device's boxes"""
        spec, H, W = self.spec, self.H, self.W
        none = lambda sb, thr: np.zeros(0, np.int64)
        errs = []
        if self.kind in ("detect_nms", "pipelined"):
            pairs = [(got, self.img, self.boxes, H, W)]
            if self.kind == "pipelined":
                im1, bx1, h1, w1 = self.first
                pairs = [(got[0], im1, bx1, h1, w1), (got[1], self.img, self.boxes, H, W)]
            for (s, b, k), img, boxes, h, w in pairs:
                rs, rb, _ = G.test_one(spec, img, boxes, 1.0, w, h, nms_fn=none)
                errs += [rel_err(s, rs), rel_err(b, rb)]
                assert_nms_every_class(s, b, k)
        elif self.kind == "detect_cached":
            rs, rb = G.detect(spec, self.img, self.boxes, 1.0)
            errs += [rel_err(got[0], rs), rel_err(got[1], rb)]
        elif self.kind == "heads_chunks":
            rc, rb = G.heads_forward(spec, G.trunk_forward(spec, self.img), O.project_rois(self.boxes, 1.0))
            errs += [rel_err(np.concatenate([c for c, _ in got]), rc), rel_err(np.concatenate([b for _, b in got]), rb)]
        else:
            return 0.0                       # test_one / trunk_image / submit_u8: the fresh model only
        assert max(errs) < TOL, (name, self.kind, errs)
        return max(errs)


def _calls(spec, seq):
    out, prev = [], None
    for kind, H, W, R, seed in seq:
        c = Call(spec, kind, H, W, R, seed, prev)
        out.append(c)
        prev = c
    return out


def run_sequence(ctx, graph, numerics, seq=SEQUENCE, oracle=True):
    spec = GRAPHS[graph]()
    calls = _calls(spec, seq)
    worst = 0.0
    with options(ctx, NUMERICS[numerics]):
        m = mpn.Model(ctx, spec, max_rois=MAX_ROIS, max_h=MAX_H, max_w=MAX_W)
        try:
            for i, c in enumerate(calls):
                got = c.run(m)
                _assert_same(got, c.fresh(ctx), f"{graph}/{numerics} call {i} ({c.kind} {c.H} x {c.W}, R = {c.R})")
                if oracle and numerics == "default":
                    worst = max(worst, c.check_oracle(got, f"{graph} call {i}"))
        finally:
            m.close()
    return worst


@pytest.mark.parametrize("graph,numerics", CASES)
def test_one_model_through_the_sequence(ctx, graph, numerics):
    worst = run_sequence(ctx, graph, numerics)
    record_parity("shape_sequence", graph=graph, numerics=numerics, oracle_max=worst)


@pytest.mark.parametrize("graph", list(GRAPHS))
def test_descending_prefix(ctx, graph):
    """the prefix alone, where no buffer grows after the first call: every later call reads buffers that hold the larger
    first call's values past its own extent"""
    run_sequence(ctx, graph, "default", SEQUENCE[:DESCENDING], oracle=False)


def test_full_size_vgg16_over_coco_shaped_images(ctx):
    """BASELINE cfg 2 (VGG-16 Fast R-CNN) on one model over four COCO-shaped images, three landscape and one portrait,
    each call bit for bit against a fresh model"""
    spec = models.vgg16_fast_rcnn(21, seed=1234)
    lim = dict(max_rois=2048, max_h=1000, max_w=1000)
    m = mpn.Model(ctx, spec, **lim)
    try:
        for i, (H, W, R) in enumerate(((600, 800, 1000), (600, 1000, 2000), (600, 667, 300), (1000, 600, 1000))):
            img = _image(spec, H, W, 20 + i, first=i == 0)
            boxes = wl.random_boxes(R, H, W, 20 + i)
            got = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
            f = mpn.Model(ctx, spec, **lim)
            want = f.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
            f.close()
            _assert_same(got, want, f"full-size call {i} ({H} x {W}, R = {R})")
    finally:
        m.close()

"""GPU suite: getImages on the device (SURVEY 8f-1, mpn_get_images / mpn_model_trunk_image; ImageDetect.lua:22-52 +
modules/ImageTransformer.lua:19-33) — bit-exact against the two-pass oracle and the committed golden fixture, and the
raw-image detect path against the host getImages path. (First GPU run: all green; the xfail markers of
round 1 are gone.)"""
import os

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from multipathnet_b200.image_detect import ImageDetect
from multipathnet_b200.modules import ImageTransformer

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("H0,W0,scale,max_size", [(60, 80, 60, 100), (48, 64, 75, 1000), (120, 90, 60, 1000), (50, 200, 100, 300), (333, 500, 600, 1000)])
@pytest.mark.parametrize("kind", ["ross", "imagenet"])
def test_get_images_matches_the_oracle_bit_for_bit(ctx, oracle_built, H0, W0, scale, max_size, kind):
    im = wl.raw_image(H0, W0, H0 + W0)
    ref, s_ref = oracle_built.get_images(im, kind, scale, max_size)
    out, s = ctx.get_images(im, kind, scale, max_size)
    assert s == s_ref and out.shape == ref.shape
    assert np.array_equal(out, ref)


def test_get_images_golden_fixture(ctx):
    g = np.load(os.path.join(os.path.dirname(__file__), "golden", "getimages_golden.npz"))
    for name in ("grow", "shrink", "capped", "same"):
        scale, max_size, s, inet = g[name + "_cfg"]
        out, so = ctx.get_images(g[name + "_im"], "imagenet" if inet else "ross", scale, max_size)
        assert so == s and np.array_equal(out, g[name + "_out"])


def test_detect_from_the_raw_image_equals_the_host_getimages_path(ctx):
    spec = models.vgg16_fast_rcnn(21, seed=3, width_div=4, fc_dim=256)
    m = mpn.Model(ctx, spec, max_rois=64, max_h=192, max_w=256)
    im = wl.raw_image(96, 128, 7)
    boxes = wl.random_boxes(32, 96, 128, 7)
    host = ImageDetect(m, ImageTransformer("ross"), scale=[120], max_size=200)
    dev = ImageDetect(m, ImageTransformer("ross"), scale=[120], max_size=200, on_device=True)
    s0, b0 = host.detect(im, boxes)
    s1, b1 = dev.detect(im, boxes)
    assert np.array_equal(s0, s1) and np.array_equal(b0, b1)           # same image bits in, same kernels after
    s2, b2 = dev.detect(None, boxes, recompute_features=False)         # cached features (ImageDetect.lua:109-111)
    assert np.array_equal(s1, s2) and np.array_equal(b1, b2)
    m.close()


@pytest.mark.parametrize("H0,W0,scale,max_size", [(60, 80, 60, 100), (120, 90, 60, 1000), (333, 500, 600, 1000), (480, 640, 600, 1000)])
@pytest.mark.parametrize("kind", ["ross", "imagenet"])
def test_get_images_from_the_decoder_bytes(ctx, oracle_built, H0, W0, scale, max_size, kind):
    """uint8 H x W x 3 in (what a JPEG decoder leaves): value = byte / 255 in fp32, then exactly the fp32 path — bit for bit
    against the oracle fed with that float image"""
    rng = np.random.default_rng(H0 * W0)
    im_u8 = rng.integers(0, 256, (H0, W0, 3), dtype=np.uint8)
    im_f = np.ascontiguousarray((im_u8.astype(np.float32) / np.float32(255.0)).transpose(2, 0, 1))
    ref, s_ref = oracle_built.get_images(im_f, kind, scale, max_size)
    out, s = ctx.get_images_u8(im_u8, kind, scale, max_size)
    assert s == s_ref and out.shape == ref.shape and np.array_equal(out, ref)
    out_f, _ = ctx.get_images(im_f, kind, scale, max_size)
    assert np.array_equal(out, out_f)


def test_raw_u8_submit_equals_the_host_getimages_path(ctx):
    """mpn_model_detect_nms_submit_u8 (raw bytes up, getImages + trunk + heads + NMS on the device) == getImages on the host +
    mpn_model_detect_nms, bit for bit, two images in flight"""
    spec = models.vgg16_fast_rcnn(21, seed=3, width_div=4, fc_dim=256)
    m = mpn.Model(ctx, spec, max_rois=128, max_h=192, max_w=256)
    rng = np.random.default_rng(5)
    ims = [rng.integers(0, 256, (96, 128, 3), dtype=np.uint8) for _ in range(3)]
    boxes = [wl.random_boxes(64, 96, 128, 40 + i) for i in range(3)]
    want = []
    for im, bx in zip(ims, boxes):
        im_f = np.ascontiguousarray((im.astype(np.float32) / np.float32(255.0)).transpose(2, 0, 1))
        img, s = ctx.get_images(im_f, "ross", 120, 200)
        want.append(m.detect_nms(img, bx, s, 128, 96, 0.0, 0.3))
    tickets = [m.detect_nms_submit_u8(ims[0], boxes[0], "ross", 120, 200, 0.0, 0.3)]
    got = []
    for i in (1, 2):
        tickets.append(m.detect_nms_submit_u8(ims[i], boxes[i], "ross", 120, 200, 0.0, 0.3))
        got.append(m.detect_nms_wait(tickets[i - 1]))
    got.append(m.detect_nms_wait(tickets[2]))
    for (s0, b0, k0), (s1, b1, k1) in zip(want, got):
        assert np.array_equal(s0, s1) and np.array_equal(b0, b1) and all(np.array_equal(a, b) for a, b in zip(k0, k1))
    m.close()

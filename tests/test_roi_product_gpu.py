"""GPU parity of the kernels the benchmark actually times on the ROI stage (VERDICT r01, weak #1):
`roi_pool_cluster_kernel` on the fp32 max pyramid (`maxpyr_*`), and the two-pass `roi_pool_split_kernel` that normalised
levels too large for its shared-memory staging fall back to, with the fused Foveal region
and the per-level L2 normalise x 1000 — checked on the POOLED TENSOR itself (mpn_model_get_pooled), not through the
whole-graph 1e-3 bar. The oracle runs on the GPU's OWN feature maps (mpn_model_get_trunk_slot), so the comparison isolates
the ROI stage:   orc_foveal (Foveal.lua:26-39) -> orc_roi_pool (imagine-nn) [-> orc_l2_normalize, x 1000
(model_utils.lua:217-220,240)] -> JoinTable(2) (model_utils.lua:229-235).

Bars. Un-normalised towers: BIT-EXACT. A feature-map value is hi + lo of two bf16 (exact in fp32), the pooled value is
the maximum of such values, and re-splitting it into (hi', lo') loses nothing, so hi' + lo' equals the oracle's fp32
maximum bit for bit. Normalised towers: the stored value is the split (hi + lo, 16-17 significant bits) of
fl(fl(x / nrm) * 1000) and the kernel's fp32 tree sum of squares differs from the oracle's double accumulation in the
last ulps, hence  |got - split(ref)| <= 1e-6 * max|ref| + 2^-16 * |ref|  elementwise (the second term is the storage
quantum of the split planes, not kernel error) and >= 99 % of the elements bit-equal to split(ref)."""
import dataclasses

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models, workloads as wl
from oracle import ref as O

pytestmark = pytest.mark.gpu


def bf16_rn(x):
    u = np.ascontiguousarray(x, np.float32).view(np.uint32).astype(np.uint64)
    r = ((u >> 16) & 1) + 0x7FFF
    return ((u + r) & 0xFFFF0000).astype(np.uint32).view(np.float32)


def split_join(x):
    """what the split-bf16 planes hold for an fp32 value: hi = rn_bf16(x), lo = rn_bf16(x - hi); hi + lo"""
    x = np.ascontiguousarray(x, np.float32)
    hi = bf16_rn(x)
    return hi + bf16_rn(x - hi)


def oracle_pooled(spec, m, rois, tower, rows):
    """n x bins x Ctot, channels-last like the product tensor, from the GPU's own trunk slots"""
    t = spec.towers[tower]
    r = np.ascontiguousarray(rois[rows], np.float32)
    n = r.shape[0]
    reg = r if t.region == 0 else np.ascontiguousarray(O.foveal(r).reshape(n, 4, 5)[:, t.region, :])
    parts = []
    for slot, scale in t.levels:
        fm = m.trunk_slot(slot)
        p = O.roi_pool(fm, reg, t.pooled_w, t.pooled_h, np.float32(scale), spec.roi_variant)      # n x C x PH x PW
        if t.normalize:
            p = O.l2_normalize(p.reshape(n, -1)).reshape(p.shape) * np.float32(1000.0)
        parts.append(p)
    x = np.concatenate(parts, axis=1)
    return np.ascontiguousarray(x.reshape(n, x.shape[1], -1).transpose(0, 2, 1))


def check_tower(spec, m, rois, tower, rows, ref=None, fp16_planes=False):
    t = spec.towers[tower]
    got = m.pooled(tower, rows.start, rows.stop - rows.start)
    ref = oracle_pooled(spec, m, rois, tower, rows) if ref is None else ref
    assert got.shape == ref.shape
    if fp16_planes:
        # the pooled tensor feeds a "w16" Linear and is stored as fp16 hi / lo planes: 22 significant bits on an absolute
        # 2^-24 grid (fp16 subnormals). The value itself is hi + lo of two bf16 planes and can carry all 24 fp32 bits (a small
        # `lo` sits far below `hi`), so: within 2^-22 relative + the grid everywhere, and exact for the bulk of the values
        assert not t.normalize
        err = np.abs(got - ref)
        assert (err <= 2.0 ** -22 * np.abs(ref) + 2.0 ** -24).all(), f"tower {tower}: worst {err.max():.3e}"
        same = float(np.mean(got == ref))
        assert same > 0.99, f"tower {tower}: only {same:.4f} of the fp16-plane values are exact"
        return same
    if not t.normalize:
        assert np.array_equal(got, ref), f"tower {tower}: {np.count_nonzero(got != ref)} of {got.size} pooled values differ"
        return 1.0
    want = split_join(ref)
    bound = 1e-6 * np.abs(ref).max() + 2.0 ** -16 * np.abs(ref)
    bad = np.abs(got - want) > bound
    assert not bad.any(), f"tower {tower}: {np.count_nonzero(bad)} values outside the bound, worst {np.abs(got - want).max():.3e}"
    same = float(np.mean(got == want))
    assert same > 0.99, f"tower {tower}: only {same:.4f} of the values are bit-equal to split(ref)"
    return same


def run_detect(m, spec, H, W, R, seed, sharp):
    img = wl.transform(wl.raw_image(H, W, seed), spec.transformer)
    boxes = (wl.sharpmask_boxes if sharp else wl.random_boxes)(R, H, W, seed)
    m.detect(img, boxes, 1.0)
    return O.project_rois(boxes, np.float32(1.0))


def test_fused_roi_small_unnormalised_and_regions_leaving_the_image(ctx):
    """Fast R-CNN head (region 0) on a small map, ROIs that touch / leave the borders, degenerate 1-px boxes"""
    spec = models.vgg16_fast_rcnn(21, seed=7, width_div=4, fc_dim=256)
    m = mpn.Model(ctx, spec, max_rois=512, max_h=256, max_w=320)
    H, W, R = 150, 203, 300
    img = wl.transform(wl.raw_image(H, W, 1), spec.transformer)
    boxes = wl.random_boxes(R, H, W, 1)
    boxes[:8] = [[1, 1, W, H], [1, 1, 1, 1], [W, H, W, H], [W - 1, 1, W, H], [1, H - 1, W, H], [5, 5, 5, 90], [7, 9, 180, 9], [100, 70, 101, 71]]
    m.detect(img, boxes, 1.0)
    rois = O.project_rois(boxes, np.float32(1.0))
    check_tower(spec, m, rois, 0, slice(0, R))
    m.close()


def test_fused_roi_multipathnet_small_all_towers(ctx):
    """cfg 3 structure at reduced width: towers 0..3 = Foveal regions x1, x1.5, x2, x4 on conv5|conv4|conv3 with per-level
    L2 normalise"""
    pytest.raises(mpn.MpnError, ctx.set_option, "roi_impl", 0)     # the kernel is chosen from the launch, not by a knob
    spec = models.vgg16_multipathnet(21, seed=11, width_div=4, fc_dim=256)
    m = mpn.Model(ctx, spec, max_rois=256, max_h=256, max_w=320)
    try:
        rois = run_detect(m, spec, 160, 208, 128, 6, sharp=True)
        for t in range(len(spec.towers)):
            check_tower(spec, m, rois, t, slice(0, 128))
    finally:
        m.close()


@pytest.mark.parametrize("fc_w16", [1, 0])
def test_fused_roi_full_size_cfg2(ctx, fc_w16):
    """BASELINE configs[1]: VGG-16 600x800, R=1000, 7x7 bins on conv5 — every pooled value of the timed kernel: bit-exact as
    bf16 planes (fc_w16 = 0), exact down to the fp16 subnormal grid as fp16 planes (the default: fc6 takes the w16 numerics)"""
    spec = models.vgg16_fast_rcnn(21, seed=1234)
    ctx.set_option("fc_w16", fc_w16)
    m = mpn.Model(ctx, spec, max_rois=1024, max_h=608, max_w=800)
    try:
        rois = run_detect(m, spec, 600, 800, 1000, 2, sharp=False)
        check_tower(spec, m, rois, 0, slice(0, 1000), fp16_planes=bool(fc_w16))
    finally:
        ctx.set_option("fc_w16", -1)
        m.close()


def test_fused_roi_full_size_cfg3_all_towers(ctx):
    """BASELINE configs[2]: all five MultiPathNet towers at full size (regions leaving the image, SURVEY A.4), a second
    detect on the same model against ONE oracle evaluation of the first (the trunk is deterministic: same feature maps
    every run)"""
    spec = models.vgg16_multipathnet(81, seed=1234)
    m = mpn.Model(ctx, spec, max_rois=1024, max_h=608, max_w=800)
    try:
        rois = run_detect(m, spec, 600, 800, 1000, 3, sharp=True)
        blocks = (slice(0, 200), slice(800, 1000))                  # 400 of the 1000 ROIs per tower: ~30 s of oracle time in all
        refs = {(t, b.start): oracle_pooled(spec, m, rois, t, b) for t in range(len(spec.towers)) for b in blocks}
        run_detect(m, spec, 600, 800, 1000, 3, sharp=True)
        for t in range(len(spec.towers)):
            for b in blocks:
                check_tower(spec, m, rois, t, b, refs[(t, b.start)])
    finally:
        m.close()


def test_fused_roi_full_size_cfg4(ctx):
    """BASELINE configs[3]: ResNet-50, 800x1000, R=2000, 14x14 bins on layer3 (1024 channels) — rows from both ends"""
    spec = models.resnet50_fast_rcnn(81, seed=1234, integral_k=6)
    m = mpn.Model(ctx, spec, max_rois=2048, max_h=808, max_w=1000)
    try:
        rois = run_detect(m, spec, 800, 1000, 2000, 4, sharp=True)
        for rows in (slice(0, 150), slice(1850, 2000)):
            check_tower(spec, m, rois, 0, rows)
    finally:
        m.close()


def test_fused_roi_normalised_level_too_large_for_shared_memory(ctx):
    """A normalised level whose quarter of the PH*PW*C vector exceeds the cluster kernel's 160 KB of staging is pooled by
    the two-pass roi_pool_split_kernel: ResNet-50's 14x14 bins on layer3 (1024 channels) with the tower normalised need
    49 x 1024 x 4 = 200,704 bytes per quarter. The pooled tensor meets the normalised bar, and a detect launches exactly one
    kernel more than with the same tower un-normalised (one cluster kernel launch)."""
    plain = models.resnet50_fast_rcnn(21, seed=5, integral_k=3)
    normed = dataclasses.replace(plain, towers=[dataclasses.replace(plain.towers[0], normalize=1)])
    launches = {}
    for spec in (plain, normed):
        m = mpn.Model(ctx, spec, max_rois=128, max_h=256, max_w=320)
        try:
            rois = run_detect(m, spec, 160, 224, 64, 8, sharp=True)
            check_tower(spec, m, rois, 0, slice(0, 64))
            n0 = ctx.launch_count
            run_detect(m, spec, 160, 224, 64, 8, sharp=True)
            launches[spec.towers[0].normalize] = ctx.launch_count - n0
        finally:
            m.close()
    assert launches[1] == launches[0] + 1, launches

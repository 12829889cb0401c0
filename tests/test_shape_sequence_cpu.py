"""Host only: the shape sequences of tests/test_shape_sequence_gpu.py and tests/test_train_sequence_gpu.py reach what they
claim, computed from the specs' shapes and the planner's host view (mpn_debug_plan), so a planner change that made a
sequence lose a crossing fails here rather than silently weakening the GPU tests."""
import ctypes

import numpy as np

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from multipathnet_b200._lib import MPN_LAYER_CONV
import test_shape_sequence_gpu as S
import test_train_sequence_gpu as T

SM = 132                                # H100 SXM
MAXPYR_ALL_SMEM = 200 * 1024            # csrc/roi.cu mpn_maxpyr_all_launch: H x W x 2 float4 of shared memory


def _plan(N, Cin, H, W, Cout, k, s, p, per_roi):
    out = (ctypes.c_int32 * 8)()
    assert mpn.load_library().mpn_debug_plan(N, Cin, H, W, Cout, k, s, p, per_roi, SM, out) == 0
    return dict(zip(("mode", "cg", "bn", "splitk", "streamk", "tn", "th", "tw"), out))


def _trunk_shapes(spec, H, W):
    """slot -> (H, W) of the trunk at an H x W image"""
    shp = {0: (H, W)}
    for L in spec.trunk_layers:
        h, w = shp[L.in_slot]
        if L.kind == MPN_LAYER_CONV:
            shp[L.out_slot] = ((h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1)
        else:
            shp[L.out_slot] = (models._pool_out(h, L.kh, L.stride, L.pad, L.ceil_mode),
                               models._pool_out(w, L.kw, L.stride, L.pad, L.ceil_mode))
    return shp


def _trunk_patches(spec, H, W):
    """per engine-planned trunk convolution (not the direct first layer) its patch (tn, th, tw)"""
    shp = _trunk_shapes(spec, H, W)
    out = {}
    for i, L in enumerate(spec.trunk_layers):
        if L.kind != MPN_LAYER_CONV or L.cin % 8:
            continue
        h, w = shp[L.in_slot]
        pl = _plan(1, L.cin, h, w, L.cout, L.kh, L.stride, L.pad, 0)
        out[i] = (pl["tn"], pl["th"], pl["tw"])
    return out


def test_sequence_sizes_stay_within_the_limits_and_the_prefix_descends():
    sizes = S.trunk_sizes()
    assert all(h <= S.MAX_H and w <= S.MAX_W for h, w in sizes)
    pre = S.trunk_sizes(S.SEQUENCE[:S.DESCENDING])
    assert all(h1 <= h0 and w1 <= w0 for (h0, w0), (h1, w1) in zip(pre, pre[1:]))
    assert S.SEQUENCE[0][3] == S.MAX_ROIS and pre[0] == max(pre, key=lambda s: s[0] * s[1])
    assert any(h > w for h, w in sizes) and any(h % 2 and w % 2 for h, w in sizes)
    area = [h * w for h, w in sizes]
    assert max(area) > area[0] and area.index(max(area)) > len(pre)          # a buffer grows after the prefix
    kinds = {k for k, *_ in S.SEQUENCE}
    assert kinds == {"detect_nms", "detect_cached", "heads_chunks", "test_one", "trunk_image", "pipelined", "submit_u8"}
    i = [k for k, *_ in S.SEQUENCE].index("detect_cached")
    assert S.SEQUENCE[i - 1][0] == "detect_nms" and S.SEQUENCE[i - 1][1:3] != S.SEQUENCE[i - 2][1:3]
    seq = [s for s in sizes]                                                   # A, B, A
    assert any(seq[j] == seq[j + 2] != seq[j + 1] for j in range(len(seq) - 2))
    first, second = S.PIPE_FIRST[:2], sizes[[k for k, *_ in S.SEQUENCE if k != "detect_cached"].index("pipelined") + 1]
    assert first != second and second[0] * second[1] == max(area)


def test_roi_counts_cover_every_edge():
    rs = S.roi_counts()
    assert {1, 63, 64, 65, 129, S.MAX_ROIS} <= set(rs)
    assert max(rs) == S.MAX_ROIS
    assert any(a > b for a, b in zip(rs, rs[1:])) and any(a < b for a, b in zip(rs, rs[1:]))
    assert S.CHUNKS == (1, 129)


def test_multipathnet_conv3_pyramid_crosses_the_one_launch_limit_both_ways():
    spec = S.GRAPHS["mpn"]()
    slot = spec.taps["conv3"]
    too_big = []
    for H, W in S.trunk_sizes():
        h, w = _trunk_shapes(spec, H, W)[slot]
        too_big.append(h * w * 32 > MAXPYR_ALL_SMEM)
    assert too_big[0] and any(a and not b for a, b in zip(too_big, too_big[1:])) and any(b and not a for a, b in zip(too_big, too_big[1:]))
    sizes = S.trunk_sizes()
    assert any(a[0] * a[1] > b[0] * b[1] for a, b in zip(sizes, sizes[1:]))  # small after large: a deeper pyramid than fresh


def test_generic_patches_change_between_consecutive_trunk_plans():
    for g in ("resnet50", "nin"):
        spec = S.GRAPHS[g]()
        pats = [_trunk_patches(spec, H, W) for H, W in S.trunk_sizes()]
        changes = [sum(a[i] != b[i] for i in a) for a, b in zip(pats, pats[1:])]
        assert sum(1 for c in changes if c) >= 3, (g, changes)


def test_per_roi_layers_do_not_move_with_r():
    for g in S.GRAPHS:
        spec = S.GRAPHS[g]()
        for Tw in spec.towers:
            shp = {0: (Tw.pooled_h, Tw.pooled_w)}
            for L in Tw.layers:
                h, w = shp[L.in_slot]
                if L.kind != MPN_LAYER_CONV:                  # FLATTEN / AVGPOOL: one pixel per ROI
                    shp[L.out_slot] = (1, 1)
                    continue
                shp[L.out_slot] = ((h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1)
                plans = {(p["bn"], p["splitk"]) for p in (_plan(R, L.cin, h, w, L.cout, L.kh, L.stride, L.pad, 1)
                                                         for R in sorted(set(S.roi_counts())))}
                assert len(plans) == 1, (g, L.cin, L.cout, plans)
        for hd in list(spec.cls_heads) + [spec.bbox_head]:
            plans = {(p["bn"], p["splitk"]) for p in (_plan(R, hd.col_len, 1, 1, hd.cout, 1, 1, 0, 1) for R in sorted(set(S.roi_counts())))}
            assert len(plans) == 1, (g, "head", plans)


def test_training_batches_cover_every_r_case():
    Rs = [sum(n for _, _, n in b) for b in T.BATCHES]
    cap = T.LIMITS["max_rois"]
    ceil64 = [(r + 63) // 64 * 64 for r in Rs]
    assert any(r < 64 for r in Rs) and 64 in Rs and cap in Rs
    assert any(Rs[k] % 64 and ceil64[k - 1] > ceil64[k] for k in range(1, len(Rs)))
    assert {len(b) for b in T.BATCHES} == {1, 2, 3}
    assert any(n == 0 for b in T.BATCHES for _, _, n in b)
    areas = [[h * w for h, w, _ in b] for b in T.BATCHES]
    assert any(a[0] == max(a) and len(a) > 1 for a in areas) and any(a[0] == min(a) and len(a) > 1 for a in areas)
    assert any(h > w for b in T.BATCHES for h, w, _ in b)
    assert all(h <= T.LIMITS["max_h"] and w <= T.LIMITS["max_w"] for b in T.BATCHES for h, w, _ in b)
    for name, (make, kw, plan) in T.SETUPS.items():
        assert len(plan) >= 5 and len(plan) <= len(T.BATCHES), name
        if kw.get("train_trunk"):                       # the image without ROIs is in a trunk-training step
            assert any(n == 0 for _, _, n in T.BATCHES[1]), name
    heads = [h for h, _, _ in T.SETUPS["b_mpn_phase2_integral"][2]]
    assert len(set(heads)) > 1 and [s for _, s, _ in T.SETUPS["b_mpn_phase2_integral"][2]].index(True) == 2
    full = [sum(n for _, _, n in b) for b in T.FULL_BATCHES]
    assert full == [256, 64, 256]

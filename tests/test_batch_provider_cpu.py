"""CPU: the training feed's rules through the product's host views (mpn_debug_attach_proposals, mpn_sample_plan,
mpn_train_images_size, mpn_debug_sample_rows, compiled from csrc/roidb_rule.cuh) against hand-computed answers and the
numpy restatement in _batch_provider_ref.py."""
import ctypes as C

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import batch_provider as bp
import _batch_provider_ref as ref

f32 = np.float32


def lib():
    return mpn.load_library()


def attach(anns, props, scores=None, best_number=1000, min_area=0.0, min_prop_area=0.0, num_classes=80):
    """anns: (x, y, w, h, area, class, crowd, difficult) -> (boxes, overlap, corr, label, n_gt) from the host view"""
    a = np.array(anns, np.float64).reshape(-1, 8)
    xywh, area = np.ascontiguousarray(a[:, :4]), np.ascontiguousarray(a[:, 4])
    cls = np.ascontiguousarray(a[:, 5], np.int32)
    flags = np.ascontiguousarray(a[:, 6].astype(np.int32) | (a[:, 7].astype(np.int32) << 1), np.int32)
    p = np.ascontiguousarray(np.asarray(props, f32).reshape(-1, 4))
    s = None if scores is None else np.ascontiguousarray(scores, f32)
    n, g = C.c_int64(), C.c_int32()
    args = (len(a), xywh.ctypes.data, area.ctypes.data, cls.ctypes.data, flags.ctypes.data, min_area, len(p), p.ctypes.data,
            None if s is None else s.ctypes.data, best_number, min_prop_area, num_classes)
    assert lib().mpn_debug_attach_proposals(*args, None, None, None, None, 0, C.byref(n), C.byref(g)) == 0
    b, o = np.empty((n.value, 4), f32), np.empty(n.value, f32)
    c, lab = np.empty(n.value, np.int32), np.empty(n.value, np.int32)
    assert lib().mpn_debug_attach_proposals(*args, b.ctypes.data, o.ctypes.data, c.ctypes.data, lab.ctypes.data, n.value, None, None) == 0
    return b, o, c, lab, g.value


def sample_rows(rois, gts, labels, s, width, flip, mean, std, Cn):
    rois, gts = (np.ascontiguousarray(x, f32).reshape(-1, 4) for x in (rois, gts))
    lab = np.ascontiguousarray(labels, np.int32)
    mean, std = np.ascontiguousarray(mean, f32), np.ascontiguousarray(std, f32)
    R = len(lab)
    b, t = np.empty((R, 4), f32), np.empty((R, 4 * Cn), f32)
    assert lib().mpn_debug_sample_rows(R, rois.ctypes.data, gts.ctypes.data, lab.ctypes.data, s, width, flip, mean.ctypes.data,
                                       std.ctypes.data, Cn, b.ctypes.data, t.ctypes.data) == 0
    return b, t


def test_gt_box_and_boxoverlap_plus_one_widths():
    """GT (x, y, w, h) -> (x, y, x + w + 1, y + h + 1); IoU with +1 widths: a 10 x 10 json box covers 11 x 11 pixels"""
    b, o, c, lab, g = attach([(0, 0, 10, 10, 100, 3, 0, 0)], [[0, 0, 10, 10], [0, 0, 11, 11], [20, 20, 30, 30]])
    assert g == 1 and np.array_equal(b[0], [0, 0, 11, 11])
    assert o[0] == 1 and c[0] == 1 and lab[0] == 3                       # the GT row overlaps itself
    assert o[1] == f32(121) / f32(144) and c[1] == 1 and lab[1] == 3      # 11 x 11 inside 12 x 12
    assert o[2] == 1                                                      # the proposal equal to the GT box
    assert o[3] == 0 and c[3] == 0 and lab[3] == 0                        # disjoint: w < 0, overlap 0, no correspondance


def test_barea_in_double_rounded_once():
    """barea is a Lua number: (b3 - b1 + 1) * (b4 - b2 + 1) in double, rounded to fp32 when added to aarea"""
    gt = [(0.1, 0.1, 4096.3, 4096.7, 1e7, 1, 0, 0)]
    prop = [[0.1, 0.1, 2000.5, 3001.25]]
    _, o, *_ = attach(gt, prop)
    g = ref.gt_rows([gt[0]])[0][0]
    assert o[1] == ref.boxoverlap(np.array(prop, f32), g)[0]
    barea32 = ((g[2] - g[0]) + f32(1)) * ((g[3] - g[1]) + f32(1))        # the all-fp32 order: a different answer here
    a = np.array(prop, f32)[0]
    aarea = ((a[2] - a[0]) + f32(1)) * ((a[3] - a[1]) + f32(1))
    x2, y2 = min(a[2], g[2]), min(a[3], g[3])
    inter = ((x2 - a[0]) + f32(1)) * ((y2 - a[1]) + f32(1))
    barea64 = (float(g[2]) - float(g[0]) + 1.0) * (float(g[3]) - float(g[1]) + 1.0)
    assert f32(barea64) != barea32
    assert o[1] == inter / ((aarea + f32(barea64)) - inter)


def test_tie_goes_to_the_lower_gt_index():
    b, o, c, lab, g = attach([(5, 5, 20, 20, 400, 4, 0, 0), (5, 5, 20, 20, 400, 7, 0, 0)], [[5, 5, 26, 26]])
    assert g == 2 and c[0] == 1 and c[1] == 1 and c[2] == 1 and lab[1] == 4 and lab[2] == 4


def test_thresholds_at_exact_overlap():
    """overlap exactly 0.5 is fg (>=) and not bg (< 0.5); overlap exactly fp32(0.1) is bg (>=)"""
    _, o, *_ = attach([(0, 0, 2, -1, 4, 2, 0, 0)], [[0, 0, 1, 0]])           # GT 4 x 1 pixels, proposal 2 x 1 inside it
    assert o[1] == f32(0.5)
    bg, fg = ref.lists(o, 0.5, 0.1, 0.5)
    assert fg.tolist() == [0, 1] and bg.tolist() == []
    _, o, *_ = attach([(0, 0, 8, -1, 10, 2, 0, 0)], [[0, 0, 0, 0]])           # GT 10 x 1, proposal 1 x 1: 1 / 10
    assert o[1] == f32(0.1)
    bg, fg = ref.lists(o, 0.5, 0.1, 0.5)
    assert fg.tolist() == [0] and bg.tolist() == [1]


def test_crowd_mask_and_negative_times_negative_intersection():
    """intersection does not zero negative widths: a box down-right of the crowd box (w < 0 and h < 0) gets a positive
    value and is masked; GT rows are exempt"""
    crowd = (0, 0, 9, 9, 100, 1, 1, 0)                   # crowd box (0, 0, 10, 10)
    gt = (50, 50, 9, 9, 100, 2, 0, 0)                    # GT far away: its own row must stay
    far = [14, 14, 15, 15]                               # w = 10 - 14 + 1 = -3, h = -3: inter 9, area 4 -> 2.25 > 0.7
    inside = [1, 1, 8, 8]
    partial = [5, 0, 30, 10]
    b, o, c, lab, g = attach([crowd, gt, (0, 0, 9, 9, 100, 3, 0, 0)], [far, inside, partial])
    assert g == 2                                        # the crowd is not a GT object
    assert o[0] == 1 and o[1] == 1                       # GT rows: exempt (the second GT row lies inside the crowd box)
    assert o[2] == -1 and o[3] == -1
    assert o[4] != -1
    assert ref.intersection(np.array([far], f32), np.array([0, 0, 10, 10], f32))[0] == f32(2.25)


def test_image_without_gt_and_with_gt_but_no_proposals():
    b, o, c, lab, g = attach([], [[0, 0, 5, 5], [1, 1, 9, 9]])
    assert g == 0 and np.all(o == 0) and np.all(c == 0) and np.all(lab == 0)
    b, o, c, lab, g = attach([(0, 0, 5, 5, 25, 2, 0, 0)], np.zeros((0, 4)))
    assert g == 1 and len(o) == 1 and o[0] == 1 and lab[0] == 2


def test_area_difficult_and_proposal_filters():
    anns = [(0, 0, 5, 5, 0.0, 1, 0, 0), (0, 0, 5, 5, 25, 2, 0, 1), (0, 0, 5, 5, 25, 3, 0, 0)]
    _, _, _, lab, g = attach(anns, np.zeros((0, 4)))
    assert g == 1 and lab[0] == 3                        # area 0 is not > 0; difficult is not GT
    props = np.array([[0, 0, 2, 2], [0, 0, 10, 10], [0, 0, 3, 3], [0, 0, 6, 6]], f32)
    scores = np.array([0.5, 0.5, 0.9, 0.1], f32)
    b, *_ = attach([], props, scores, best_number=3)
    assert np.array_equal(b, props[[2, 0, 1]])           # best 3 by score, ties in their original order
    b, *_ = attach([], props, scores, min_prop_area=4.0)
    assert np.array_equal(b, props[[1, 2, 3]])           # (x2 - x1) * (y2 - y1) > 4
    b, *_ = attach([], props, None, best_number=2)
    assert np.array_equal(b, props)                      # no scores: no score filter


def test_refusals_of_the_host_view():
    a = np.array([[0, 0, 5, 5]], np.float64)
    area, cls, fl = np.array([25.0]), np.array([90], np.int32), np.zeros(1, np.int32)
    n = C.c_int64()
    assert lib().mpn_debug_attach_proposals(1, a.ctypes.data, area.ctypes.data, cls.ctypes.data, fl.ctypes.data, 0.0, 0, None, None, 10, 0.0,
                                            80, None, None, None, None, 0, C.byref(n), None) != 0     # class 90 > 80
    a[0, 2] = np.inf
    cls[0] = 1
    assert lib().mpn_debug_attach_proposals(1, a.ctypes.data, area.ctypes.data, cls.ctypes.data, fl.ctypes.data, 0.0, 0, None, None, 10, 0.0,
                                            80, None, None, None, None, 0, C.byref(n), None) != 0     # not finite


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_attach_agrees_with_the_restatement(seed):
    gt, props, _ = ref.synthetic_coco(24, 6, seed)
    thr = [(0.5, 0.1, 0.5), (0.7, 0.0, 0.7)]
    R = ref.restate_roidb(gt, props, 6, thr, best_number=40)
    cat_index = {c["id"]: k + 1 for k, c in enumerate(sorted(gt["categories"], key=lambda c: c["id"]))}
    pidx = {f: k for k, f in enumerate(props["images"])}
    for i, im in enumerate(sorted(gt["images"], key=lambda im: im["id"])):
        anns = [(*a["bbox"], a["area"], cat_index[a["category_id"]], a["iscrowd"], 0) for a in gt["annotations"] if a["image_id"] == im["id"]]
        k = pidx[im["file_name"]]
        b, o, c, lab, g = attach(anns, props["boxes"][k], props["scores"][k], best_number=40, num_classes=6)
        allb, corr, rlab, lists, ov = R[i]
        assert np.array_equal(b, allb) and np.array_equal(o.view(np.uint32), ov.view(np.uint32))
        assert np.array_equal(c, corr) and np.array_equal(lab, rlab)


def test_philox_draws_and_plan_match_the_restatement():
    n_bg = np.array([0, 3, 0, 5, 2, 0, 1], np.int32)
    n_fg = np.array([2, 0, 0, 4, 0, 1, 0], np.int32)
    for seed, step in [(555, 0), (555, 1), (2 ** 40 + 7, 12345)]:
        P = bp.sample_plan(n_bg, n_fg, seed, step, 1, 4)
        assert np.array_equal(P, ref.plan(n_bg, n_fg, seed, step, 1, 4))
        for img, b, f, fl in P:
            assert n_bg[b] > 0 and n_fg[f] > 0 and (img == b or img == f) and fl in (0, 1)
    assert bp.sample_plan(n_bg, n_fg, 1, 2, 0, 3).tolist() != bp.sample_plan(n_bg, n_fg, 1, 3, 0, 3).tolist()
    u = ref.draw_u32(0, 0, 0, 0, 0, [0])                 # counter word 3 = 0, zero key: Random123's known answer
    assert int(u[0]) == 0x6627e8d5


def test_permute_idx_merge_quirk():
    """no image has both kinds: a slot still completes, its bg rows from one image and its fg rows from another, and it
    trains on the image its last draw found"""
    n_bg = np.array([4, 0, 0], np.int32)
    n_fg = np.array([0, 0, 3], np.int32)
    P = bp.sample_plan(n_bg, n_fg, 9, 4, 0, 8)
    assert np.all(P[:, 1] == 0) and np.all(P[:, 2] == 2)
    assert set(P[:, 0].tolist()) <= {0, 2}
    with pytest.raises(mpn.MpnError):
        bp.sample_plan(n_bg, np.zeros(3, np.int32), 9, 4, 0, 2)   # no fg anywhere: the reference would draw forever


def test_training_size_rule_and_max_size_clamp_per_dim():
    assert bp.train_images_size(480, 640, 600, 1000) == (600, 800, 600 / 480)
    h, w, s = bp.train_images_size(400, 1200, 600, 1000)  # dim 2: 1800 > 1000
    assert (h, w) == ref.train_size(400, 1200, 600, 1000)[:2] == (333, 1000) and s == ref.train_size(400, 1200, 600, 1000)[2]
    h, w, s = bp.train_images_size(1300, 500, 600, 1000)  # dim 1 first: 1560 > 1000
    assert (h, w, s) == ref.train_size(1300, 500, 600, 1000) and h == 1000 and w == 384
    r = ref.train_size(333, 517, 600, 1000)
    assert bp.train_images_size(333, 517, 600, 1000) == r and r[1] == int(517 * 600 / 333)


def test_boxes_flip_against_the_truncated_width_and_targets_in_the_label_block():
    mean, std = np.array([0.01, -0.02, 0.1, 0.05], f32), np.array([0.1, 0.12, 0.2, 0.22], f32)
    rois = np.array([[10, 20, 50, 60], [5.5, 7.25, 80, 90], [1, 1, 30, 40]], f32)
    gts = np.array([[0, 0, 0, 0], [6, 8, 82, 88], [2, 3, 28, 44]], f32)
    labels = np.array([1, 3, 2], np.int32)
    h, w, s = ref.train_size(333, 517, 600, 1000)       # im_s width 931.53..., image width 931
    for flip in (0, 1):
        b, t = sample_rows(rois, gts, labels, s, w, flip, mean, std, 4)
        rb, rt = ref.sample_rows(rois, gts, labels, s, w, flip, mean, std, 4)
        assert np.array_equal(b, rb) and np.array_equal(t, rt)
        assert np.all(t[0] == 0) and np.all(t[1, :8] == 0) and np.all(t[1, 12:] == 0) and np.all(t[1, 8:12] != 0)
        assert np.all(t[2, :4] == 0) and np.all(t[2, 8:] == 0)
    b0, _ = sample_rows(rois, gts, labels, s, w, 0, mean, std, 4)
    b1, _ = sample_rows(rois, gts, labels, s, w, 1, mean, std, 4)
    assert np.array_equal(b1[:, 0], (w - b0[:, 2].astype(np.float64) + 1).astype(f32))
    assert np.array_equal(b1[:, 1::2], b0[:, 1::2])
    x = ((f32(10) - f32(1)) * f32(s)) + f32(1)
    assert b0[0, 0] == x


@pytest.mark.parametrize("seed", [3, 4])
def test_random_rows_agree_with_the_restatement(seed):
    rng = np.random.default_rng(seed)
    R, Cn = 200, 81
    x1, y1 = rng.uniform(1, 400, R), rng.uniform(1, 300, R)
    rois = np.stack([x1, y1, x1 + rng.uniform(20, 300, R), y1 + rng.uniform(20, 200, R)], 1).astype(f32)
    gts = (rois + rng.normal(0, 3, (R, 4))).astype(f32)
    labels = rng.integers(1, Cn + 1, R).astype(np.int32)
    mean, std = rng.normal(0, 0.05, 4).astype(f32), rng.uniform(0.1, 0.3, 4).astype(f32)
    for flip in (0, 1):
        b, t = sample_rows(rois, gts, labels, 1.37, 913, flip, mean, std, Cn)
        rb, rt = ref.sample_rows(rois, gts, labels, 1.37, 913, flip, mean, std, Cn)
        assert np.array_equal(b, rb) and np.array_equal(t.view(np.uint32), rt.view(np.uint32))


def test_draws_are_with_replacement_and_in_range():
    u = ref.draw_u32(555, 0, 0, 0, ref.DRAW_BG, np.arange(96))
    pos = ref.rand_int(u, 5)
    assert pos.min() >= 1 and pos.max() <= 5 and len(np.unique(pos)) < 96     # 96 draws of 5 rows: repeats
    assert ref.rand_int([0xFFFFFFFF], 7)[0] == 7 and ref.rand_int([0], 7)[0] == 1

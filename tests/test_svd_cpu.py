"""Host only: models.svd_compress, the truncated-SVD transform of utils.SVDlinear (models/model_utils.lua:56-77), its FLOP
counts and refusals, the import of the graph SVDlinear leaves (nn.LinearNB) by t7 and lua/model_desc.lua, the training
refusal, and the planner's split for the first factors."""
import ctypes
import io
import os
import re

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models, t7, train
from multipathnet_b200._lib import MPN_LAYER_CONV, MPN_LAYER_FLATTEN, MpnError
from multipathnet_b200.t7 import T7Object

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SM = 132                                # H100 SXM


@pytest.fixture(scope="module")
def small():
    spec = models.vgg16_fast_rcnn(21, seed=7, width_div=4, fc_dim=256)
    return spec, models.svd_compress(spec, (128, 64))


def _linears(t):
    """the layers after a tower's FLATTEN"""
    fl = [i for i, L in enumerate(t.layers) if L.kind == MPN_LAYER_FLATTEN][0]
    return t.layers[fl + 1:]


def _chain_ok(t):
    """every layer reads a slot written before it (or the pooled input), and the tower output is written last"""
    seen = {0}
    for L in t.layers:
        assert L.in_slot in seen
        assert L.out_slot not in seen
        seen.add(L.out_slot)
    return t.layers[-1].out_slot == t.out_slot


def test_factors_are_the_best_rank_l_approximation(small):
    spec, svd = small
    before, after = _linears(spec.towers[0]), _linears(svd.towers[0])
    assert len(after) == 4 and _chain_ok(svd.towers[0])
    for k, r in enumerate((128, 64)):
        L, L1, L2 = before[k], after[2 * k], after[2 * k + 1]
        assert (L1.cin, L1.cout, L1.relu, L1.bias) == (L.cin, r, 0, -1)
        assert (L2.cin, L2.cout, L2.relu, L2.bias) == (r, L.cout, L.relu, L.bias)
        W = spec.weights[L.weight].astype(np.float64)
        w1, w2 = svd.weights[L1.weight], svd.weights[L2.weight]
        assert w1.shape == (r, L.cin) and w2.shape == (L.cout, r) and w1.dtype == w2.dtype == np.float32
        u, s, vt = np.linalg.svd(W.T)
        # SVDlinear: L1.W = (U_L diag(S_L))^T, L2.W = V_L; both rounded once to fp32
        np.testing.assert_array_equal(np.abs(w1), np.abs(((u[:, :r] * s[:r]).T).astype(np.float32)))
        np.testing.assert_array_equal(np.abs(w2), np.abs(vt[:r].T.astype(np.float32)))
        err = np.linalg.norm(W - w2.astype(np.float64) @ w1.astype(np.float64))
        best = np.sqrt(np.sum(s[r:] ** 2))
        # fp32 storage of the factors: relative 2^-24 of each entry, ||W|| ~ sqrt(sum s^2)
        assert abs(err - best) <= 1e-6 * np.linalg.norm(s), (err, best)


def test_full_rank_reproduces_w():
    spec = models.vgg16_fast_rcnn(21, seed=3, width_div=8, fc_dim=64)
    L = _linears(spec.towers[0])[1]                       # fc7: 64 -> 64
    svd = models.svd_compress(spec, (0, 64))
    L1, L2 = _linears(svd.towers[0])[1:3]
    W = spec.weights[L.weight].astype(np.float64)
    A = svd.weights[L2.weight].astype(np.float64) @ svd.weights[L1.weight].astype(np.float64)
    assert np.linalg.norm(W - A) <= 1e-6 * np.linalg.norm(W)


def test_input_spec_is_unchanged_and_towers_factor_their_own_weights():
    spec = models.vgg16_multipathnet(21, seed=11, width_div=8, fc_dim=128)
    rng = np.random.default_rng(0)
    t1 = _linears(spec.towers[1])                         # give tower 1 its own fc6
    spec.weights[t1[0].weight] = spec.weights[t1[0].weight] + rng.standard_normal(spec.weights[t1[0].weight].shape).astype(np.float32) * 0.01
    snap = ([np.copy(w) for w in spec.weights], [[vars(L).copy() for L in t.layers] for t in spec.towers], spec.name)
    svd = models.svd_compress(spec, (64, 64))
    assert [vars(L) for t in spec.towers for L in t.layers] == [d for t in snap[1] for d in t] and spec.name == snap[2]
    assert len(spec.weights) == len(snap[0]) and all(np.array_equal(a, b) for a, b in zip(spec.weights, snap[0]))
    f = [_linears(t) for t in svd.towers]
    assert all(len(x) == 4 for x in f) and all(_chain_ok(t) for t in svd.towers)
    idx = [x[0].weight for x in f]
    assert len(set(idx)) == 5                             # every tower has its own factor tensors
    w0, w1, w2 = (svd.weights[i] for i in idx[:3])
    assert not np.array_equal(np.abs(w0), np.abs(w1))     # tower 1's own weights
    np.testing.assert_array_equal(w0, w2)                 # towers 0 and 2 hold the same clone, so the same factors
    for t0, t in zip(spec.towers, svd.towers):            # each tower's product approximates its own fc6
        W = spec.weights[_linears(t0)[0].weight].astype(np.float64)
        L1, L2 = _linears(t)[:2]
        s = np.linalg.svd(W, compute_uv=False)
        err = np.linalg.norm(W - svd.weights[L2.weight].astype(np.float64) @ svd.weights[L1.weight].astype(np.float64))
        assert abs(err - np.sqrt(np.sum(s[64:] ** 2))) <= 1e-6 * np.linalg.norm(s)


def test_flop_counts():
    for spec, towers in ((models.vgg16_fast_rcnn(21, seed=1, width_div=4, fc_dim=256), 1),
                         (models.vgg16_multipathnet(21, seed=1, width_div=8, fc_dim=128), 5)):
        k6 = _linears(spec.towers[0])[0].cin
        f = _linears(spec.towers[0])[1].cout
        svd = models.svd_compress(spec, (128, 64))
        d = models.head_flops_per_roi(spec) - models.head_flops_per_roi(svd)
        saved = 2.0 * (k6 * f - (k6 * 128 + 128 * f)) + 2.0 * (f * f - (f * 64 + 64 * f))
        assert d == towers * saved
        assert models.head_flops_per_roi(models.svd_compress(spec, (0, 64))) == models.head_flops_per_roi(spec) - towers * 2.0 * (f * f - 128 * f)
    # the single-tower w16 Linears of a factored VGG-16: fc6's first factor (25088 -> 1024) only, as csrc/model.cu plans them
    L1 = models.Layer(MPN_LAYER_CONV, 1, 4, cin=25088, cout=1024, bias=-1)
    L2 = models.Layer(MPN_LAYER_CONV, 4, 2, cin=1024, cout=4096, relu=1)
    spec = models.vgg16_fast_rcnn(21, seed=None, fc_dim=256)
    t = spec.towers[0]
    t.layers = [t.layers[0], L1, L2]
    t.out_slot = 2
    assert models.w16_flops_per_roi(spec) == 2.0 * 25088 * 1024


def test_refusals():
    spec = models.vgg16_fast_rcnn(21, seed=None, width_div=4, fc_dim=256)
    for ranks, what in (((100, 0), "multiple of 64"), ((-64, 0), "multiple of 64"), ((0, 0), "nothing to factor"),
                        ((320, 0), "above min"), ((0, 320), "above min"), ((64, 64, 64), "not a Linear")):
        with pytest.raises(ValueError, match=what):
            models.svd_compress(spec, ranks)
    with pytest.raises(ValueError, match="no FLATTEN"):
        models.svd_compress(models.resnet18_fast_rcnn(5, seed=None, integral_k=0, blocks=(1, 1, 1, 1)), (64,))


def _svdlinear(W, b, r):
    """utils.SVDlinear as model_utils.lua:58-77 writes it: Sequential{LinearNB(N, L) = (U_L diag(S_L))^T, Linear(L, K) = V_L, b}"""
    u, s, vt = np.linalg.svd(np.asarray(W, np.float64).T, full_matrices=False)
    l1 = T7Object("nn.LinearNB", {"weight": ((u[:, :r] * s[:r]).T).astype(np.float32)})
    l2 = T7Object("nn.Linear", {"weight": vt[:r].T.astype(np.float32), "bias": np.asarray(b, np.float32)})
    return T7Object("nn.Sequential", {"modules": [l1, l2]})


def _same_graph(a, b):
    for ta, tb in zip(a.towers, b.towers):
        la, lb = [L for L in ta.layers if L.kind == MPN_LAYER_CONV], [L for L in tb.layers if L.kind == MPN_LAYER_CONV]
        assert [(L.cin, L.cout, L.relu, L.bias < 0) for L in la] == [(L.cin, L.cout, L.relu, L.bias < 0) for L in lb]
        for x, y in zip(la, lb):
            assert np.abs(a.weights[x.weight] - b.weights[y.weight].reshape(a.weights[x.weight].shape)).max() <= 1e-6
            if x.bias >= 0:
                np.testing.assert_array_equal(a.weights[x.bias], b.weights[y.bias])


@pytest.mark.parametrize("reader", ["fast_rcnn_from_t7", "model_from_t7"])
def test_svdlinear_top_imports_to_the_same_spec(small, reader):
    spec, svd = small
    g = t7.model_to_t7(spec)
    mods = g.modules
    lin = [i for i, m in enumerate(mods) if m.typename == "nn.Linear"]
    assert len(lin) == 2
    for i, r in zip(lin, (128, 64)):
        mods[i] = _svdlinear(mods[i].weight, mods[i].bias, r)
    buf = io.BytesIO()
    t7.save(buf, g)
    buf.seek(0)
    back = getattr(t7, reader)(t7.load(buf))
    _same_graph(svd, back)
    assert models.head_flops_per_roi(back) == models.head_flops_per_roi(svd)
    assert models.is_svd_compressed(back)


def test_factored_spec_round_trips_through_model_to_t7(small):
    _, svd = small
    buf = io.BytesIO()
    t7.save(buf, t7.model_to_t7(svd))
    buf.seek(0)
    g = t7.load(buf)
    assert [m.typename for m in g.modules].count("nn.LinearNB") == 2
    _same_graph(svd, t7.model_from_t7(g))


def test_linear_without_bias_is_accepted_by_the_flat_reader(small):
    spec, _ = small
    g = t7.model_to_t7(spec)
    i = [k for k, m in enumerate(g.modules) if m.typename == "nn.Linear"][0]
    g.modules[i] = T7Object("nn.Linear", {"weight": g.modules[i].weight})
    back = t7.fast_rcnn_from_t7(g)
    L = _linears(back.towers[0])[0]
    assert L.bias >= 0 and not back.weights[L.bias].any()


def test_trainer_refuses_a_factored_model(small):
    _, svd = small
    with pytest.raises(MpnError, match="SVD-compressed"):
        train.check_spec(svd)
    train.check_spec(small[0])


def test_lua_model_desc_takes_linearnb_without_a_bias():
    src = open(os.path.join(ROOT, "lua", "model_desc.lua")).read()
    m = re.search(r"elseif b == 'Linear' or b == 'LinearNB' then(.*?)\n   elseif", src, re.S)
    assert m, "the Linear branch of model_desc.lua does not take nn.LinearNB"
    body = m.group(1)
    assert re.search(r"local bias = nil\s*\n\s*if b == 'Linear' then bias = ", body)
    assert re.search(r"b = bias\}\)", body)
    assert "if not t then return -1 end" in src                      # widx(nil): no bias -> -1


def _plan(N, K, Cout, per_roi):
    out = (ctypes.c_int32 * 8)()
    assert mpn.load_library().mpn_debug_plan(N, K, 1, 1, Cout, 1, 1, 0, per_roi, SM, out) == 0
    return out[2], out[3]


def test_planner_splits_the_first_factors_and_nothing_else():
    for R in (1, 64, 129, 1000, 2048, 5000):
        assert _plan(R, 25088, 1024, 2) == (256, 4)        # fc6's first factor: 4 N tiles x 4 splits x 8 M tiles at 1000 ROIs
        assert _plan(R, 4096, 256, 2) == (256, 8)          # fc7's first factor: 64 K blocks, 8 per split
        assert _plan(R, 25088, 2048, 2) == (256, 2)
        assert _plan(R, 25088, 4096, 2) == (256, 1)        # full rank: 16 N tiles already fill the SMs
        assert _plan(R, 6272, 192, 2) == (256, 11)       # 12 splits of 9 K blocks leave 11 non-empty
        assert _plan(R, 1024, 4096, 1) == (256, 1) and _plan(R, 256, 4096, 1) == (256, 1)     # second factors: as before
        # the existing per-ROI layers keep the plans tests/test_abi_cpu.py pins
        assert _plan(R, 25088, 4096, 1) == (256, 1) and _plan(R, 4096, 4096, 1) == (256, 1)
        assert _plan(R, 4096, 21, 1) == (64, 8) and _plan(R, 4096, 84, 1) == (128, 8)
        assert _plan(R, 6272, 256, 1) == (256, 1) and _plan(R, 4096, 324, 1) == (256, 1)

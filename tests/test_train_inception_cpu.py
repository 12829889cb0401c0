"""CPU: Inception-v3 Fast R-CNN with fixed batch norm (models.inception_v3_fast_rcnn(fixed_bn=True)): the builder's records
and that fixed_bn=False builds the very model it always did, and the host-only check mpn_train_check_ext (accepts, the
refusals of hand-broken graphs, the unchanged refusal of a model without records, trunk training)."""
import copy
import ctypes as C
import dataclasses
import hashlib

import numpy as np
import pytest

from multipathnet_b200 import models
from multipathnet_b200._lib import (CLayerExt, CTrainOptim, Model, MpnError, MPN_LAYER_CONV, MPN_LAYER_MAXPOOL, load_library)
from multipathnet_b200.train import _train_spec, check_spec


def _digest(spec):
    h = hashlib.sha256()
    for w in spec.weights:
        h.update(np.ascontiguousarray(w, np.float32).tobytes())
    return h.hexdigest()


@pytest.mark.parametrize("args,digest", [
    (dict(num_classes=5, seed=21), "266a9384677abad180f45cea8cbcee198c086e91791a053e28c0e1129cedfb38"),
    (dict(num_classes=81, seed=1234, integral_k=6), "cf96915edefa567c8f89400f91ec721462c6e1c0818a0ce4789cfa7197702dee")])
def test_fixed_bn_false_is_the_model_it_always_was(args, digest):
    """the digests are those of every weight array the builder drew before fixed_bn existed"""
    a, b = models.inception_v3_fast_rcnn(**args), models.inception_v3_fast_rcnn(**args, fixed_bn=False)
    assert _digest(a) == _digest(b) == digest
    assert a.trunk_layers == b.trunk_layers and a.towers == b.towers and a.fixed_bn == b.fixed_bn == {}


def test_fixed_bn_records_every_tower_convolution_and_keeps_the_trunk():
    plain = models.inception_v3_fast_rcnn(5, seed=21)
    spec = models.inception_v3_fast_rcnn(5, seed=21, fixed_bn=True)
    assert spec.trunk_layers == plain.trunk_layers and spec.towers == plain.towers and spec.trunk_train_from == 0
    ntrunk = max(max(L.weight, L.bias) for L in spec.trunk_layers) + 1
    assert all(np.array_equal(x, y) for x, y in zip(spec.weights[:ntrunk], plain.weights[:ntrunk]))
    convs = [L for L in spec.towers[0].layers if L.kind == MPN_LAYER_CONV]
    assert len(convs) == 24 and set(spec.fixed_bn) == {L.weight for L in convs}
    for L in convs:
        a = spec.fixed_bn[L.weight]
        assert a.shape == (L.cout,) and np.all((a >= 0.5) & (a <= 2.0))
        assert L.cin % 64 == 0 and L.cout % 64 == 0


def _check(spec, trunk_from=0, records=None, ext=None):
    """mpn_train_check_ext on spec's description (records: the fixed_bn dict to pass; ext: the records, default the spec's)"""
    lib = load_library()
    d, _keep = Model.build_desc(spec)
    s, _arrays = _train_spec(dataclasses.replace(spec, fixed_bn=spec.fixed_bn if records is None else records), trunk_from, False, False)
    ext = Model.layer_ext(spec) if ext is None else ext
    recs = (CLayerExt * max(len(ext), 1))(*ext)
    msg = C.create_string_buffer(512)
    rc = lib.mpn_train_check_ext(C.byref(d), recs, len(ext), C.byref(s), C.byref(CTrainOptim(0, 0, 0.9, 0.999, 1e-8, 0.99)), msg, len(msg))
    return rc, msg.value.decode()


@pytest.fixture(scope="module")
def spec():
    return models.inception_v3_fast_rcnn(5, seed=None, fixed_bn=True)


def _broken(spec, pick, **change):
    """a copy of spec whose first tower layer with pick(L) takes `change`"""
    s = copy.deepcopy(spec)
    i = next(i for i, L in enumerate(s.towers[0].layers) if pick(L))
    s.towers[0].layers[i] = dataclasses.replace(s.towers[0].layers[i], **change)
    return s, s.towers[0].layers[i]


def test_the_recorded_spec_is_accepted(spec):
    assert _check(spec) == (0, "")
    check_spec(spec)
    check_spec(models.inception_v3_fast_rcnn(81, seed=None, integral_k=6, fixed_bn=True), integral=True)


def test_wrong_pad_per_axis_is_refused(spec):
    s, _ = _broken(spec, lambda L: L.kh == 1 and L.kw == 7, pad_w=2)
    rc, msg = _check(s)
    assert rc != 0 and "pad of (k - 1) / 2 per axis" in msg


def test_cout_off_the_64_grid_is_refused(spec):
    s, _ = _broken(spec, lambda L: L.kh == 7 and L.kw == 1, cout=200)
    rc, msg = _check(s)
    assert rc != 0 and "multiples of 64 channels" in msg


def test_an_unrecorded_1x7_is_refused(spec):
    L = next(L for L in spec.towers[0].layers if L.kh == 1 and L.kw == 7)
    rec = {k: v for k, v in spec.fixed_bn.items() if k != L.weight}
    rc, msg = _check(spec, records=rec)
    assert rc != 0 and "without a fixed-batch-norm record must be a 1x1" in msg


def test_a_max_pool_reading_a_trained_slot_is_refused(spec):
    conv = next(L for L in spec.towers[0].layers if L.kind == MPN_LAYER_CONV and L.in_slot == 0)
    s, _ = _broken(spec, lambda L: L.kind == MPN_LAYER_MAXPOOL, in_slot=conv.out_slot)
    rc, msg = _check(s)
    assert rc != 0 and "max pool" in msg and "not built" in msg


def test_trunk_training_names_the_k_tails(spec):
    rc, msg = _check(spec, trunk_from=5)
    assert rc != 0 and "K tails" in msg and "48, 96, 160" in msg
    with pytest.raises(MpnError, match="K tails"):
        check_spec(spec, trunk_from=5)


def test_without_records_the_refusal_is_unchanged(spec):
    rc, msg = _check(spec, records={})
    assert rc != 0 and "Inception-v3 runs inference only" in msg and "trunk layer 7" in msg
    plain = models.inception_v3_fast_rcnn(5, seed=None)
    with pytest.raises(MpnError, match="Inception-v3.*trunk layer 7"):
        check_spec(plain)


def test_n_ext_0_keeps_the_rules_of_mpn_train_check_optim(spec):
    """without the records the library cannot see the pads per axis: the tower's 1 x 7 is refused as ever"""
    lib = load_library()
    d, _keep = Model.build_desc(spec)
    s, _arrays = _train_spec(spec, 0, False, False)
    a, b = C.create_string_buffer(512), C.create_string_buffer(512)
    o = CTrainOptim(0, 0, 0.9, 0.999, 1e-8, 0.99)
    assert lib.mpn_train_check_optim(C.byref(d), C.byref(s), C.byref(o), a, len(a)) != 0
    assert lib.mpn_train_check_ext(C.byref(d), None, 0, C.byref(s), C.byref(o), b, len(b)) != 0
    assert a.value == b.value and b"fixed-batch-norm layer must be a 1x1 or 3x3" in a.value


def test_model_from_t7_records_const_affine_after_the_towers_bias_free_convolutions():
    """inceptionv3.lua after BNtoFixed: each classifier convolution bias-free, then inn.ConstAffine(a, b); built here from the
    fixed_bn spec's graph (model_to_t7) with every tower convolution so replaced, then read back: the same records"""
    from multipathnet_b200 import t7
    from multipathnet_b200.t7 import T7Object as T
    spec = models.inception_v3_fast_rcnn(5, seed=21, fixed_bn=True)
    convs = [L for L in spec.towers[0].layers if L.kind == MPN_LAYER_CONV]
    by_bytes = {np.asarray(spec.weights[L.weight], np.float32).tobytes(): L for L in convs}
    g = t7.model_to_t7(spec)
    seen = []

    def fixed(m):
        L = by_bytes[np.ascontiguousarray(m.weight, np.float32).tobytes()]
        seen.append(L.weight)
        a = np.asarray(spec.fixed_bn[L.weight], np.float32)
        fields = {k: v for k, v in m.fields.items() if k != "bias"}
        fields["weight"] = (np.asarray(m.weight, np.float64) / a[:, None, None, None]).astype(np.float32)
        return [T(m.typename, fields), T("inn.ConstAffine", dict(a=a, b=np.asarray(spec.weights[L.bias], np.float32)))]

    def walk(m):
        mods = m.get("modules") if isinstance(m, T) else None
        if not mods:
            return
        out = []
        for c in mods:
            if c.typename.endswith("SpatialConvolution") and np.ascontiguousarray(c.weight, np.float32).tobytes() in by_bytes:
                pair = fixed(c)
                out += pair if m.typename == "nn.Sequential" else [T("nn.Sequential", dict(modules=pair))]
            else:
                walk(c)
                out.append(c)
        mods[:] = out
    walk(g)
    assert sorted(seen) == sorted(L.weight for L in convs)
    back = t7.model_from_t7(g, name="inceptionv3.t7")
    bconvs = [L for L in back.towers[0].layers if L.kind == MPN_LAYER_CONV]
    assert [(L.kh, L.kw, L.pad, L.padw, L.stride, L.out_c_off, L.out_c_total) for L in bconvs] == \
           [(L.kh, L.kw, L.pad, L.padw, L.stride, L.out_c_off, L.out_c_total) for L in convs]
    assert set(back.fixed_bn) == {L.weight for L in bconvs}
    for L, M in zip(convs, bconvs):
        assert np.array_equal(back.fixed_bn[M.weight], spec.fixed_bn[L.weight])
        assert np.array_equal(back.weights[M.bias], spec.weights[L.bias])
        np.testing.assert_allclose(back.weights[M.weight], spec.weights[L.weight], rtol=1e-6, atol=1e-7)
    assert not (set(back.fixed_bn) & {L.weight for L in back.trunk_layers}) and back.trunk_train_from == 0
    check_spec(back)

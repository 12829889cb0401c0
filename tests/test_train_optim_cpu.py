"""CPU: train.lua's other optim methods (adam, adamax, adagrad, rmsprop) and learningRateDecay through the host view
mpn_debug_optim, bit for bit against a numpy restatement of csrc/train_rule.cuh's op order; sgd there against
mpn_debug_sgd; the refusals of mpn_train_check_optim and check_spec; three-state checkpoints and the optim fingerprint."""
import ctypes as C
import math
import types

import numpy as np
import pytest

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from multipathnet_b200._lib import CTrainConfig, CTrainOptim
from multipathnet_b200.train import Trainer, _train_optim, check_spec

pytestmark = pytest.mark.filterwarnings("ignore:overflow encountered:RuntimeWarning")   # the huge gradients' g * g
f32 = np.float32
METHODS = ("sgd", "adam", "adamax", "adagrad", "rmsprop")


def _fma(a, b, c):
    """one fmaf, computed exactly in long double and rounded once to fp32"""
    L = np.longdouble
    return (L(a) * L(b) + L(c)).astype(f32)


def _scalars(o: CTrainOptim, lr, wd, t):
    """mpn_optim_scalars: doubles from the fp32 rate, rounded once"""
    T, lr = t + 1.0, float(f32(lr))
    clr = lr / (1.0 + t * o.lr_decay)
    h = dict(lr=f32(clr), wd=f32(wd), b1=f32(o.beta1), c1=f32(1.0 - o.beta1), b2=f32(o.beta2), c2=f32(1.0 - o.beta2), eps=f32(o.epsilon))
    if o.method == 1:
        h["lr"] = f32(clr * math.sqrt(1.0 - o.beta2 ** T) / (1.0 - o.beta1 ** T))
    elif o.method == 2:
        h["lr"] = f32(lr / (1.0 - o.beta1 ** T))
    elif o.method == 3:
        h["eps"] = f32(1e-10)
    elif o.method == 4:
        h.update(lr=f32(lr), b2=f32(o.alpha), c2=f32(1.0 - o.alpha))
    return h


def _dir(method, g, s1, s2, h):
    if method == 1:
        s1 = _fma(h["c1"], g, h["b1"] * s1)
        s2 = _fma(h["c2"], g * g, h["b2"] * s2)
        return s1 / (np.sqrt(s2) + h["eps"]), s1, s2
    if method == 2:
        s1 = _fma(h["c1"], g, h["b1"] * s1)
        s2 = np.maximum(h["b2"] * s2, np.abs(g) + h["eps"])
        return s1 / s2, s1, s2
    s1 = _fma(g, g, s1) if method == 3 else _fma(h["c2"], g * g, h["b2"] * s1)
    return g / (np.sqrt(s1) + h["eps"]), s1, s2


def restate(o, w, g, s1, s2, a, lr, wd, t, momentum=0.9, dampening=0.0):
    """csrc/train_rule.cuh's op order in numpy fp32 (g None: the no-gradient variant; a: fixed-batch-norm scales)"""
    w, s1, s2 = (np.array(x, f32) for x in (w, s1, s2))
    g = np.zeros_like(w) if g is None else np.asarray(g, f32)
    h = _scalars(o, lr, wd, t)
    if o.method == 0:
        gg = (a * a) * g if a is not None else g
        gg = _fma(h["wd"], w, gg) if wd != 0 else gg
        if momentum != 0:
            s1 = gg.copy() if t == 0 else _fma(f32(momentum), s1, f32(1.0 - f32(dampening)) * gg)
            gg = s1
        return _fma(-h["lr"], gg, w), s1, s2
    if a is None:
        gg = _fma(h["wd"], w, g) if wd != 0 else g
        q, s1, s2 = _dir(o.method, gg, s1, s2, h)
        return _fma(-h["lr"], q, w), s1, s2
    gw = a * g
    gg = _fma(h["wd"], w / a, gw) if wd != 0 else gw
    q, s1, s2 = _dir(o.method, gg, s1, s2, h)
    return _fma(-a, h["lr"] * q, w), s1, s2


def device_rule(o, w, g, s1, s2, a, lr, wd, t, momentum=0.9, dampening=0.0):
    lib = mpn.load_library()
    w, s1, s2 = (np.array(x, f32) for x in (w, s1, s2))
    keep = [None if x is None else np.ascontiguousarray(x, f32) for x in (g, a)]
    p = lambda x: None if x is None else x.ctypes.data          # noqa: E731
    assert lib.mpn_debug_optim(p(w), p(keep[0]), p(s1), p(s2), p(keep[1]), w.size, C.byref(o), lr, momentum, dampening, wd, t) == 0
    return w, s1, s2


def _case(seed, n=4096):
    rng = np.random.default_rng(seed)
    w = rng.standard_normal(n).astype(f32) * f32(0.05)
    gs = []
    for k in range(6):
        g = rng.standard_normal(n).astype(f32) * f32(10.0 ** rng.uniform(-4, 0))
        g[:64] = 0.0                                               # zeros
        g[64:128] = rng.standard_normal(64).astype(f32) * f32(1e-30)  # tiny: g * g underflows, subnormal states
        g[128:160] = rng.standard_normal(32).astype(f32) * f32(1e19)  # huge: g * g overflows in fp32
        gs.append(g)
    a = rng.standard_normal(n).astype(f32)
    a[np.abs(a) < 0.05] = f32(0.5)
    a[:8] = -np.abs(a[:8])                                         # negative scales
    return w, gs, a


def _eq(x, y):
    return np.array_equal(x.view(np.uint32), y.view(np.uint32))


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("variant", ["plain", "no_grad", "fixed"])
@pytest.mark.parametrize("wd", [0.0, 5e-4])
def test_host_view_matches_the_numpy_restatement_bit_for_bit(method, variant, wd):
    lrd = 0.0 if method in ("adamax", "rmsprop") else 1e-2          # lr_decay where it applies (the others ignore it)
    o = _train_optim(method, lr_decay=lrd)
    w, gs, a = _case(METHODS.index(method) * 10 + ["plain", "no_grad", "fixed"].index(variant) * 2 + int(wd > 0))
    a = a if variant == "fixed" else None
    dev = ref = (w, np.zeros_like(w), np.zeros_like(w))
    for t, g in enumerate(gs):
        g = None if variant == "no_grad" else g
        lr = f32(1e-3) if t < 4 else f32(1e-4)                      # a decay between steps
        dev = device_rule(o, *dev[:1], g, *dev[1:], a, lr, wd, t)
        ref = restate(o, *ref[:1], g, *ref[1:], a, lr, wd, t)
        for x, y in zip(dev, ref):
            assert _eq(x, y), (method, variant, t)
    assert np.isfinite(dev[0]).all() or method == "sgd"
    if variant == "no_grad" and wd > 0 and method != "sgd":
        assert not np.array_equal(dev[0], w)                      # an idle head keeps moving under weight decay


def test_sgd_through_the_optim_view_is_mpn_debug_sgd():
    lib = mpn.load_library()
    w, gs, _ = _case(7)
    o = _train_optim("sgd")
    a = (w.copy(), np.zeros_like(w))
    b = (w.copy(), np.zeros_like(w))
    for t, g in enumerate(gs):
        a = device_rule(o, a[0], g, a[1], np.zeros_like(w), None, f32(1e-3), 5e-4, t)[:2]
        w2, b2 = b[0].copy(), b[1].copy()
        assert lib.mpn_debug_sgd(w2.ctypes.data, g.ctypes.data, b2.ctypes.data, w.size, f32(1e-3), 0.9, 0.0, 5e-4, int(t == 0)) == 0
        b = (w2, b2)
        assert _eq(a[0], b[0]) and _eq(a[1], b[1])


def test_adamax_zero_gradient_gives_the_subnormal_epsilon_and_a_finite_step():
    o = _train_optim("adamax")
    z = np.zeros(16, f32)
    w, m, u = device_rule(o, np.ones(16, f32), z, z, z, None, f32(2e-3), 0.0, 0)
    assert np.all(u == f32(1e-38)) and u[0] != 0 and u[0] < np.finfo(f32).tiny      # subnormal, not flushed
    assert np.all(m == 0) and np.all(w == 1.0)


def test_sgd_with_lr_decay_uses_clr():
    o = _train_optim("sgd", lr_decay=0.5)
    w = np.ones(8, f32)
    g = np.full(8, 2.0, f32)
    got = device_rule(o, w, g, np.zeros(8, f32), np.zeros(8, f32), None, f32(1e-2), 0.0, 3, momentum=0.0)[0]
    assert _eq(got, _fma(-f32(1e-2 / 2.5), g, w))


def _desc_spec():
    return models.vgg16_fast_rcnn(21, seed=None, width_div=16, fc_dim=64)


def test_refusals_without_a_gpu():
    spec = _desc_spec()
    with pytest.raises(mpn.MpnError, match="unknown optim method 'adamw'"):
        check_spec(spec, optim={"method": "adamw"})
    with pytest.raises(mpn.MpnError, match="nag.*fEvalMod"):
        check_spec(spec, optim={"method": "nag"})
    with pytest.raises(mpn.MpnError, match="adadelta.*1000x"):
        check_spec(spec, optim={"method": "adadelta"})
    for m in ("asgd", "rprop", "lbfgs", "cg", "cmaes"):
        with pytest.raises(mpn.MpnError, match="refused"):
            check_spec(spec, optim={"method": m})
    for kw, what in ((dict(beta1=1.0), "beta1"), (dict(beta2=-0.1), "beta2"), (dict(alpha=1.5), "alpha"), (dict(epsilon=-1.0), "epsilon"),
                     (dict(lr_decay=-1e-3), "lr_decay"), (dict(epsilon=float("inf")), "epsilon")):
        with pytest.raises(mpn.MpnError, match=what):
            check_spec(spec, optim=dict(method="adam", **kw))
    for m in METHODS:
        check_spec(spec, optim={"method": m, "lr_decay": 1e-4})
    check_spec(spec, optim={"method": "rmsprop", "alpha": 1.0, "beta1": 0.0})
    # the library's own check: a method out of range; the optimiser is checked before the graph
    lib = mpn.load_library()
    d, _keep = mpn.Model.build_desc(models.vgg16_fast_rcnn(21, seed=None, width_div=16, fc_dim=64, integral_k=3))
    from multipathnet_b200.train import _train_spec
    s, _arrays = _train_spec(models.vgg16_fast_rcnn(21, seed=None, width_div=16, fc_dim=64, integral_k=3), 0, False, False)
    msg = C.create_string_buffer(256)
    assert lib.mpn_train_check_optim(C.byref(d), C.byref(s), C.byref(CTrainOptim(5, 0, 0.9, 0.999, 1e-8, 0.99)), msg, 256) != 0
    assert b"method out of range" in msg.value
    assert lib.mpn_train_check_optim(C.byref(d), C.byref(s), None, msg, 256) != 0 and b"integral head" in msg.value
    assert lib.mpn_train_check(C.byref(d), C.byref(s), msg, 256) != 0 and b"integral head" in msg.value


class _Recorder:
    def __init__(self, n):
        self.n = n

    def state_dict(self):
        ts = tuple(np.full((2, 3), k, np.float32) for k in range(self.n))
        return {"fingerprint": {"name": "rec", "optim": {"method": "adam"}}, "config": {}, "state": {"steps": 1}, "tensors": {5: ts}}


@pytest.mark.parametrize("n", [2, 3])
def test_checkpoint_files_keep_two_or_three_tensors(tmp_path, n):
    path = str(tmp_path / "c.npz")
    mpn.save_checkpoint(path, _Recorder(n))
    with np.load(path) as z:
        assert ("c5" in z.files) == (n == 3)
    d = mpn.load_checkpoint(path)
    assert len(d["tensors"][5]) == n and d["fingerprint"]["optim"] == {"method": "adam"}
    for k, a in enumerate(d["tensors"][5]):
        assert a.dtype == np.float32 and np.all(a == k)


def _offline(spec, method="sgd", **optim):
    """a Trainer as its constructor leaves it for load_state_dict's checks, without a device"""
    t = Trainer.__new__(Trainer)
    t.model = types.SimpleNamespace(spec=spec)
    t.cfg = CTrainConfig(1e-3, 0.9, 0.0, 5e-4, 0.5, 1.0, 555)
    t.trunk_from, t.phase2, t.phase = 0, False, 1
    t.trained = sorted(t._trained_indices())
    t._fingerprint = {"name": spec.name, "shapes": [list(np.shape(w)) for w in spec.weights], "trained": list(t.trained), "trunk_from": 0,
                      "phase2_from": 0, "integral_k": len(spec.cls_heads), "fixed_bn": sorted(spec.fixed_bn)}
    if method != "sgd" or optim:
        t.method = method
        o = _train_optim(method, **optim)
        t._fingerprint["optim"] = dict({k: getattr(o, k) for k, _ in CTrainOptim._fields_ if k != "method"}, method=method)
    return t


def _ckpt(t):
    return {"fingerprint": dict(t._fingerprint), "config": {k: getattr(t.cfg, k) for k, _ in CTrainConfig._fields_},
            "state": {"step": 0, "lr": 1e-3, "head": 0, "last_head": 0, "phase2": 0, "steps": 0}, "tensors": {}}


def test_a_checkpoint_of_another_method_or_setting_is_refused():
    spec = _desc_spec()
    sgd, adam = _offline(spec), _offline(spec, "adam")
    with pytest.raises(mpn.MpnError, match="optim is sgd with lr_decay 0, this trainer's .*adam"):
        adam.load_state_dict(_ckpt(sgd))
    with pytest.raises(mpn.MpnError, match="optim is .*adam.*this trainer's sgd with lr_decay 0"):
        sgd.load_state_dict(_ckpt(adam))
    with pytest.raises(mpn.MpnError, match="optim"):
        _offline(spec, "adam", beta1=0.8).load_state_dict(_ckpt(adam))
    with pytest.raises(mpn.MpnError, match="optim"):
        sgd.load_state_dict(_ckpt(_offline(spec, "sgd", lr_decay=1e-4)))
    # the same method passes the fingerprint; a two-tensor entry is refused by a two-state method
    with pytest.raises(mpn.MpnError, match="holds tensors"):
        adam.load_state_dict(_ckpt(adam))
    two = {i: (np.zeros(np.shape(spec.weights[i]), f32),) * 2 for i in adam.trained}
    with pytest.raises(mpn.MpnError, match="1 optim states in the checkpoint, adam keeps 2"):
        adam.load_state_dict(dict(_ckpt(adam), tensors=two))

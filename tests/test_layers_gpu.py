"""Every layer of every model graph against fp64 on its own device inputs, in each inference numerics (teacher forcing).

After one detect_nms on the product plan (conv_impl 0, as bench.py runs it), the planes each layer read and wrote are
read back (mpn_model_get_slot_planes, mpn_model_get_head_outputs) and the layer is recomputed in fp64 from the read
planes with the operand rule of the numerics (tests/_layer_ref.py). The error then does not grow with depth, and every
layer is held to the per-GEMM bar of the engine tests:

  rule                                      bar (normwise, max|a - b| / max|ref|)
  default (hi + lo x fp32 weight), heads    1e-4, 2e-4 for K > 4608 (fp32 accumulation over 1568 k16 steps)
  w16 (fc6 / fc7 of single-tower graphs)    3e-5 vs the w16 emulation for K <= 4096, 2e-4 above; 3e-4 vs exact fp64
  bf16 (hi x rn_bf16(w))                    1e-5, 5e-5 for K > 4608
  fp8 (e4m3 per sample / per channel)       1e-4
  + 2^-17 on the w16 / bf16 / fp8 layers whose output is stored as split planes (the re-split's own rounding)
  max pool                                  bit-equal values to the window max of the read-back input (an unfused pool)
  fused conv + 2x2 pool                     the conv's bar on max(ReLU(fp64 conv)) against the pool output
  avgpool                                   1e-6 + 2^-17

Full-size maps are row-sampled (borders, 16-row patch edges, the middle, seeded rows; ROI rows at the 128-row tile
edges and seeded); the small graphs are checked on every element. Negative controls show the bars pin the numerics:
against the nearest wrong operand rule, the first layer the rule covers and fc6 are outside the bar (ResNet: against
the residual left out; fp8's per-tensor exponent is recorded only, see per_roi_control). The fp8 quantizer is
checked bit for bit at model scale on every slot the plan quantizes, and the fp16 plane formats on the slots the w16 rule
names. Options are set in try / finally, as in test_fp8_gpu.py."""
import contextlib
import ctypes as C

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import multipathnet_b200 as mpn
from multipathnet_b200 import models
from multipathnet_b200._lib import MPN_LAYER_AVGPOOL, MPN_LAYER_CONV, MPN_LAYER_FLATTEN, MPN_LAYER_MAXPOOL
from conftest import rel_err, record_parity
from test_model_gpu import _inputs
import _fp8_oracle as F8
import _layer_ref as LR

pytestmark = pytest.mark.gpu
SPLIT = 2.0 ** -17


@contextlib.contextmanager
def options(ctx, opts):
    for k, v in opts.items():
        ctx.set_option(k, v)
    try:
        yield
    finally:
        for k in opts:
            ctx.set_option(k, -1)


# name -> (spec builder, H, W, R, input seed, sharpmask boxes, model limits, row-sampled)
SMALL = dict(max_rois=256, max_h=256, max_w=320)
GRAPHS = {
    "vgg_small": (lambda: models.vgg16_fast_rcnn(21, seed=7, width_div=4, fc_dim=256), 150, 203, 200, 2, False, SMALL, False),
    "vgg_small_fc1024": (lambda: models.vgg16_fast_rcnn(21, seed=7, width_div=4, fc_dim=1024), 150, 203, 200, 2, False, SMALL, False),
    "mpn_small": (lambda: models.vgg16_multipathnet(21, seed=11, width_div=4, fc_dim=256), 160, 208, 128, 6, True, SMALL, False),
    "mpn_small_integral": (lambda: models.vgg16_multipathnet(21, seed=11, width_div=4, fc_dim=256, integral_k=2), 160, 208, 128, 6, True,
                           SMALL, False),
    "resnet_small": (lambda: models.resnet50_fast_rcnn(21, seed=5, integral_k=3), 160, 224, 48, 8, True, SMALL, False),
    "cfg2": (lambda: models.vgg16_fast_rcnn(21, seed=1234), 600, 800, 1000, 2, False, dict(max_rois=1048, max_h=608, max_w=800), True),
    "cfg3": (lambda: models.vgg16_multipathnet(81, seed=1234), 600, 800, 1000, 3, True, dict(max_rois=1048, max_h=608, max_w=800), True),
    "cfg4": (lambda: models.resnet50_fast_rcnn(81, seed=1234, integral_k=6), 800, 1000, 2000, 4, True,
             dict(max_rois=2048, max_h=808, max_w=1000), True),
}
NUMERICS = {"default": {}, "w16_off": {"fc_w16": 0}, "bf16": {"bf16": 1}, "fp8": {"fp8": 1}}
W16_GRAPHS = ("vgg_small_fc1024", "cfg2")          # single-tower graphs with a Linear the w16 rule takes
CASES = [(g, n) for g in GRAPHS for n in NUMERICS if n != "w16_off" or g in W16_GRAPHS]

# the nearest wrong operand rules of each rule (negative controls)
# (fp8's per-tensor instead of per-ROI exponent: per_roi_control below)
WRONG = {"exact": ("bf16_of_exact",), "bf16": ("exact",), "fp8": ("bf16",), "w16": ("w16_bf16w",)}


def conv_bar(rule, K, split_out):
    if rule in ("exact", "first"):
        return 1e-4 if K <= 4608 else 2e-4            # K = 25088: the tensor pipe's fp32 accumulation (DESIGN 4)
    if rule == "w16":
        base = 3e-5 if K <= 4096 else 2e-4
    elif rule == "bf16":
        base = 1e-5 if K <= 4608 else 5e-5
    else:
        base = 1e-4
    return base + (SPLIT if split_out else 0.0)


class Slot:
    """read-back planes of one slot: hi / lo values as fp32 N x C x H x W torch tensors (+ the raw planes)"""

    def __init__(self, p):
        self.raw, self.fmt, self.dims = p, p["fmt"], p["dims"]
        self.hi_nhwc = LR.plane_values(p["hi"], self.fmt)
        self.lo_nhwc = LR.plane_values(p["lo"], self.fmt)
        self.hi, self.lo = LR.nhwc_to_nchw(self.hi_nhwc), LR.nhwc_to_nchw(self.lo_nhwc)

    def value(self):
        return self.hi.double() + self.lo.double()


def _runs(rows):
    out, a = [], rows[0]
    for i in range(1, len(rows) + 1):
        if i == len(rows) or rows[i] != rows[i - 1] + 1:
            out.append((a, rows[i - 1] + 1))
            if i < len(rows):
                a = rows[i]
    return out


def read_slot(m, tower, slot, rows=None, fp8=False):
    if rows is None:
        return Slot(m.slot_planes(tower, slot, fp8=fp8))
    parts = [m.slot_planes(tower, slot, a, b - a, fp8=fp8) for a, b in _runs(rows)]
    p = dict(parts[0])
    for k in ("hi", "lo", "q8", "e8"):
        if k in p:
            p[k] = np.concatenate([q[k] for q in parts])
    return Slot(p)


def _is_elided(m, slot):
    try:
        m.slot_planes(-1, slot)
        return False
    except mpn.MpnError as e:
        assert "fused" in str(e), str(e)
        return True


def expected_w16_slots(spec, t, numerics):
    """tower slots plan_heads stores as fp16 planes: the input of a per-ROI Linear on a 1 x 1 map with >= 2048 inputs and
    >= 1024 outputs (and the FLATTEN's input in front of it), single-tower graphs, default numerics only"""
    if numerics != "default" or len(spec.towers) != 1:
        return set()
    T = spec.towers[t]
    shp, s = {0: (T.pooled_h, T.pooled_w)}, set()
    for L in T.layers:
        h, w = shp[L.in_slot]
        if L.kind == MPN_LAYER_CONV:
            ho, wo = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1
            if (h, w) == (1, 1) and L.kh == 1 and L.pad == 0 and L.residual_slot < 0 and L.cin >= 2048 and L.cout >= 1024:
                s.add(L.in_slot)
            shp[L.out_slot] = (ho, wo)
        else:
            shp[L.out_slot] = (1, 1)
    for L in T.layers:
        if L.kind == MPN_LAYER_FLATTEN and L.out_slot in s:
            s.add(L.in_slot)
    s.discard(T.out_slot)
    return s


class Walk:
    """the checks of one (graph, numerics) run: every result is recorded, failures collected with their location"""

    def __init__(self, graph, numerics):
        self.graph, self.numerics, self.fails, self.worst = graph, numerics, [], {}

    def check(self, layer, got, ref, bar, rows=None, per_roi=False, note=""):
        got, ref = got.double(), ref.double()
        assert got.shape == ref.shape, (layer, tuple(got.shape), tuple(ref.shape))
        err = rel_err(got.numpy(), ref.numpy())
        record_parity("layer", graph=self.graph, numerics=self.numerics, layer=layer, error=err, bar=bar)
        self.worst[layer] = (err, bar)
        if not err < bar:
            d = (got - ref).abs()
            idx = np.unravel_index(int(torch.argmax(d)), tuple(d.shape))
            n, c = int(idx[0]), int(idx[1])
            h, w = (int(idx[2]), int(idx[3])) if len(idx) == 4 else (0, 0)
            if rows is not None:
                n, h = (rows[n], h) if per_roi else (n, rows[h])
            self.fails.append(f"{self.graph} / {self.numerics} / {layer}{note}: error {err:.3e} >= bar {bar:.3e}; worst element "
                              f"(n, c, h, w) = ({n}, {c}, {h}, {w}), 16 x 8 patch ({h // 16}, {w // 8}), 128-wide N tile {c // 128}: "
                              f"device {float(got[idx]):.8g} vs {float(ref[idx]):.8g}")
        return err

    def outside(self, layer, what, err, bar):
        record_parity("layer_control", graph=self.graph, numerics=self.numerics, layer=layer, control=what, error=err, bar=bar)
        if not err > bar:
            self.fails.append(f"{self.graph} / {self.numerics} / {layer}: negative control '{what}' is inside the bar "
                              f"({err:.3e} <= {bar:.3e}): the bar does not pin the numerics")


def _w(spec, idx):
    return torch.from_numpy(np.ascontiguousarray(spec.weights[idx], np.float32))


def _bias(spec, L):
    return _w(spec, L.bias).double() if L.bias >= 0 else None


def walk_trunk(walk, m, spec, img, numerics, sampled, rng):
    rule = {"default": "exact", "w16_off": "exact", "bf16": "bf16", "fp8": "fp8"}[numerics]
    slots, elided = {}, set()
    image = torch.from_numpy(np.ascontiguousarray(img, np.float32))[None].double()
    first_covered = None
    layers = spec.trunk_layers
    skip = set()
    for i, L in enumerate(layers):
        if i in skip:
            continue
        if L.out_slot not in slots and L.out_slot not in elided:
            if _is_elided(m, L.out_slot):
                elided.add(L.out_slot)
            else:
                slots[L.out_slot] = read_slot(m, -1, L.out_slot)
        name = f"trunk[{i}]"
        if L.kind == MPN_LAYER_CONV:
            H = image.shape[2] if L.in_slot == 0 else slots[L.in_slot].hi.shape[2]
            if L.in_slot == 0:
                lrule, x = "first", None
            else:
                lrule, x = rule, slots[L.in_slot]
            w4 = _w(spec, L.weight).reshape(L.cout, L.cin, L.kh, L.kw)
            K = L.cin * L.kh * L.kw

            def ref_fn(r, with_res=True, rows=None, pool=False, L=L, x=x, w4=w4, H=H):
                if x is None:
                    get, wt = (lambda a, b: image[:, :, a:b]), w4.double()
                else:
                    e = LR.act_exponents(r, x.hi)
                    get = lambda a, b: LR.act_operand(r, x.hi[:, :, a:b], x.lo[:, :, a:b], e)
                    wt = LR.weight_operand(r, w4)
                if pool:
                    return LR.conv_pool_rows(get, H, wt, _bias(spec, L), L.pad, L.relu, rows)
                y = LR.conv_rows(get, H, wt, _bias(spec, L), L.stride, L.pad, rows)
                if L.residual_slot >= 0 and with_res:
                    y = y + slots[L.residual_slot].value()[:, :, rows]
                return F.relu(y) if L.relu else y

            if L.out_slot in elided:              # conv + pool fused, the conv's output never written: check the pair
                P = layers[i + 1]
                assert P.kind == MPN_LAYER_MAXPOOL and P.in_slot == L.out_slot, f"{name}: an elided slot not read by a pool"
                skip.add(i + 1)
                slots[P.out_slot] = out = read_slot(m, -1, P.out_slot)
                Hp = out.hi.shape[2]
                rows = LR.trunk_rows(Hp, rng) if sampled else list(range(Hp))
                bar = conv_bar(lrule, K, True)
                ref = ref_fn(lrule, rows=rows, pool=True)
                walk.check(name + "+pool", out.value()[:, :, rows], ref, bar, rows)
                unit = dict(name=name + "+pool", got=out.value()[:, :, rows], fn=lambda r, wr=True, f=ref_fn, rw=rows: f(r, wr, rw, True),
                            bar=bar, res=False)
            else:
                out = slots[L.out_slot]
                Ho = out.hi.shape[2]
                rows = LR.trunk_rows(Ho, rng) if sampled else list(range(Ho))
                bar = conv_bar(lrule, K, True)
                walk.check(name, out.value()[:, :, rows], ref_fn(lrule, rows=rows), bar, rows)
                unit = dict(name=name, got=out.value()[:, :, rows], fn=lambda r, wr=True, f=ref_fn, rw=rows: f(r, wr, rw),
                            bar=bar, res=L.residual_slot >= 0)
            if lrule != "first" and first_covered is None:
                first_covered = unit
            if unit["res"] and "residual" not in walk.worst:
                walk.worst["residual"] = True
                walk.outside(unit["name"], "residual left out", rel_err(unit["got"].numpy(), unit["fn"](lrule, False).numpy()), unit["bar"])
        elif L.kind == MPN_LAYER_MAXPOOL:
            x, out = slots[L.in_slot], slots[L.out_slot]
            H, Ho = x.hi.shape[2], out.hi.shape[2]
            rows = LR.trunk_rows(Ho, rng) if sampled else list(range(Ho))
            xv = (x.hi + x.lo)                                           # the fp32 value the pool kernel compares
            want = LR.maxpool_rows(lambda a, b: xv[:, :, a:b], H, L.kh, L.stride, L.pad, L.ceil_mode, rows)
            got = (out.hi + out.lo)[:, :, rows]
            if torch.equal(got, want):
                walk.check(name, got, want, 1e-30, rows)
                continue
            # not bit-equal: only a pool fused into its conv's epilogue (pooling the fp32 accumulator) may differ
            Pc = layers[i - 1] if i > 0 else None
            fusable = (Pc is not None and Pc.kind == MPN_LAYER_CONV and Pc.out_slot == L.in_slot and Pc.kh == 3 and Pc.stride == 1
                       and L.kh == 2 and L.stride == 2 and L.pad == 0 and Pc.in_slot != 0)
            if not fusable:
                walk.check(name, got, want, 1e-30, rows)
                continue
            xin = slots[Pc.in_slot]
            e = LR.act_exponents(rule, xin.hi)
            get = lambda a, b: LR.act_operand(rule, xin.hi[:, :, a:b], xin.lo[:, :, a:b], e)
            ref = LR.conv_pool_rows(get, xin.hi.shape[2], LR.weight_operand(rule, _w(spec, Pc.weight).reshape(Pc.cout, Pc.cin, 3, 3)),
                                    _bias(spec, Pc), Pc.pad, Pc.relu, rows)
            walk.check(name + " (fused)", out.value()[:, :, rows], ref, conv_bar(rule, Pc.cin * 9, True), rows)
    return slots, elided, first_covered


def tower_rule(numerics, fmt):
    if numerics == "bf16":
        return "bf16"
    if numerics == "fp8":
        return "fp8"
    return "w16" if fmt == 1 else "exact"


def walk_towers(walk, m, spec, numerics, R, sampled, rng):
    rows = LR.roi_rows(R, rng) if sampled else list(range(R))
    outs, fc6, spread = [], None, None
    for t, T in enumerate(spec.towers):
        slots, flat = {0: read_slot(m, t, 0, rows)}, {}
        want16 = expected_w16_slots(spec, t, numerics)
        for li, L in enumerate(T.layers):
            name = f"tower{t}[{li}]"
            if L.out_slot not in slots:
                slots[L.out_slot] = read_slot(m, t, L.out_slot, rows)
            x, out = slots[L.in_slot], slots[L.out_slot]
            if L.kind == MPN_LAYER_FLATTEN:
                flat[L.out_slot] = x
                assert np.array_equal(out.raw["hi"].reshape(len(rows), -1), x.raw["hi"].reshape(len(rows), -1)), name
                continue
            if L.kind == MPN_LAYER_AVGPOOL:
                walk.check(name + " avgpool", out.value(), x.value().mean(dim=(2, 3), keepdim=True), 1e-6 + SPLIT, rows, True)
                continue
            if L.kind == MPN_LAYER_MAXPOOL:
                xv = x.hi + x.lo
                want = F.max_pool2d(xv, L.kh, L.stride, L.pad, ceil_mode=bool(L.ceil_mode))
                walk.check(name, out.hi + out.lo, want, 1e-30, rows, True)
                continue
            assert (x.fmt == 1) == (L.in_slot in want16), f"{name}: input plane format {x.fmt}"
            if L.in_slot in flat:                     # (ph, pw, c) rows -> Torch's (c, ph, pw)
                src = flat[L.in_slot]
                hi = LR.flatten_nhwc_to_torch(torch.from_numpy(src.hi_nhwc))[:, :, None, None]
                lo = LR.flatten_nhwc_to_torch(torch.from_numpy(src.lo_nhwc))[:, :, None, None]
                w4 = _w(spec, L.weight).reshape(L.cout, -1, 1, 1)
            else:
                hi, lo = x.hi, x.lo
                w4 = _w(spec, L.weight).reshape(L.cout, L.cin, L.kh, L.kw)
            K = w4[0].numel()
            rule = tower_rule(numerics, x.fmt)

            def ref_fn(r, with_res=True, L=L, hi=hi, lo=lo, w4=w4, slots=slots):
                y = F.conv2d(LR.act_operand(r, hi, lo, LR.act_exponents(r, hi)), LR.weight_operand(r, w4), _bias(spec, L),
                             stride=L.stride, padding=L.pad)
                if L.residual_slot >= 0 and with_res:
                    y = y + slots[L.residual_slot].value()
                return F.relu(y) if L.relu else y

            split = out.fmt == 0
            bar = conv_bar(rule, K, split)
            got = out.value()
            walk.check(name, got, ref_fn(rule), bar, rows, True)
            if rule == "w16":
                walk.check(name + " vs exact", got, ref_fn("exact"), 3e-4 + (SPLIT if split else 0.0), rows, True)
            if t == 0 and fc6 is None and (L.in_slot in flat or not any(q.kind == MPN_LAYER_FLATTEN for q in T.layers)):
                fc6 = dict(name=name, got=got, fn=ref_fn, bar=bar, rule=rule)
            if rule == "fp8":                      # the fp8 layer whose sampled ROIs spread widest over exponents
                e = LR.act_exponents("fp8", hi)
                if spread is None or int(e.max() - e.min()) > int(spread["e"].max() - spread["e"].min()):
                    spread = dict(name=name, got=got, fn=ref_fn, bar=bar, e=e)
        outs.append(slots[T.out_slot])
    return rows, outs, fc6, spread


def walk_heads(walk, m, spec, numerics, rows, outs):
    hi = torch.cat([o.hi.reshape(len(rows), -1) for o in outs], 1)
    lo = torch.cat([o.lo.reshape(len(rows), -1) for o in outs], 1)
    cls, bbox = m.head_outputs()
    rule = "bf16" if numerics == "bf16" else "exact"
    heads = [(f"cls{k}", h, torch.from_numpy(cls[k][rows])) for k, h in enumerate(spec.cls_heads)]
    heads.append(("bbox", spec.bbox_head, torch.from_numpy(bbox[rows])))
    for name, h, got in heads:
        A = LR.act_operand(rule, hi[:, h.col_begin:h.col_begin + h.col_len], lo[:, h.col_begin:h.col_begin + h.col_len])
        ref = F.linear(A, LR.weight_operand(rule, _w(spec, h.weight)), _w(spec, h.bias).double())
        walk.check(name, got, ref, conv_bar(rule, h.col_len, False), rows, True)


def check_quantizer(walk, m, spec, numerics, R, rows):
    """fp8: every slot the plan quantizes holds q8 / e8 == _fp8_oracle.quantize of its hi plane, bit for bit, and exactly
    the fp8 layers' inputs have e4m3 planes"""
    trunk_want = {L.in_slot for L in spec.trunk_layers if L.kind == MPN_LAYER_CONV and L.in_slot != 0} if numerics == "fp8" else set()
    trunk_slots = {L.out_slot for L in spec.trunk_layers}
    got = set()
    for s in sorted(trunk_slots):
        if _is_elided(m, s):
            assert s not in trunk_want
            continue
        try:
            p = m.slot_planes(-1, s, fp8=True)
        except mpn.MpnError:
            continue
        got.add(s)
        _quant_equal(walk, f"trunk slot {s}", p)
    assert got == trunk_want, (got, trunk_want)
    for t, T in enumerate(spec.towers):
        want = {L.in_slot for L in T.layers if L.kind == MPN_LAYER_CONV} if numerics == "fp8" else set()
        got = set()
        for s in sorted({0} | {L.out_slot for L in T.layers}):
            try:
                p = m.slot_planes(t, s, rows[0], 1, fp8=True)
            except mpn.MpnError:
                continue
            got.add(s)
            for a, b in _runs(rows):
                _quant_equal(walk, f"tower{t} slot {s} rows {a}..{b - 1}", m.slot_planes(t, s, a, b - a, fp8=True))
        assert got == want, (t, got, want)


def _quant_equal(walk, what, p):
    assert p["fmt"] == 0, what
    h = torch.from_numpy(LR.bf16_values(p["hi"]))
    q, e = F8.quantize(h)
    codes = q.to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    if not (np.array_equal(codes, p["q8"]) and np.array_equal(e.numpy().astype(np.int32), p["e8"])):
        bad = np.argwhere(codes != p["q8"])[:4].tolist()
        walk.fails.append(f"{walk.graph} / {walk.numerics} / fp8 quantizer, {what}: e4m3 plane or exponents differ from the host rule "
                          f"(exponents {p['e8'][:4].tolist()} vs {e[:4].tolist()}, first differing codes at (n, h, w, c) {bad})")


@pytest.mark.parametrize("graph,numerics", CASES)
def test_every_layer(ctx, graph, numerics):
    build, H, W, R, seed, sharp, limits, sampled = GRAPHS[graph]
    spec = build()
    img, boxes = _inputs(spec, H, W, R, seed, sharp=sharp)
    rng = np.random.default_rng(seed)
    walk = Walk(graph, numerics)
    with options(ctx, NUMERICS[numerics]):
        m = mpn.Model(ctx, spec, **limits)
        try:
            m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3, want_raw=False)
            _, _, first = walk_trunk(walk, m, spec, img, numerics, sampled, rng)
            rows, outs, fc6, spread = walk_towers(walk, m, spec, numerics, R, sampled, rng)
            walk_heads(walk, m, spec, numerics, rows, outs)
            check_quantizer(walk, m, spec, numerics, R, rows)
            assert (models.w16_flops_per_roi(spec) > 0) == bool(expected_w16_slots(spec, 0, "default"))
        finally:
            m.close()
    # negative controls: the first layer the rule covers and fc6, against the nearest wrong rules
    trunk_rule = {"default": "exact", "w16_off": "exact", "bf16": "bf16", "fp8": "fp8"}[numerics]
    for wrong in WRONG[trunk_rule]:
        if wrong == "fp8_per_tensor":
            continue                              # one sample (the image) per trunk slot: per tensor is per sample
        walk.outside(first["name"], wrong, rel_err(first["got"].numpy(), first["fn"](wrong).numpy()), first["bar"])
    for wrong in WRONG[fc6["rule"]]:
        walk.outside(fc6["name"], wrong, rel_err(fc6["got"].numpy(), fc6["fn"](wrong).numpy()), fc6["bar"])
    if spread is not None:
        per_roi_control(walk, spread)
    worst = max(((v[0], k) for k, v in walk.worst.items() if isinstance(v, tuple)), default=(0.0, ""))
    record_parity("layer_worst", graph=graph, numerics=numerics, layer=worst[1], error=worst[0])
    assert not walk.fails, "\n".join(walk.fails)


def per_roi_control(walk, c):
    """fp8 per-ROI exponents vs one exponent for all ROI rows. A power-of-two scale only moves which values fall into
    e4m3's subnormals, so the two rules differ on the rows whose own exponent is not the shared one, and on those only by
    their small values: the error is taken per row (max|a - b| / max|ref| of the row) over those rows. A layer whose
    sampled rows all share one exponent cannot tell the rules apart at all. Measured on an H100, the per-row distance is
    3-7e-5 on every graph, inside the 1e-4 bar: this control is recorded, not asserted. What pins the per-ROI exponents is
    check_quantizer (e8 equal to the host rule's per-sample exponents, bit for bit)."""
    e = c["e"]
    diff = torch.nonzero(e != e.min()).flatten()
    if len(diff) == 0:
        record_parity("layer_control", graph=walk.graph, numerics=walk.numerics, layer=c["name"], control="fp8_per_tensor (void: one exponent)",
                      error=0.0, bar=c["bar"])
        return
    got, ref = c["got"][diff].double(), c["fn"]("fp8_per_tensor")[diff].double()
    err = max(rel_err(got[i].numpy(), ref[i].numpy()) for i in range(len(diff)))
    record_parity("layer_control", graph=walk.graph, numerics=walk.numerics, layer=c["name"],
                  control=f"fp8_per_tensor ({len(diff)} rows off the shared exponent, per row)", error=err, bar=c["bar"])


def test_hook_refusals(ctx):
    """an elided slot, an unknown tower or slot, rows out of range, a capacity too small and q8 where the plan keeps none:
    MpnError, never a device fault"""
    build, H, W, R, seed, sharp, limits, _ = GRAPHS["vgg_small"]
    spec = build()
    img, boxes = _inputs(spec, H, W, R, seed, sharp=sharp)
    m = mpn.Model(ctx, spec, **limits)
    try:
        with pytest.raises(mpn.MpnError):
            m.slot_planes(-1, 1)                                  # no pass yet
        with pytest.raises(mpn.MpnError):
            m.head_outputs()
        m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        conv12 = spec.trunk_layers[1]
        with pytest.raises(mpn.MpnError, match="fused"):
            m.slot_planes(-1, conv12.out_slot)                    # conv1_2 -> pool1 fused: never written
        for tower, slot in ((1, 0), (-2, 1), (-1, 999), (-1, 0), (0, 999)):
            with pytest.raises(mpn.MpnError):
                m.slot_planes(tower, slot)
        with pytest.raises(mpn.MpnError):
            m.slot_planes(-1, 1, r0=1, n=1)                       # a trunk slot has one row (the image)
        with pytest.raises(mpn.MpnError):
            m.slot_planes(0, 0, r0=R - 1, n=2)
        with pytest.raises(mpn.MpnError):
            m.slot_planes(0, 0, r0=R, n=1)
        with pytest.raises(mpn.MpnError):
            m.slot_planes(0, 1, fp8=True)                          # the default numerics keep no e4m3 planes
        hi, lo = np.empty(64, np.uint16), np.empty(64, np.uint16)
        fmt, dims = C.c_int32(), (C.c_int64 * 4)()
        rc = ctx.lib.mpn_model_get_slot_planes(m.h, 0, 0, 0, 1, hi.ctypes.data, lo.ctypes.data, None, None, hi.size, C.byref(fmt), dims)
        with pytest.raises(mpn.MpnError, match="too small"):
            ctx.check(rc, "get_slot_planes")
        p = m.slot_planes(0, 3, 5, 2)                             # the tower's output: its concat columns
        assert p["dims"] == (R, 1, 1, 256) and p["hi"].shape == (2, 1, 1, 256)
        cls, bbox = m.head_outputs()
        assert cls.shape == (1, R, 21) and bbox.shape == (R, 84)
        ctx.synchronize()                                        # the context is healthy after the refusals
    finally:
        m.close()
    with options(ctx, {"fp8": 1}):
        m = mpn.Model(ctx, spec, **limits)
        try:
            m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
            with pytest.raises(mpn.MpnError):
                m.slot_planes(0, 0, fp8=True)                      # the pooled slot is read by FLATTEN, not by an fp8 layer
            assert m.slot_planes(0, 1, fp8=True)["q8"].shape == (R, 1, 1, 128 * 49)
        finally:
            m.close()


def test_head_outputs_are_raw(ctx):
    """detect_nms leaves the logits and deltas raw (scores = softmax(logits)); heads() applies BBoxNorm to the deltas in
    place, which head_outputs then shows"""
    from oracle import ref as O
    build, H, W, R, seed, sharp, limits, _ = GRAPHS["vgg_small"]
    spec = build()
    img, boxes = _inputs(spec, H, W, R, seed, sharp=sharp)
    m = mpn.Model(ctx, spec, **limits)
    try:
        scores, _, _ = m.detect_nms(img, boxes, 1.0, W, H, -1.5, 0.3)
        cls, raw = m.head_outputs()
        np.testing.assert_allclose(torch.softmax(torch.from_numpy(cls[0]).double(), 1).numpy(), scores, rtol=0, atol=2e-6)
        _, normed = m.heads(O.project_rois(boxes, 1.0))              # the same ROIs on the cached trunk
        _, after = m.head_outputs()
        assert np.array_equal(after, normed)
        np.testing.assert_allclose(normed, O.bbox_norm(raw, spec.bbox_mean, spec.bbox_std), rtol=1e-6, atol=1e-9)
        assert not np.array_equal(normed, raw)
    finally:
        m.close()

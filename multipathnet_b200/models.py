"""Model descriptions: the graphs of models/{vgg,multipathnet,resnet,alexnet}.lua as data.

The reference builds these graphs by slicing pretrained `.t7` nets that are not in the
tree (vgg.lua:14, multipathnet.lua:26, resnet.lua:25); the layer lists are restated from
the module indices the reference slices at (SURVEY 8a5-a7, A.5). Weights are seeded
synthetic (no network for checkpoints): He-normal convs/fcs, heads N(0,0.01)/N(0,0.001)
with zero bias as model_utils.lua:105-112. All arrays are in Torch layout
(conv Cout x Cin x kh x kw, Linear out x in).
"""
from __future__ import annotations

from typing import List, Tuple

import numpy as np

from ._lib import (Head, Layer, ModelSpec, Tower, MPN_LAYER_AVGPOOL, MPN_LAYER_CONV, MPN_LAYER_FLATTEN,
                   MPN_LAYER_LRN, MPN_LAYER_MAXPOOL)

VGG16_CFG = [64, 64, "M", 128, 128, "M", 256, 256, 256, "M", 512, 512, 512, "M", 512, 512, 512]


class _W:
    """weight list builder with a seeded generator; seed=None builds the STRUCTURE only (all-zero weights, allocated lazily:
    for tests of layer tables / FLOP counts that never look at a weight)"""

    def __init__(self, seed):
        self.skeleton = seed is None
        self.rng = np.random.default_rng(0 if seed is None else seed)
        self.arrays: List[np.ndarray] = []

    def add(self, a: np.ndarray) -> int:
        self.arrays.append(np.ascontiguousarray(a, dtype=np.float32))
        return len(self.arrays) - 1

    def conv(self, cout, cin, kh, kw, gain=1.0, bias_std=0.05) -> Tuple[int, int]:
        std = gain * np.sqrt(2.0 / (cin * kh * kw))
        if self.skeleton:
            return self.add(np.zeros((cout, cin, kh, kw), np.float32)), self.add(np.zeros(cout, np.float32))
        w = self.rng.standard_normal((cout, cin, kh, kw), dtype=np.float32) * np.float32(std)
        b = self.rng.standard_normal(cout, dtype=np.float32) * np.float32(bias_std)
        return self.add(w), self.add(b)

    def linear(self, cout, cin, std=None, zero_bias=False, bias_std=0.05) -> Tuple[int, int]:
        std = np.sqrt(2.0 / cin) if std is None else std
        if self.skeleton:
            return self.add(np.zeros((cout, cin), np.float32)), self.add(np.zeros(cout, np.float32))
        w = self.rng.standard_normal((cout, cin), dtype=np.float32) * np.float32(std)
        b = np.zeros(cout, np.float32) if zero_bias else self.rng.standard_normal(cout, dtype=np.float32) * np.float32(bias_std)
        return self.add(w), self.add(b)

    def clone(self, idx: int) -> int:
        a = self.arrays[idx]
        return self.add(np.zeros(a.shape, np.float32) if self.skeleton else a.copy())


def _vgg_trunk(W: _W, width_div: int = 1, first_gain: float = 1.0 / 64.0):
    """13 x (conv3x3 s1 p1 + ReLU) with 2x2/2 ceil-mode max-pools after conv1_2, 2_2, 3_3, 4_3; no pool5
    (vgg.lua:18 conv indices, multipathnet.lua:35-46 slices). Returns layers and the taps.
    first_gain scales conv1_1 so activations stay O(1) for a +-128 input (well-conditioned parity)."""
    layers: List[Layer] = []
    slot, cin = 0, 3
    taps = {}
    nconv = 0
    for v in VGG16_CFG:
        if v == "M":
            layers.append(Layer(MPN_LAYER_MAXPOOL, slot, slot + 1, kh=2, kw=2, stride=2, pad=0, ceil_mode=1))
        else:
            cout = max(v // width_div, 64)       # tensor-core K blocks are 64 channels wide
            wi, bi = W.conv(cout, cin, 3, 3, gain=first_gain if nconv == 0 else 1.0)
            layers.append(Layer(MPN_LAYER_CONV, slot, slot + 1, cin=cin, cout=cout, kh=3, kw=3, stride=1, pad=1, relu=1,
                                weight=wi, bias=bi))
            cin = cout
            nconv += 1
            if nconv == 7:
                taps["conv3"] = slot + 1
            if nconv == 10:
                taps["conv4"] = slot + 1
            if nconv == 13:
                taps["conv5"] = slot + 1
        slot += 1
    return layers, taps, cin


def vgg16_fast_rcnn(num_classes: int = 21, seed: int = 1234, width_div: int = 1, fc_dim: int = 4096) -> ModelSpec:
    """models/vgg.lua:23-31 + train.lua:137 (BBoxNorm). width_div / fc_dim shrink the net for fast tests."""
    W = _W(seed)
    trunk, taps, c5 = _vgg_trunk(W, width_div)
    k6 = c5 * 49
    w6, b6 = W.linear(fc_dim, k6)
    w7, b7 = W.linear(fc_dim, fc_dim)
    tl = [Layer(MPN_LAYER_FLATTEN, 0, 1),
          Layer(MPN_LAYER_CONV, 1, 2, cin=k6, cout=fc_dim, relu=1, weight=w6, bias=b6),
          Layer(MPN_LAYER_CONV, 2, 3, cin=fc_dim, cout=fc_dim, relu=1, weight=w7, bias=b7)]
    tower = Tower(region=0, levels=[(taps["conv5"], 1.0 / 16)], pooled_w=7, pooled_h=7, normalize=0, layers=tl, out_slot=3)
    wc, bc = W.linear(num_classes, fc_dim, std=0.01, zero_bias=True)
    wb, bb = W.linear(4 * num_classes, fc_dim, std=0.001, zero_bias=True)
    return ModelSpec(name=f"vgg16_fast_rcnn/{width_div}", trunk_layers=trunk, towers=[tower],
                     cls_heads=[Head(0, fc_dim, num_classes, wc, bc)], bbox_head=Head(0, fc_dim, 4 * num_classes, wb, bb),
                     num_classes=num_classes, weights=W.arrays, transformer="ross", taps=taps)


def vgg16_multipathnet(num_classes: int = 81, seed: int = 1234, width_div: int = 1, fc_dim: int = 4096,
                       integral_k: int = 0) -> ModelSpec:
    """models/multipathnet.lua:30-121 with model_het=true, model_conv345_norm=true: four foveal towers
    (regions x1, x1.5, x2, x4; conv3 only on tower 1, conv4 on towers 1-3) + the 'het' tower on region 2
    with conv5+4+3; class head over towers 1-4, bbox head over the het tower (multipathnet.lua:115-117).
    integral_k>0 adds the integral-loss head (model_utils.lua:275-317, eval = mean of K softmaxes)."""
    W = _W(seed)
    trunk, taps, c5 = _vgg_trunk(W, width_div)
    c4 = c5
    c3 = max(256 // width_div, 64)
    mix_out = c5
    k6 = mix_out * 49
    w6, b6 = W.linear(fc_dim, k6)        # `classifier` — every tower gets classifier:clone() (multipathnet.lua:89,107)
    w7, b7 = W.linear(fc_dim, fc_dim)

    def tower(region, use3, use4):
        levels = [(taps["conv5"], 1.0 / 16)]
        tot = c5
        if use4:
            levels.append((taps["conv4"], 1.0 / 8)); tot += c4
        if use3:
            levels.append((taps["conv3"], 1.0 / 4)); tot += c3
        wm, bm = W.conv(mix_out, tot, 1, 1, gain=0.7)          # conv_mix (model_utils.lua:242), no ReLU after
        layers = [Layer(MPN_LAYER_CONV, 0, 1, cin=tot, cout=mix_out, kh=1, kw=1, relu=0, weight=wm, bias=bm),
                  Layer(MPN_LAYER_FLATTEN, 1, 2),
                  Layer(MPN_LAYER_CONV, 2, 3, cin=k6, cout=fc_dim, relu=1, weight=W.clone(w6), bias=W.clone(b6)),
                  Layer(MPN_LAYER_CONV, 3, 4, cin=fc_dim, cout=fc_dim, relu=1, weight=W.clone(w7), bias=W.clone(b7))]
        return Tower(region=region, levels=levels, pooled_w=7, pooled_h=7, normalize=1, layers=layers, out_slot=4)

    towers = [tower(0, True, True), tower(1, False, True), tower(2, False, True), tower(3, False, False),
              tower(1, True, True)]                                   # het: region 2 (=Select(1,2)) with conv3+4+5
    nreg = 4
    k = max(integral_k, 1)
    cls = []
    for _ in range(k):
        wc, bc = W.linear(num_classes, nreg * fc_dim, std=0.01, zero_bias=True)
        cls.append(Head(0, nreg * fc_dim, num_classes, wc, bc))
    wb, bb = W.linear(4 * num_classes, fc_dim, std=0.001, zero_bias=True)
    return ModelSpec(name=f"vgg16_multipathnet/{width_div}", trunk_layers=trunk, towers=towers, cls_heads=cls,
                     bbox_head=Head(nreg * fc_dim, fc_dim, 4 * num_classes, wb, bb), num_classes=num_classes,
                     weights=W.arrays, no_softmax=1 if integral_k > 0 else 0, transformer="ross", taps=taps)


def alexnet_fast_rcnn(num_classes: int = 21, seed: int = 1234) -> ModelSpec:
    """models/alexnet.lua:14-26 (CaffeNet Fast R-CNN, ROIPooling(6,6,1/16), fc6 9216->4096). BASELINE configs[0]:
    the reference's own CPU-runnable plumbing case — used with the CPU oracle only (grouped convs + LRN are not
    part of the GPU path; Model() refuses this spec)."""
    W = _W(seed)
    L: List[Layer] = []
    def conv(i, o, cin, cout, k, s, p, g=1, gain=1.0):
        w, b = W.conv(cout, cin // g, k, k, gain=gain)
        L.append(Layer(MPN_LAYER_CONV, i, o, cin=cin, cout=cout, kh=k, kw=k, stride=s, pad=p, relu=1, weight=w, bias=b, groups=g))
    conv(0, 1, 3, 96, 11, 4, 0, gain=1.0 / 64)
    L.append(Layer(MPN_LAYER_MAXPOOL, 1, 2, kh=3, kw=3, stride=2, ceil_mode=1))
    L.append(Layer(MPN_LAYER_LRN, 2, 3))
    conv(3, 4, 96, 256, 5, 1, 2, g=2)
    L.append(Layer(MPN_LAYER_MAXPOOL, 4, 5, kh=3, kw=3, stride=2, ceil_mode=1))
    L.append(Layer(MPN_LAYER_LRN, 5, 6))
    conv(6, 7, 256, 384, 3, 1, 1)
    conv(7, 8, 384, 384, 3, 1, 1, g=2)
    conv(8, 9, 384, 256, 3, 1, 1, g=2)
    w6, b6 = W.linear(4096, 256 * 36)
    w7, b7 = W.linear(4096, 4096)
    tl = [Layer(MPN_LAYER_FLATTEN, 0, 1), Layer(MPN_LAYER_CONV, 1, 2, cin=9216, cout=4096, relu=1, weight=w6, bias=b6),
          Layer(MPN_LAYER_CONV, 2, 3, cin=4096, cout=4096, relu=1, weight=w7, bias=b7)]
    tower = Tower(region=0, levels=[(9, 1.0 / 16)], pooled_w=6, pooled_h=6, normalize=0, layers=tl, out_slot=3)
    wc, bc = W.linear(num_classes, 4096, std=0.01, zero_bias=True)
    wb, bb = W.linear(4 * num_classes, 4096, std=0.001, zero_bias=True)
    return ModelSpec(name="alexnet_fast_rcnn", trunk_layers=L, towers=[tower], cls_heads=[Head(0, 4096, num_classes, wc, bc)],
                     bbox_head=Head(0, 4096, 4 * num_classes, wb, bb), num_classes=num_classes, weights=W.arrays,
                     transformer="ross", taps={"conv5": 9})


def _bottleneck(W: _W, layers: List[Layer], slot_in: int, next_slot: int, cin: int, mid: int, cout: int, stride: int):
    """fb.resnet.torch bottleneck, BN folded into conv+bias (resnet.lua:33-36): 1x1 -> 3x3(stride) -> 1x1,
    + shortcut (1x1 conv with the same stride when shape changes), ReLU after the add."""
    s = next_slot
    w1, b1 = W.conv(mid, cin, 1, 1)
    w2, b2 = W.conv(mid, mid, 3, 3)
    w3, b3 = W.conv(cout, mid, 1, 1, gain=0.5)
    layers.append(Layer(MPN_LAYER_CONV, slot_in, s, cin=cin, cout=mid, kh=1, kw=1, relu=1, weight=w1, bias=b1))
    layers.append(Layer(MPN_LAYER_CONV, s, s + 1, cin=mid, cout=mid, kh=3, kw=3, stride=stride, pad=1, relu=1, weight=w2, bias=b2))
    res_slot = slot_in
    nxt = s + 2
    if stride != 1 or cin != cout:
        ws, bs = W.conv(cout, cin, 1, 1, gain=0.5)
        layers.append(Layer(MPN_LAYER_CONV, slot_in, nxt, cin=cin, cout=cout, kh=1, kw=1, stride=stride, relu=0, weight=ws, bias=bs))
        res_slot = nxt
        nxt += 1
    layers.append(Layer(MPN_LAYER_CONV, s + 1, nxt, cin=mid, cout=cout, kh=1, kw=1, relu=1, residual_slot=res_slot, weight=w3, bias=b3))
    return nxt, nxt + 1


def resnet50_fast_rcnn(num_classes: int = 81, seed: int = 1234, width_div: int = 1, integral_k: int = 6,
                       blocks=(3, 4, 6, 3)) -> ModelSpec:
    """models/resnet.lua:28-50 on ResNet-50 (+ model_utils.integral with K heads, train.lua:125-127):
    trunk = conv1 7x7/2, maxpool 3x3/2 p1, layer1-3; ROIPooling(14,14,1/16); per-ROI layer4 + avgpool 7."""
    W = _W(seed)
    base = 64; assert width_div == 1, 'ResNet widths below 64 do not fill a 64-channel K block'
    trunk: List[Layer] = []
    w, b = W.conv(base, 3, 7, 7, gain=1.0 / 2.0)
    trunk.append(Layer(MPN_LAYER_CONV, 0, 1, cin=3, cout=base, kh=7, kw=7, stride=2, pad=3, relu=1, weight=w, bias=b))
    trunk.append(Layer(MPN_LAYER_MAXPOOL, 1, 2, kh=3, kw=3, stride=2, pad=1, ceil_mode=0))
    slot, nxt, cin = 2, 3, base
    for li, nb in enumerate(blocks[:3]):
        mid = base * (2 ** li)
        for bi in range(nb):
            stride = 2 if (bi == 0 and li > 0) else 1
            slot, nxt = _bottleneck(W, trunk, slot, nxt, cin, mid, mid * 4, stride)
            cin = mid * 4
    taps = {"layer3": slot}
    tl: List[Layer] = []
    tslot, tnxt, tc = 0, 1, cin
    mid = base * 8
    for bi in range(blocks[3]):
        tslot, tnxt = _bottleneck(W, tl, tslot, tnxt, tc, mid, mid * 4, 2 if bi == 0 else 1)
        tc = mid * 4
    tl.append(Layer(MPN_LAYER_AVGPOOL, tslot, tnxt))
    tower = Tower(region=0, levels=[(slot, 1.0 / 16)], pooled_w=14, pooled_h=14, normalize=0, layers=tl, out_slot=tnxt)
    k = max(integral_k, 1)
    cls = []
    for _ in range(k):
        wc, bc = W.linear(num_classes, tc, std=0.01, zero_bias=True)
        cls.append(Head(0, tc, num_classes, wc, bc))
    wb, bb = W.linear(4 * num_classes, tc, std=0.001, zero_bias=True)
    return ModelSpec(name=f"resnet50_fast_rcnn/{width_div}", trunk_layers=trunk, towers=[tower], cls_heads=cls,
                     bbox_head=Head(0, tc, 4 * num_classes, wb, bb), num_classes=num_classes, weights=W.arrays,
                     no_softmax=1 if integral_k > 0 else 0, transformer="imagenet", taps=taps)


# ---- analytic FLOP counts (SURVEY 8d: conv 2*Cin*Cout*kh*kw*Ho*Wo, linear 2*M*K*N) ---------------------
def _pool_out(n, k, s, p, ceil_mode):
    o = (n + 2 * p - k + (s - 1 if ceil_mode else 0)) // s + 1
    if ceil_mode and (o - 1) * s >= n + p:
        o -= 1
    return o


def trunk_flops(spec: ModelSpec, H: int, W: int) -> float:
    shp = {0: (H, W)}
    fl = 0.0
    for L in spec.trunk_layers:
        h, w = shp[L.in_slot]
        if L.kind == MPN_LAYER_CONV:
            ho, wo = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1
            fl += 2.0 * L.cin * L.cout * L.kh * L.kw * ho * wo
        else:
            ho, wo = _pool_out(h, L.kh, L.stride, L.pad, L.ceil_mode), _pool_out(w, L.kw, L.stride, L.pad, L.ceil_mode)
        shp[L.out_slot] = (ho, wo)
    return fl


def head_flops_per_roi(spec: ModelSpec) -> float:
    fl = 0.0
    for t in spec.towers:
        shp = {0: (t.pooled_h, t.pooled_w)}
        for L in t.layers:
            h, w = shp[L.in_slot]
            if L.kind == MPN_LAYER_CONV:
                ho, wo = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1
                fl += 2.0 * L.cin * L.cout * L.kh * L.kw * ho * wo
                shp[L.out_slot] = (ho, wo)
            else:
                shp[L.out_slot] = (1, 1)
    for hd in list(spec.cls_heads) + [spec.bbox_head]:
        fl += 2.0 * hd.col_len * hd.cout
    return fl


def w16_flops_per_roi(spec: ModelSpec) -> float:
    """algorithmic FLOPs per ROI of the Linears that take the two-product "w16" numerics by default (csrc/model.cu, plan_heads:
    single-tower graphs only; a Linear on a 1 x 1 map — incl. the one that follows a FLATTEN, whose kernel spans the pooled
    map — with >= 2048 inputs and >= 1024 outputs, no residual): what `issued` MMA work is counted x2 instead of x3 for"""
    if len(spec.towers) != 1:
        return 0.0
    fl = 0.0
    for t in spec.towers:
        shp = {0: (t.pooled_h, t.pooled_w)}
        for L in t.layers:
            h, w = shp[L.in_slot]
            if L.kind == MPN_LAYER_CONV:
                ho, wo = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.pad - L.kw) // L.stride + 1
                k_in = L.cin * L.kh * L.kw
                if ho == 1 and wo == 1 and L.kh == h and L.kw == w and L.pad == 0 and L.residual_slot < 0 and k_in >= 2048 and L.cout >= 1024:
                    fl += 2.0 * k_in * L.cout
                shp[L.out_slot] = (ho, wo)
            else:
                shp[L.out_slot] = (1, 1)
    return fl

"""Model descriptions: the graphs of models/{vgg,multipathnet,resnet,alexnet,nin,inceptionv3}.lua as data.

The reference builds these graphs by slicing pretrained `.t7` nets that are not in the
tree (vgg.lua:14, multipathnet.lua:26, resnet.lua:25); the layer lists are restated from
the module indices the reference slices at (SURVEY 8a5-a7, A.5). Weights are seeded
synthetic (no network for checkpoints): He-normal convs/fcs, heads N(0,0.01)/N(0,0.001)
with zero bias as model_utils.lua:105-112. All arrays are in Torch layout
(conv Cout x Cin x kh x kw, Linear out x in).
"""
from __future__ import annotations

import dataclasses
from typing import List, Tuple

import numpy as np

from ._lib import (Head, Layer, ModelSpec, Tower, MPN_LAYER_AVGPOOL, MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_CONV, MPN_LAYER_FLATTEN,
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

    def conv_fixed_bn(self, cout, cin, kh, kw, gain=1.0) -> Tuple[int, int, np.ndarray]:
        """a bias-free convolution W followed by inn.ConstAffine (y = a[c] * x + b[c], a ~ U[0.5, 2], b small), stored
        folded as W' = fl(a * W) with bias b; returns (weight, bias, a). W is drawn He-normal over E[a^2] = 1.75 so the
        folded layer keeps the He scale."""
        if self.skeleton:
            wi, bi = self.conv(cout, cin, kh, kw)
            return wi, bi, np.ones(cout, np.float32)
        std = gain * np.sqrt(2.0 / (cin * kh * kw) / 1.75)
        w = self.rng.standard_normal((cout, cin, kh, kw), dtype=np.float32) * np.float32(std)
        a = self.rng.uniform(0.5, 2.0, cout).astype(np.float32)
        b = self.rng.standard_normal(cout, dtype=np.float32) * np.float32(0.05)
        return self.add(a[:, None, None, None] * w), self.add(b), a


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


def vgg16_fast_rcnn(num_classes: int = 21, seed: int = 1234, width_div: int = 1, fc_dim: int = 4096, integral_k: int = 0) -> ModelSpec:
    """models/vgg.lua:23-31 + train.lua:137 (BBoxNorm). width_div / fc_dim shrink the net for fast tests. integral_k > 0
    gives K = integral_k class heads over the same columns as the bbox head (model_utils.integral; each head drawn from
    the generator in turn, as vgg16_multipathnet does); integral_k = 0 builds exactly the single-head model."""
    W = _W(seed)
    trunk, taps, c5 = _vgg_trunk(W, width_div)
    k6 = c5 * 49
    w6, b6 = W.linear(fc_dim, k6)
    w7, b7 = W.linear(fc_dim, fc_dim)
    tl = [Layer(MPN_LAYER_FLATTEN, 0, 1),
          Layer(MPN_LAYER_CONV, 1, 2, cin=k6, cout=fc_dim, relu=1, weight=w6, bias=b6),
          Layer(MPN_LAYER_CONV, 2, 3, cin=fc_dim, cout=fc_dim, relu=1, weight=w7, bias=b7)]
    tower = Tower(region=0, levels=[(taps["conv5"], 1.0 / 16)], pooled_w=7, pooled_h=7, normalize=0, layers=tl, out_slot=3)
    cls = []
    for _ in range(max(integral_k, 1)):
        wc, bc = W.linear(num_classes, fc_dim, std=0.01, zero_bias=True)
        cls.append(Head(0, fc_dim, num_classes, wc, bc))
    wb, bb = W.linear(4 * num_classes, fc_dim, std=0.001, zero_bias=True)
    return ModelSpec(name=f"vgg16_fast_rcnn/{width_div}", trunk_layers=trunk, towers=[tower],
                     cls_heads=cls, bbox_head=Head(0, fc_dim, 4 * num_classes, wb, bb),
                     num_classes=num_classes, weights=W.arrays, no_softmax=1 if integral_k > 0 else 0, transformer="ross", taps=taps,
                     trunk_train_from=6)              # vgg.lua:18-19: conv1_1 .. pool2 frozen, conv3_1 onwards trains


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
                     weights=W.arrays, no_softmax=1 if integral_k > 0 else 0, transformer="ross", taps=taps,
                     phase2_from=6)             # vggSetPhase2_outer: the skip trunk's first 10 modules (conv1_1 .. pool2) stay frozen


def alexnet_fast_rcnn(num_classes: int = 21, seed: int = 1234, first_gain: float = 1.0 / 64) -> ModelSpec:
    """models/alexnet.lua:14-26 (CaffeNet Fast R-CNN, ROIPooling(6,6,1/16), fc6 9216->4096), BASELINE configs[0]. Runs on
    the device (Model) in the default and bf16 numerics, inference only: conv1 11 x 11 / 4 on the first-layer kernel,
    conv2 (5 x 5, 2 groups), conv4 and conv5 (3 x 3, 2 groups) as one engine problem per group, norm1 / norm2 on
    lrn_split_kernel (MPN_LAYER_LRN, CaffeNet's constants). first_gain scales conv1's He weights; the default 1/64 keeps
    activations O(1) for a +-128 input, where the LRN is nearly the identity (a * S small), so tests of the LRN pass a
    larger gain."""
    W = _W(seed)
    L: List[Layer] = []
    def conv(i, o, cin, cout, k, s, p, g=1, gain=1.0):
        w, b = W.conv(cout, cin // g, k, k, gain=gain)
        L.append(Layer(MPN_LAYER_CONV, i, o, cin=cin, cout=cout, kh=k, kw=k, stride=s, pad=p, relu=1, weight=w, bias=b, groups=g))
    conv(0, 1, 3, 96, 11, 4, 0, gain=first_gain)
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


def _conv(W: _W, fixed_bn, cout, cin, k, gain=1.0) -> Tuple[int, int]:
    """a ResNet convolution: BN folded into conv + bias (fixed_bn None), or the fixed-batch-norm form
    (W.conv_fixed_bn), its scale recorded in the dict fixed_bn under the weight's index"""
    if fixed_bn is None:
        return W.conv(cout, cin, k, k, gain=gain)
    wi, bi, a = W.conv_fixed_bn(cout, cin, k, k, gain=gain)
    fixed_bn[wi] = a
    return wi, bi


def _bottleneck(W: _W, layers: List[Layer], slot_in: int, next_slot: int, cin: int, mid: int, cout: int, stride: int,
                fixed_bn=None):
    """fb.resnet.torch bottleneck, BN folded into conv+bias (resnet.lua:33-36): 1x1 -> 3x3(stride) -> 1x1,
    + shortcut (1x1 conv with the same stride when shape changes), ReLU after the add."""
    s = next_slot
    w1, b1 = _conv(W, fixed_bn, mid, cin, 1)
    w2, b2 = _conv(W, fixed_bn, mid, mid, 3)
    w3, b3 = _conv(W, fixed_bn, cout, mid, 1, gain=0.5)
    layers.append(Layer(MPN_LAYER_CONV, slot_in, s, cin=cin, cout=mid, kh=1, kw=1, relu=1, weight=w1, bias=b1))
    layers.append(Layer(MPN_LAYER_CONV, s, s + 1, cin=mid, cout=mid, kh=3, kw=3, stride=stride, pad=1, relu=1, weight=w2, bias=b2))
    res_slot = slot_in
    nxt = s + 2
    if stride != 1 or cin != cout:
        ws, bs = _conv(W, fixed_bn, cout, cin, 1, gain=0.5)
        layers.append(Layer(MPN_LAYER_CONV, slot_in, nxt, cin=cin, cout=cout, kh=1, kw=1, stride=stride, relu=0, weight=ws, bias=bs))
        res_slot = nxt
        nxt += 1
    layers.append(Layer(MPN_LAYER_CONV, s + 1, nxt, cin=mid, cout=cout, kh=1, kw=1, relu=1, residual_slot=res_slot, weight=w3, bias=b3))
    return nxt, nxt + 1


def _basic_block(W: _W, layers: List[Layer], slot_in: int, next_slot: int, cin: int, cout: int, stride: int, fixed_bn=None):
    """fb.resnet.torch basic block (ResNet-18 / 34): 3x3(stride) -> 3x3, + shortcut (1x1 conv with the same stride when
    the shape changes, shortcut type B), ReLU after the add."""
    s = next_slot
    w1, b1 = _conv(W, fixed_bn, cout, cin, 3)
    layers.append(Layer(MPN_LAYER_CONV, slot_in, s, cin=cin, cout=cout, kh=3, kw=3, stride=stride, pad=1, relu=1, weight=w1, bias=b1))
    res_slot, nxt = slot_in, s + 1
    if stride != 1 or cin != cout:
        ws, bs = _conv(W, fixed_bn, cout, cin, 1, gain=0.5)
        layers.append(Layer(MPN_LAYER_CONV, slot_in, nxt, cin=cin, cout=cout, kh=1, kw=1, stride=stride, relu=0, weight=ws, bias=bs))
        res_slot, nxt = nxt, nxt + 1
    w2, b2 = _conv(W, fixed_bn, cout, cout, 3, gain=0.5)
    layers.append(Layer(MPN_LAYER_CONV, s, nxt, cin=cout, cout=cout, kh=3, kw=3, pad=1, relu=1, residual_slot=res_slot, weight=w2, bias=b2))
    return nxt, nxt + 1


def _resnet_fast_rcnn(name: str, bottleneck: bool, num_classes: int, seed, integral_k: int, blocks, fixed_bn: bool) -> ModelSpec:
    """models/resnet.lua:28-50 (+ model_utils.integral with K heads, train.lua:125-127): trunk = conv1 7x7/2, maxpool
    3x3/2 p1, layer1-3; ROIPooling(14,14,1/16); per-ROI layer4 + avgpool 7. fixed_bn: every convolution of layer2 ..
    layer4 in the fixed-batch-norm form of resnet.lua's BNtoFixed (scales in spec.fixed_bn), and the trunk trains from
    layer2's first convolution (disableFeatureBackprop(features, 5): conv1 .. layer1 frozen)."""
    W = _W(seed)
    base = 64
    rec = {} if fixed_bn else None
    trunk: List[Layer] = []
    w, b = W.conv(base, 3, 7, 7, gain=1.0 / 2.0)
    trunk.append(Layer(MPN_LAYER_CONV, 0, 1, cin=3, cout=base, kh=7, kw=7, stride=2, pad=3, relu=1, weight=w, bias=b))
    trunk.append(Layer(MPN_LAYER_MAXPOOL, 1, 2, kh=3, kw=3, stride=2, pad=1, ceil_mode=0))
    expand = 4 if bottleneck else 1

    def block(layers, slot, nxt, cin, width, stride, fb):
        if bottleneck:
            return _bottleneck(W, layers, slot, nxt, cin, width, width * 4, stride, fb)
        return _basic_block(W, layers, slot, nxt, cin, width, stride, fb)

    slot, nxt, cin = 2, 3, base
    train_from = 0
    for li, nb in enumerate(blocks[:3]):
        width = base * (2 ** li)
        if li == 1 and fixed_bn:
            train_from = len(trunk)
        for bi in range(nb):
            stride = 2 if (bi == 0 and li > 0) else 1
            slot, nxt = block(trunk, slot, nxt, cin, width, stride, rec if li > 0 else None)
            cin = width * expand
    taps = {"layer3": slot}
    tl: List[Layer] = []
    tslot, tnxt, tc = 0, 1, cin
    width = base * 8
    for bi in range(blocks[3]):
        tslot, tnxt = block(tl, tslot, tnxt, tc, width, 2 if bi == 0 else 1, rec)
        tc = width * expand
    tl.append(Layer(MPN_LAYER_AVGPOOL, tslot, tnxt))
    tower = Tower(region=0, levels=[(slot, 1.0 / 16)], pooled_w=14, pooled_h=14, normalize=0, layers=tl, out_slot=tnxt)
    k = max(integral_k, 1)
    cls = []
    for _ in range(k):
        wc, bc = W.linear(num_classes, tc, std=0.01, zero_bias=True)
        cls.append(Head(0, tc, num_classes, wc, bc))
    wb, bb = W.linear(4 * num_classes, tc, std=0.001, zero_bias=True)
    return ModelSpec(name=name, trunk_layers=trunk, towers=[tower], cls_heads=cls,
                     bbox_head=Head(0, tc, 4 * num_classes, wb, bb), num_classes=num_classes, weights=W.arrays,
                     no_softmax=1 if integral_k > 0 else 0, transformer="imagenet", taps=taps, trunk_train_from=train_from,
                     fixed_bn=rec or {})


def resnet50_fast_rcnn(num_classes: int = 81, seed: int = 1234, width_div: int = 1, integral_k: int = 6,
                       blocks=(3, 4, 6, 3), fixed_bn: bool = False) -> ModelSpec:
    """models/resnet.lua:28-50 on ResNet-50: bottleneck blocks (see _resnet_fast_rcnn). fixed_bn=False builds exactly the
    BN-folded model that inference has always run."""
    assert width_div == 1, 'ResNet widths below 64 do not fill a 64-channel K block'
    return _resnet_fast_rcnn(f"resnet50_fast_rcnn/{width_div}", True, num_classes, seed, integral_k, blocks, fixed_bn)


def resnet18_fast_rcnn(num_classes: int = 81, seed: int = 1234, integral_k: int = 6, blocks=(2, 2, 2, 2),
                       fixed_bn: bool = False) -> ModelSpec:
    """models/resnet.lua:28-50 on ResNet-18 (the README's `model=resnet resnet_path=.../resnet-18.t7` recipe): basic
    blocks 3x3(stride) -> 3x3, 1x1 projection shortcuts where the shape changes (see _resnet_fast_rcnn)."""
    return _resnet_fast_rcnn("resnet18_fast_rcnn", False, num_classes, seed, integral_k, blocks, fixed_bn)


def nin_fast_rcnn(num_classes: int = 21, seed: int = 1234, fixed_bn: bool = False, integral_k: int = 0) -> ModelSpec:
    """models/nin.lua on imagenet-multiGPU.torch's `ninbn` (block contents as recalled, parity unpinned): 9-module blocks
    conv -> BN -> ReLU -> (1x1 conv -> BN -> ReLU) x 2, BN folded into conv + bias, each ReLU fused into its convolution.
      features 1..29 = block(3 -> 96, 11x11 / 4 / 5), max pool 3x3 / 2 / 1 (floor), block(96 -> 256, 5x5 / 1 / 2), max pool,
                       block(256 -> 384, 3x3 / 1 / 1): 11 trunk layers, 384 x 14 x 14 at 224 px (stride 16);
      ROIPooling(7, 7, 1/16), classifier 31..40 = block(384 -> 1024, 3x3 / 1 / 1) + SpatialAveragePooling(7, 7) + View:
                       one tower of three convolutions and a global AVGPOOL, 1024 features per ROI;
      classAndBBoxLinear(1024), ImagenetTransformer.
    Block 1's 96 channels do not fill the engine's 64-channel K blocks: its two 1x1 convolutions and block 2's 5x5 run with a
    K tail (conv_k_pad in csrc/common.cuh). fixed_bn: every convolution of blocks 2-4 in the fixed-batch-norm form of
    nin.lua's BNtoFixed (scales in spec.fixed_bn), and the trunk trains from block 2's 5x5 convolution
    (disableFeatureBackprop(features, 10)); block 1 stays folded. integral_k as resnet*_fast_rcnn."""
    W = _W(seed)
    rec = {} if fixed_bn else None
    trunk: List[Layer] = []

    def block(layers, slot, cin, cout, k, stride, pad, fb, first_gain=1.0):
        for i, (ci, kk, s, p) in enumerate(((cin, k, stride, pad), (cout, 1, 1, 0), (cout, 1, 1, 0))):
            wi, bi = _conv(W, fb, cout, ci, kk, gain=first_gain if i == 0 else 1.0)
            layers.append(Layer(MPN_LAYER_CONV, slot, slot + 1, cin=ci, cout=cout, kh=kk, kw=kk, stride=s, pad=p, relu=1,
                                weight=wi, bias=bi))
            slot += 1
        return slot

    slot = block(trunk, 0, 3, 96, 11, 4, 5, None, first_gain=0.5)
    trunk.append(Layer(MPN_LAYER_MAXPOOL, slot, slot + 1, kh=3, kw=3, stride=2, pad=1, ceil_mode=0)); slot += 1
    train_from = len(trunk) if fixed_bn else 0
    slot = block(trunk, slot, 96, 256, 5, 1, 2, rec)
    trunk.append(Layer(MPN_LAYER_MAXPOOL, slot, slot + 1, kh=3, kw=3, stride=2, pad=1, ceil_mode=0)); slot += 1
    slot = block(trunk, slot, 256, 384, 3, 1, 1, rec)
    tl: List[Layer] = []
    ts = block(tl, 0, 384, 1024, 3, 1, 1, rec)
    tl.append(Layer(MPN_LAYER_AVGPOOL, ts, ts + 1))
    tower = Tower(region=0, levels=[(slot, 1.0 / 16)], pooled_w=7, pooled_h=7, normalize=0, layers=tl, out_slot=ts + 1)
    cls = []
    for _ in range(max(integral_k, 1)):
        wc, bc = W.linear(num_classes, 1024, std=0.01, zero_bias=True)
        cls.append(Head(0, 1024, num_classes, wc, bc))
    wb, bb = W.linear(4 * num_classes, 1024, std=0.001, zero_bias=True)
    return ModelSpec(name="nin_fast_rcnn", trunk_layers=trunk, towers=[tower], cls_heads=cls,
                     bbox_head=Head(0, 1024, 4 * num_classes, wb, bb), num_classes=num_classes, weights=W.arrays,
                     no_softmax=1 if integral_k > 0 else 0, transformer="imagenet", taps={"block3": slot},
                     trunk_train_from=train_from, fixed_bn=rec or {})


class _Graph:
    """slot bookkeeping for a branching graph: every layer writes a fresh slot, or its channel slice of a concatenation
    slot (Layer.out_c_off / out_c_total); every convolution is followed by a folded batch norm and a ReLU, or, with
    fixed_bn (a dict), by the fixed-batch-norm form (W.conv_fixed_bn), its scale recorded there as _conv does"""

    def __init__(self, W: _W, first_slot: int, fixed_bn=None):
        self.W, self.layers, self.next, self.fixed_bn = W, [], first_slot, fixed_bn

    def slot(self) -> int:
        self.next += 1
        return self.next - 1

    def conv(self, src, cin, cout, kh, kw, stride=1, ph=0, pw=0, dst=None, gain=1.0):
        """dst = (slot, channel offset, slot width) writes a branch of a concatenation; returns the output slot"""
        if self.fixed_bn is None:
            wi, bi = self.W.conv(cout, cin, kh, kw, gain=gain)
        else:
            wi, bi, a = self.W.conv_fixed_bn(cout, cin, kh, kw, gain=gain)
            self.fixed_bn[wi] = a
        out, off, tot = dst if dst else (self.slot(), 0, 0)
        self.layers.append(Layer(MPN_LAYER_CONV, src, out, cin=cin, cout=cout, kh=kh, kw=kw, stride=stride, pad=ph, relu=1,
                                 weight=wi, bias=bi, pad_w=pw if pw != ph else -1, out_c_off=off, out_c_total=tot))
        return out

    def pool(self, kind, src, k, s, p, dst=None, exclude_pad=0):
        out, off, tot = dst if dst else (self.slot(), 0, 0)
        self.layers.append(Layer(kind, src, out, kh=k, kw=k, stride=s, pad=p, out_c_off=off, out_c_total=tot,
                                 exclude_pad=exclude_pad))
        return out


def _mixed_5(g: _Graph, x, cin, pool_c, xp):
    """Mixed_5b / 5c / 5d (35 x 35): 1x1 64 | 1x1 48 -> 5x5 64 | 1x1 64 -> 3x3 96 -> 3x3 96 | avg pool -> 1x1 pool_c"""
    tot = 224 + pool_c
    o = g.slot()
    g.conv(x, cin, 64, 1, 1, dst=(o, 0, tot))
    g.conv(g.conv(x, cin, 48, 1, 1), 48, 64, 5, 5, ph=2, pw=2, dst=(o, 64, tot))
    b = g.conv(g.conv(x, cin, 64, 1, 1), 64, 96, 3, 3, ph=1, pw=1)
    g.conv(b, 96, 96, 3, 3, ph=1, pw=1, dst=(o, 128, tot))
    g.conv(g.pool(MPN_LAYER_AVGPOOL_WIN, x, 3, 1, 1, exclude_pad=xp), cin, pool_c, 1, 1, dst=(o, 224, tot))
    return o, tot


def _mixed_6a(g: _Graph, x, cin):
    """Mixed_6a (35 -> 17): 3x3/2 v 384 | 1x1 64 -> 3x3 96 -> 3x3/2 v 96 | max pool 3x3/2 v"""
    tot = 384 + 96 + cin
    o = g.slot()
    g.conv(x, cin, 384, 3, 3, stride=2, dst=(o, 0, tot))
    b = g.conv(g.conv(x, cin, 64, 1, 1), 64, 96, 3, 3, ph=1, pw=1)
    g.conv(b, 96, 96, 3, 3, stride=2, dst=(o, 384, tot))
    g.pool(MPN_LAYER_MAXPOOL, x, 3, 2, 0, dst=(o, 480, tot))
    return o, tot


def _mixed_6(g: _Graph, x, cin, c, xp):
    """Mixed_6b..6e (17 x 17): 1x1 192 | 1x1 c -> 1x7 c -> 7x1 192 | 1x1 c -> 7x1 c -> 1x7 c -> 7x1 c -> 1x7 192 |
    avg pool -> 1x1 192; a 1 x n kernel pads (0, (n - 1) / 2), an n x 1 kernel ((n - 1) / 2, 0)"""
    o, tot = g.slot(), 768
    g.conv(x, cin, 192, 1, 1, dst=(o, 0, tot))
    b = g.conv(g.conv(x, cin, c, 1, 1), c, c, 1, 7, pw=3)
    g.conv(b, c, 192, 7, 1, ph=3, dst=(o, 192, tot))
    b = g.conv(x, cin, c, 1, 1)
    b = g.conv(g.conv(g.conv(b, c, c, 7, 1, ph=3), c, c, 1, 7, pw=3), c, c, 7, 1, ph=3)
    g.conv(b, c, 192, 1, 7, pw=3, dst=(o, 384, tot))
    g.conv(g.pool(MPN_LAYER_AVGPOOL_WIN, x, 3, 1, 1, exclude_pad=xp), cin, 192, 1, 1, dst=(o, 576, tot))
    return o, tot


def _mixed_7a(g: _Graph, x, cin):
    """Mixed_7a (17 -> 8): 1x1 192 -> 3x3/2 v 320 | 1x1 192 -> 1x7 -> 7x1 -> 3x3/2 v 192 | max pool 3x3/2 v"""
    tot = 320 + 192 + cin
    o = g.slot()
    g.conv(g.conv(x, cin, 192, 1, 1), 192, 320, 3, 3, stride=2, dst=(o, 0, tot))
    b = g.conv(g.conv(g.conv(x, cin, 192, 1, 1), 192, 192, 1, 7, pw=3), 192, 192, 7, 1, ph=3)
    g.conv(b, 192, 192, 3, 3, stride=2, dst=(o, 320, tot))
    g.pool(MPN_LAYER_MAXPOOL, x, 3, 2, 0, dst=(o, 512, tot))
    return o, tot


def _mixed_7(g: _Graph, x, cin, xp):
    """Mixed_7b / 7c (8 x 8): 1x1 320 | 1x1 384 -> {1x3, 3x1} 384 each | 1x1 448 -> 3x3 384 -> {1x3, 3x1} 384 each |
    avg pool -> 1x1 192; the {1x3, 3x1} pairs are nested concatenations, written straight into the block's slot"""
    o, tot = g.slot(), 2048
    g.conv(x, cin, 320, 1, 1, dst=(o, 0, tot))
    b = g.conv(x, cin, 384, 1, 1)
    g.conv(b, 384, 384, 1, 3, pw=1, dst=(o, 320, tot))
    g.conv(b, 384, 384, 3, 1, ph=1, dst=(o, 704, tot))
    b = g.conv(g.conv(x, cin, 448, 1, 1), 448, 384, 3, 3, ph=1, pw=1)
    g.conv(b, 384, 384, 1, 3, pw=1, dst=(o, 1088, tot))
    g.conv(b, 384, 384, 3, 1, ph=1, dst=(o, 1472, tot))
    g.conv(g.pool(MPN_LAYER_AVGPOOL_WIN, x, 3, 1, 1, exclude_pad=xp), cin, 192, 1, 1, dst=(o, 1856, tot))
    return o, tot


def inception_v3_fast_rcnn(num_classes: int = 21, seed: int = 1234, integral_k: int = 0, exclude_pad: bool = True,
                           fixed_bn: bool = False) -> ModelSpec:
    """models/inceptionv3.lua on Moodstocks' inceptionv3.t7 (the conversion of Google's Inception-v3; block contents as
    recalled, parity unpinned). Every convolution is followed by batch norm (folded into conv + bias) and a ReLU.
      features 1..25 = the stem — conv 3x3/2 v 3 -> 32, 3x3 v 32 -> 32, 3x3 p1 32 -> 64, max pool 3x3/2 v, 1x1 64 -> 80,
                       3x3 v 80 -> 192, max pool 3x3/2 v — then Mixed_5b/5c/5d, Mixed_6a, Mixed_6b..6e: 17 x 17 x 768 at
                       299 px (stride ~17.6: ROIPooling(17, 17):setSpatialScale(17/299));
      classifier 26..30 = Mixed_7a, 7b, 7c, SpatialAveragePooling(8, 8) + View: one tower, 2048 features per ROI;
      classAndBBoxLinear(2048), ImageTransformer({1,1,1}, nil, 2) ("inception": 2 x - 1).
    Each Mixed block's branches write their channel slices of one slot (Layer.out_c_off / out_c_total); its 3 x 3 / 1 / 1
    average pools divide by the in-image count when exclude_pad (TensorFlow's SAME pooling, which the conversion
    carries over as setCountExcludePad), else by 9. integral_k as resnet*_fast_rcnn. fixed_bn: every convolution of the
    tower (Mixed_7a .. 7c) in the fixed-batch-norm form of inceptionv3.lua's BNtoFixed (scales in spec.fixed_bn), so that
    `Trainer` trains the tower and heads (the classifier, modules 26..30); the trunk stays folded and frozen. Without it
    the model runs inference only: training refuses."""
    W = _W(seed)
    rec = {} if fixed_bn else None
    xp = 1 if exclude_pad else 0
    g = _Graph(W, 1)
    x = g.conv(0, 3, 32, 3, 3, stride=2, gain=0.5)
    x = g.conv(x, 32, 32, 3, 3)
    x = g.conv(x, 32, 64, 3, 3, ph=1, pw=1)
    x = g.pool(MPN_LAYER_MAXPOOL, x, 3, 2, 0)
    x = g.conv(x, 64, 80, 1, 1)
    x = g.conv(x, 80, 192, 3, 3)
    x = g.pool(MPN_LAYER_MAXPOOL, x, 3, 2, 0)
    x, c = _mixed_5(g, x, 192, 32, xp)
    x, c = _mixed_5(g, x, c, 64, xp)
    x, c = _mixed_5(g, x, c, 64, xp)
    x, c = _mixed_6a(g, x, c)
    for cc in (128, 160, 160, 192):
        x, c = _mixed_6(g, x, c, cc, xp)
    trunk, tap = g.layers, x
    t = _Graph(W, 1, rec)
    y, c = _mixed_7a(t, 0, c)
    y, c = _mixed_7(t, y, c, xp)
    y, c = _mixed_7(t, y, c, xp)
    out = t.slot()
    t.layers.append(Layer(MPN_LAYER_AVGPOOL, y, out))
    tower = Tower(region=0, levels=[(tap, 17.0 / 299.0)], pooled_w=17, pooled_h=17, normalize=0, layers=t.layers, out_slot=out)
    cls = []
    for _ in range(max(integral_k, 1)):
        wc, bc = W.linear(num_classes, c, std=0.01, zero_bias=True)
        cls.append(Head(0, c, num_classes, wc, bc))
    wb, bb = W.linear(4 * num_classes, c, std=0.001, zero_bias=True)
    return ModelSpec(name="inception_v3_fast_rcnn", trunk_layers=trunk, towers=[tower], cls_heads=cls,
                     bbox_head=Head(0, c, 4 * num_classes, wb, bb), num_classes=num_classes, weights=W.arrays,
                     no_softmax=1 if integral_k > 0 else 0, transformer="inception", taps={"mixed_6e": tap}, fixed_bn=rec or {})


def is_inference_only(spec: ModelSpec) -> str:
    """'' when every layer of `spec` is what mpn_layer alone says; else the first layer that is not: CaffeNet's grouped
    convolutions and LRN layers (caffenet_layer), which never train here, or Inception-v3's layers (a windowed average pool,
    a convolution with a horizontal pad of its own, a branch of a concatenation), which train only in a tower with fixed
    batch norm, inception_v3_fast_rcnn(fixed_bn=True)"""
    for where, layers in [("trunk", spec.trunk_layers)] + [(f"tower {t}", T.layers) for t, T in enumerate(spec.towers)]:
        for i, L in enumerate(layers):
            if L.kind in (MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_LRN) or L.ext(0, 0) is not None:
                return f"{where} layer {i}"
    return ""


def caffenet_layer(spec: ModelSpec) -> str:
    """'' when `spec` has no grouped convolution and no LRN; else the first such layer (CaffeNet's conv2 / norm1 / ...), by
    name as the library names it. Such a model runs inference only: their backward is not built."""
    for where, layers in [("trunk", spec.trunk_layers)] + [(f"tower {t}", T.layers) for t, T in enumerate(spec.towers)]:
        for i, L in enumerate(layers):
            if L.kind == MPN_LAYER_LRN:
                return f"{where} layer {i} (LRN)"
            if L.groups != 1:
                return f"{where} layer {i} ({L.kh}x{L.kw} convolution {L.cin} -> {L.cout} in {L.groups} groups)"
    return ""


def svd_compress(spec: ModelSpec, ranks) -> ModelSpec:
    """utils.SVDlinear (models/model_utils.lua:56-77) on the per-ROI Linears of every tower: the truncated SVD of Fast
    R-CNN (Girshick 2015, section 3.1), a test-time transform. ranks[i] applies to the i-th layer after each tower's
    FLATTEN (fc6, fc7 of VGG-16 Fast R-CNN and of MultiPathNet's five towers), 0 = leave that layer as it is. A Linear
    W (K x N, bias b) becomes a biasless Linear N -> L holding (U_L diag(S_L))^T, with no ReLU, followed by a Linear L -> K
    holding V_L with the bias b and the original ReLU, where W^T = U S V^T (numpy's SVD in fp64), so that the product of
    the two factors is the best rank-L approximation of W. Returns a new spec; `spec` is not modified, and each tower
    factors its own weights. Raises ValueError for a rank that is negative, not a multiple of 64 (the engine's K blocks)
    or above min(N, K), for ranks that are all 0, and for a target that is not a Linear."""
    ranks = [int(r) for r in ranks]
    if not any(ranks):
        raise ValueError("svd_compress: every rank is 0, so there is nothing to factor")
    for r in ranks:
        if r < 0 or r % 64:
            raise ValueError(f"svd_compress: rank {r} must be a non-negative multiple of 64 (the engine's K blocks)")
    weights = list(spec.weights)                  # arrays are shared until replaced; none is written in place
    done = []                                     # (weight array, rank, (first factor, second factor)): towers with equal weights
    towers = []
    for ti, t in enumerate(spec.towers):
        fl = [i for i, L in enumerate(t.layers) if L.kind == MPN_LAYER_FLATTEN]
        layers = [Layer(**vars(L)) for L in t.layers]
        slot = max([t.out_slot] + [max(L.in_slot, L.out_slot) for L in t.layers]) + 1
        pos = {}
        if any(ranks) and not fl:
            raise ValueError(f"svd_compress: tower {ti} of {spec.name} has no FLATTEN, so no Linear to factor")
        for k, r in enumerate(ranks):
            if r == 0:
                continue
            i = fl[0] + 1 + k
            L = layers[i] if i < len(layers) else None
            if L is None or L.kind != MPN_LAYER_CONV or (L.kh, L.kw, L.stride, L.pad) != (1, 1, 1, 0) or L.residual_slot >= 0:
                raise ValueError(f"svd_compress: layer {k + 1} after the FLATTEN of tower {ti} of {spec.name} is not a Linear")
            w = spec.weights[L.weight]
            if r > min(L.cin, L.cout):
                raise ValueError(f"svd_compress: rank {r} of the {L.cin} -> {L.cout} Linear (tower {ti}) is above min(N, K) = "
                                 f"{min(L.cin, L.cout)}")
            hit = next((f for a, rr, f in done if rr == r and a.shape == w.shape and np.array_equal(a, w)), None)
            if hit is None:
                u, s, vt = np.linalg.svd(np.asarray(w, np.float64).reshape(L.cout, L.cin).T, full_matrices=False)
                hit = (np.ascontiguousarray((u[:, :r] * s[:r]).T, np.float32), np.ascontiguousarray(vt[:r].T, np.float32))
                done.append((w, r, hit))
            weights += [hit[0], hit[1]]
            w1, w2 = len(weights) - 2, len(weights) - 1
            pos[i] = (Layer(MPN_LAYER_CONV, L.in_slot, slot, cin=L.cin, cout=r, relu=0, weight=w1, bias=-1),
                      Layer(MPN_LAYER_CONV, slot, L.out_slot, cin=r, cout=L.cout, relu=L.relu, weight=w2, bias=L.bias))
            slot += 1
        new_layers = []
        for i, L in enumerate(layers):
            new_layers.extend(pos.get(i, (L,)))
        towers.append(Tower(region=t.region, levels=list(t.levels), pooled_w=t.pooled_w, pooled_h=t.pooled_h,
                            normalize=t.normalize, layers=new_layers, out_slot=t.out_slot))
    tag = "/".join(str(r) for r in ranks)
    return dataclasses.replace(spec, name=f"{spec.name}/svd{tag}", towers=towers, weights=weights)


def is_svd_compressed(spec: ModelSpec) -> bool:
    """True when a tower holds a Linear without a bias: the first factor svd_compress (or utils.SVDlinear's nn.LinearNB,
    imported by t7.model_from_t7) leaves behind"""
    return any(L.kind == MPN_LAYER_CONV and L.bias < 0 for t in spec.towers for L in t.layers)


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
            ho, wo = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.padw - L.kw) // L.stride + 1
            fl += 2.0 * L.cin * L.cout * L.kh * L.kw * ho * wo / L.groups      # a group sees Cin / groups input channels
        elif L.kind == MPN_LAYER_LRN:
            ho, wo = h, w
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
                ho, wo = (h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.padw - L.kw) // L.stride + 1
                fl += 2.0 * L.cin * L.cout * L.kh * L.kw * ho * wo
                shp[L.out_slot] = (ho, wo)
            elif L.kind in (MPN_LAYER_MAXPOOL, MPN_LAYER_AVGPOOL_WIN):
                shp[L.out_slot] = (_pool_out(h, L.kh, L.stride, L.pad, L.ceil_mode), _pool_out(w, L.kw, L.stride, L.pad, L.ceil_mode))
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

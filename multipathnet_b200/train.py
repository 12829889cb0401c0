"""Training on the device: train.lua's step (train.lua:221-370, engines/Optim.lua).

By default the per-ROI layers train and the trunk is frozen. For `models.vgg16_multipathnet` that is the whole of what
trains: the skip trunk sits under nn.NoBackprop (multipathnet.lua:60-62), so the parameters are each tower's conv_mix,
fc6 and fc7 and the two heads. `Trainer(model, train_trunk=True)` also trains the trunk layers from
`spec.trunk_train_from` upward: for `models.vgg16_fast_rcnn` that is conv3_1 .. conv5_3, the recipe of vgg.lua:18-19
(conv1_1 .. pool2 under nn.NoBackprop). A step takes a minibatch the caller built (`step`), or one that
`batch_provider.BatchProviderROI` sampled on the device from a dataset and its proposals (`step_batch`).

MultiPathNet's own recipe has two phases (multipathnet.lua:123-124, train.lua:239-269): `Trainer(model, phase2=True)`
runs phase 1 exactly as `Trainer(model)`, and `set_phase2(lr)` switches to phase 2, in which the trunk from
`spec.phase2_from` (conv3_1) trains as well, through every tower's foveal, normalised ROI pooling.

An integral model (K > 1 class heads, `integral_k`) trains, with `Trainer(model, integral=True)`, the integral loss of
train.lua:288-294: each step trains one class head, the one `select_head` picked for `step`, or the head of the batch's
threshold set for `step_batch` (`BatchProviderROI.sample_integral` draws that set per step). The other heads get a zero
gradient and still take optim.sgd's step, as Optim.lua updates every module.

A model with fixed batch norm (`spec.fixed_bn`, e.g. `models.resnet18_fast_rcnn(fixed_bn=True)`) trains as resnet.lua
does after BNtoFixed: each recorded convolution W is followed by the constant inn.ConstAffine y = a * x + b, so W
trains and a, b do not. The spec holds the folded W' = a * W, and everything here is in that parameterisation:
optim.sgd on W is run on W' with the gradient scaled by a^2 per output channel, and `weights`, `gradient` and
`momentum_buffer` report W', dL/dW' and a * (the buffer of W). For ResNets the trunk trains from layer2
(`spec.trunk_train_from`), layer4 and the heads per ROI. For Inception-v3 (`models.inception_v3_fast_rcnn(fixed_bn=True)`)
the tower Mixed_7a .. 7c and the heads train with the trunk frozen; its branches' concatenations, 1 x n / n x 1 kernels
and windowed average pools are checked with their mpn_layer_ext records (mpn_train_check_ext).

`Trainer(model, bf16=True)` is mixed-precision training: every convolution and Linear after the first layer, forward
and backward, issues one bf16 tensor-core product per MAC on rn_bf16 of its operands (the "bf16" inference numerics)
instead of the default three, which are faithful to fp32. Masters, momentum buffers, the update, the criteria, ROI
pooling and its backward stay fp32. Inference after it runs in the context's own numerics.

`Trainer(model, method="adam")` trains every tensor with train.lua's `method` (train.lua:64, :368): sgd (the default),
adam, adamax, adagrad or rmsprop, each with its own state, and `lr_decay` is train.lua's learningRateDecay
(engines/Optim.lua:46-81). The rules are restated as recalled, with the op order of csrc/train_rule.cuh; parity is
unpinned. Methods that cannot be reproduced are refused by name with the reason (`_REFUSED`).

`Trainer(model, replicas=(m_1, ..., m_{K-1}))` trains on K replicas at once, as train.lua's train_nGPU wraps the model in
nn.DataParallelTable: each step's images are split into K contiguous shards (`shard_plan`), each replica runs the
forward, criteria and backward of its shard, the gradients are summed over the replicas on the device in replica order,
and every replica runs the same update on the sum. The criteria divide by the whole minibatch's row count and the dropout
masks are keyed by the global row, so every row's logits, deltas and masks are those of a single trainer; the summed
gradients differ from it only by the order of fp32 additions. Every replica keeps the same masters and states.
"""
from __future__ import annotations

import ctypes as C
import dataclasses
import json
from typing import List, Sequence, Tuple

import numpy as np

from ._lib import CLayerExt, CTrainConfig, CTrainOptim, CTrainSpec, CTrainState, Model, MpnError, ModelSpec, _f32p, _i32p, _ptr, _vp, load_library
from .models import caffenet_layer, is_inference_only, is_svd_compressed

OPTIM_METHODS = {"sgd": 0, "adam": 1, "adamax": 2, "adagrad": 3, "rmsprop": 4}            # MPN_OPTIM_*
# optim's default epsilon per method (sgd has none; adagrad adds a fixed 1e-10 and reads no epsilon)
_EPSILON = {"sgd": 0.0, "adam": 1e-8, "adamax": 1e-38, "adagrad": 0.0, "rmsprop": 1e-8}
_DERIVATIVE_FREE = "a derivative-free method: it reads no gradient and evaluates the loss many times per step"
_REFUSED = {
    "nag": "optim.nag moves x by the momentum before it evaluates the gradient, and Optim.lua's fEvalMod returns the gradient "
           "taken before that move, so what the reference computes is an artefact",
    "adadelta": "whether optim.adadelta scales its step by learningRate changed between optim versions; with train.lua's "
                "config the two readings differ by 1000x",
    "asgd": "averaged SGD keeps a second, averaged copy of the weights that train.lua never reads",
    "rprop": "optim.rprop is a full-batch method; it steps on gradient signs that one minibatch does not give",
    "lbfgs": "optim.lbfgs is a full-batch method that evaluates the loss several times per step",
    "cg": "optim.cg is a full-batch method that evaluates the loss several times per step",
    "fista": "optim.FistaLS needs a proximal operator and a line search that evaluates the loss several times per step",
    "cmaes": _DERIVATIVE_FREE, "de": _DERIVATIVE_FREE,
}


def _train_optim(method: str = "sgd", lr_decay: float = 0.0, beta1: float = 0.9, beta2: float = 0.999, epsilon: float = None,
                 alpha: float = 0.99):
    """train.lua's `method` and learningRateDecay as the library's mpn_train_optim (epsilon None: the method's default),
    or MpnError for a method this training does not run; the ranges are the library's to check"""
    if method in _REFUSED:
        raise MpnError(f"optim method {method!r} is refused: {_REFUSED[method]}")
    if method not in OPTIM_METHODS:
        raise MpnError(f"unknown optim method {method!r}: one of {', '.join(OPTIM_METHODS)}")
    eps = _EPSILON[method] if epsilon is None else float(epsilon)
    return CTrainOptim(OPTIM_METHODS[method], float(lr_decay), float(beta1), float(beta2), eps, float(alpha))


def _train_spec(spec: ModelSpec, trunk_from: int, integral: bool, phase2: bool):
    """what trains, as the library's mpn_train_spec (phase2: the trunk range from spec.phase2_from, idle until the
    switch; spec.fixed_bn as the records), and the arrays it points into, which must outlive the call"""
    idx = np.array(sorted(spec.fixed_bn), np.int32)
    scales = [np.ascontiguousarray(spec.fixed_bn[int(i)], np.float32).reshape(-1) for i in idx]
    for i, a in zip(idx, scales):
        if a.shape[0] != spec.weights[int(i)].shape[0]:
            raise MpnError(f"fixed_bn: the scale of weight {int(i)} has {a.shape[0]} entries for {spec.weights[int(i)].shape[0]} output channels")
    ptrs = (_vp * max(len(scales), 1))(*[a.ctypes.data for a in scales])
    s = CTrainSpec(int(spec.phase2_from) if phase2 else int(trunk_from), int(bool(phase2)), int(bool(integral)), len(idx),
                   idx.ctypes.data_as(_i32p), ptrs)
    return s, (idx, scales, ptrs)


def _refuse_caffenet(spec: ModelSpec) -> None:
    where = caffenet_layer(spec)
    if where:
        raise MpnError(f"training: {spec.name} has CaffeNet's layers (first: {where}), which run inference only here: the "
                       "backward of a grouped convolution or an LRN is not built")


def check_spec(spec: ModelSpec, trunk_from: int = 0, integral: bool = False, phase2: bool = False, optim: dict = None) -> None:
    """raise MpnError unless every per-ROI layer of `spec` is a 1x1 convolution, FLATTEN or Linear with one class head
    (integral: K class heads over the same columns, trained with the integral loss), and, for trunk_from > 0, the trunk
    layers from trunk_from up can train (the library's own check, mpn_train_check; no GPU needed). With spec.fixed_bn,
    the recorded convolutions may also be 3x3, stride 2 or residual, and a tower may end in a global AVGPOOL. phase2:
    the trunk layers from spec.phase2_from up can train in MultiPathNet's phase 2, through every tower's foveal,
    normalised pooling (trunk_from is not read); a model with fixed batch norm has no phase 2. optim: the Trainer's
    optimiser keywords (method, lr_decay, beta1, beta2, epsilon, alpha); None is sgd with lr_decay 0. They are checked
    first. An SVD-compressed model (models.svd_compress, utils.SVDlinear) is refused: the factoring is a test-time
    transform, and the backward of its biasless factors is not part of the training step."""
    if is_svd_compressed(spec):
        raise MpnError(f"training: {spec.name} is SVD-compressed (a tower Linear without a bias, as svd_compress and "
                       "utils.SVDlinear leave): factor a trained model for testing instead")
    _refuse_caffenet(spec)
    where = is_inference_only(spec)
    if where and not spec.fixed_bn:
        raise MpnError(f"training: {spec.name} has Inception-v3's layers (first: {where}: a windowed average pool, a 1 x n / n x 1 "
                       "kernel or a branch of a concatenation), which run inference only here")
    o = _train_optim(**(optim or {}))
    d, _keep = Model.build_desc(spec, grouped=True)
    s, _arrays = _train_spec(spec, trunk_from, integral, phase2)
    ext = Model.layer_ext(spec)
    recs = (CLayerExt * max(len(ext), 1))(*ext)
    msg = C.create_string_buffer(512)
    if load_library().mpn_train_check_ext(C.byref(d), recs, len(ext), C.byref(s), C.byref(o), msg, len(msg)) != 0:
        raise MpnError(msg.value.decode())


def shard_plan(rois_per_image: Sequence[int], k: int) -> List[Tuple[int, int, int, int]]:
    """train_nGPU's split of one minibatch over k replicas, along the batch as nn.DataParallelTable scatters it: replica j
    takes images j * n / k .. (j + 1) * n / k - 1 and their rows, as (first image, end image, first row, end row). MpnError
    when k does not divide the image count (train.lua:101) or a shard has no rows."""
    counts = [int(c) for c in rois_per_image]
    n, k = len(counts), int(k)
    if k < 1:
        raise MpnError("replicas: at least one")
    if n < 1 or n % k != 0:
        raise MpnError(f"images_per_batch must be a multiple of train_nGPU: {n} images over {k} replicas")
    per, out, row = n // k, [], 0
    for j in range(k):
        r = sum(counts[j * per:(j + 1) * per])
        if r <= 0:
            raise MpnError(f"training shard: replica {j}'s images {j * per}..{(j + 1) * per - 1} have no ROIs")
        out.append((j * per, (j + 1) * per, row, row + r))
        row += r
    return out


def _same_spec(a: ModelSpec, b: ModelSpec) -> bool:
    if a is b:
        return True
    for f in dataclasses.fields(ModelSpec):
        x, y = getattr(a, f.name), getattr(b, f.name)
        if f.name == "weights":
            if len(x) != len(y) or any(u is not v and (np.shape(u) != np.shape(v) or not np.array_equal(u, v)) for u, v in zip(x, y)):
                return False
        elif f.name == "fixed_bn":
            if sorted(x) != sorted(y) or any(not np.array_equal(x[i], y[i]) for i in x):
                return False
        elif x != y:
            return False
    return True


def check_replicas(model, replicas: Sequence) -> None:
    """MpnError unless every replica is another Model of model's spec (same description and weights)"""
    seen = [model]
    for j, r in enumerate(replicas, 1):
        if any(r is m for m in seen):
            raise MpnError(f"replicas: replica {j} is the same Model as replica {[m is r for m in seen].index(True)}")
        if not _same_spec(model.spec, r.spec):
            raise MpnError(f"replicas: replica {j} has another spec than the model ({r.spec.name} / {model.spec.name}, or other "
                           "layers or weights)")
        seen.append(r)


def check_step(spec: ModelSpec, limits: Tuple[int, int, int], images, rois_per_image, labels, bbox_targets):
    """the arguments of one step as contiguous arrays, or MpnError: images 3 x H_i x W_i within max_h x max_w, R x 4 ROIs
    per image, 0 < R <= max_rois, labels in 1..C, bbox_targets R x 4C"""
    max_rois, max_h, max_w = limits
    if len(images) < 1 or len(images) != len(rois_per_image):
        raise MpnError("training step: one ROI array per image, at least one image")
    ims = [np.ascontiguousarray(im, np.float32) for im in images]
    for im in ims:
        if im.ndim != 3 or im.shape[0] != 3:
            raise MpnError("training step: images are 3 x H x W")
        if im.shape[1] > max_h or im.shape[2] > max_w:
            raise MpnError(f"training step: image {im.shape[1]} x {im.shape[2]} is larger than max_h x max_w = {max_h} x {max_w}")
    rois = [np.ascontiguousarray(r, np.float32).reshape(-1, 4) for r in rois_per_image]
    R = sum(r.shape[0] for r in rois)
    if R < 1 or R > max_rois:
        raise MpnError(f"training step: R = {R} out of range (0 < R <= max_rois = {max_rois})")
    C_ = spec.num_classes
    lab = np.ascontiguousarray(labels, np.int32).reshape(-1)
    if lab.shape[0] != R:
        raise MpnError(f"training step: {lab.shape[0]} labels for {R} ROIs")
    if lab.min() < 1 or lab.max() > C_:
        raise MpnError(f"training step: labels must lie in 1..{C_} (1 = background)")
    tg = np.ascontiguousarray(bbox_targets, np.float32)
    if tg.shape != (R, 4 * C_):
        raise MpnError(f"training step: bbox_targets must be {R} x {4 * C_}, got {tg.shape}")
    return ims, np.concatenate(rois, 0), lab, tg


class Trainer:
    """SGD on the per-ROI layers of `model` (an mpn.Model that has not run a heads / detect call yet). Defaults are
    train.lua's: lr 1e-3, momentum 0.9, dampening 0, weight decay 5e-4 (0 for biases), dropout p = 0.5 after fc6 / fc7
    (0 = train_remove_dropouts), bbox_regression 1. After each step every inference call of `model` uses the new weights;
    the step leaves no cached trunk features, so `heads` / `detect(recompute_features=False)` need a trunk call first.
    train_trunk: also train the trunk layers from `model.spec.trunk_train_from` up (MpnError when that is 0); the model
    must not have run a trunk call yet either. integral: train an integral model (K > 1 class heads) with the integral
    loss, one head per step (`select_head`, or the batch's set in `step_batch`); without it such a model is refused.
    phase2: a two-phase MultiPathNet run (multipathnet.lua:123-124, train.lua:239-269). Until `set_phase2` it is exactly
    `Trainer(model)`; the fp32 weights of the trunk layers from `model.spec.phase2_from` up are kept on the device, so the
    model must not have run a trunk call yet; after the switch those layers train too. Composes with `integral`.
    bf16: mixed-precision training (the context option "train_bf16", set around the begin call and then restored): one
    bf16 product per MAC in every forward and backward GEMM of the step. Composes with every option above; a checkpoint
    of one numerics does not load into a trainer of the other.
    method: train.lua's optim method for every tensor, "sgd", "adam", "adamax", "adagrad" or "rmsprop" (momentum and
    dampening are sgd's only); lr_decay: learningRateDecay, clr = lr / (1 + t * lr_decay) for sgd, adam and adagrad
    (adamax and rmsprop ignore it, as optim does); beta1, beta2 (adam, adamax), alpha (rmsprop) and epsilon (adam, adamax,
    rmsprop; None: optim's default, 1e-8 or adamax's 1e-38). Composes with every option above; a checkpoint of one
    method or setting does not load into a trainer of another.
    replicas: further Models of model's spec (same description and weights, any contexts and devices) that have run no
    trunk, heads or detect call; each step is split over the K = 1 + len(replicas) models (`shard_plan`) and their
    gradients summed. `model` is replica 0: the getters read it (the gradient is the sum), `dropout_mask`, `relu_gate` and
    `outputs` join the replicas' rows in order, and the setters set every replica. The checkpoint is that of a single
    trainer, so it loads into a trainer with any number of replicas."""

    method = "sgd"       # the class-level default: what a Trainer built without __init__ reads

    def __init__(self, model: Model, lr: float = 1e-3, momentum: float = 0.9, weight_decay: float = 5e-4, dampening: float = 0.0,
                 dropout: float = 0.5, bbox_regression: float = 1.0, seed: int = 555, train_trunk: bool = False,
                 integral: bool = False, phase2: bool = False, bf16: bool = False, method: str = "sgd", lr_decay: float = 0.0,
                 beta1: float = 0.9, beta2: float = 0.999, epsilon: float = None, alpha: float = 0.99, replicas: Sequence[Model] = ()):
        trunk_from = 0
        replicas = list(replicas)
        check_replicas(model, replicas)
        for j, r in enumerate(replicas, 1):
            n = C.c_int32()
            r.ctx.check(r.ctx.lib.mpn_model_weights_prepared(r.h, C.byref(n)), "mpn_model_weights_prepared")
            if n.value:
                raise MpnError(f"replicas: replica {j} already ran inference (a trunk, heads or detect call); a replica must be a "
                               "fresh Model")
        _refuse_caffenet(model.spec)
        if train_trunk and phase2:
            raise MpnError("train_trunk and phase2 exclude each other: phase 2 trains the trunk from set_phase2 on")
        if train_trunk:
            trunk_from = int(model.spec.trunk_train_from)
            if trunk_from == 0 and is_inference_only(model.spec):
                raise MpnError(f"train_trunk: the trunk of {model.spec.name} does not train here: Inception-v3's Mixed_5b .. 6e "
                               "hold layers that read 48, 96, 160 and 288 channels, K tails whose backward is not built; its "
                               "tower and heads train with Trainer(model) on a fixed_bn=True spec")
            if trunk_from == 0:
                raise MpnError(f"train_trunk: the trunk of {model.spec.name} does not train (spec.trunk_train_from is 0)")
        optim = dict(method=method, lr_decay=lr_decay, beta1=beta1, beta2=beta2, epsilon=epsilon, alpha=alpha)
        check_spec(model.spec, trunk_from, integral, phase2, optim)
        o = _train_optim(**optim)
        if not (0.0 <= dropout < 1.0):
            raise MpnError("dropout p must lie in [0, 1)")
        self.model, self.ctx = model, model.ctx
        self.models = [model] + replicas
        self._handles = (_vp * len(self.models))(*[m.h.value for m in self.models])
        self.trunk_from = trunk_from
        self.cfg = CTrainConfig(float(lr), float(momentum), float(dampening), float(weight_decay), float(dropout), float(bbox_regression),
                                int(seed) & 0xFFFFFFFFFFFFFFFF)
        s, _arrays = _train_spec(model.spec, trunk_from, integral, phase2)
        for j, m in enumerate(self.models):
            # the library has no getter for an option: the previous value is what Context.set_option last set (-1, the
            # default, when it was never set that way). A value set straight through mpn_ctx_set_option is restored as -1.
            prev = m.ctx.options.get("train_bf16", -1)
            m.ctx.set_option("train_bf16", 1 if bf16 else -1)
            try:
                m.ctx.check(m.ctx.lib.mpn_model_train_begin_optim(m.h, C.byref(self.cfg), C.byref(s), C.byref(o)),
                            "mpn_model_train_begin_optim" + (f" (replica {j})" if j else ""))
            except MpnError:
                for done in self.models[:j]:
                    done.ctx.lib.mpn_model_train_end(done.h)
                raise
            finally:
                m.ctx.set_option("train_bf16", prev)
        self.bf16 = bool(bf16)
        self.phase2 = bool(phase2)
        self.phase = 1
        self.trained = sorted(self._trained_indices())
        self.steps = 0
        self.head = 0
        self._fingerprint = {"name": model.spec.name, "shapes": [list(np.shape(w)) for w in model.spec.weights], "trained": list(self.trained),
                             "trunk_from": trunk_from, "phase2_from": int(model.spec.phase2_from) if phase2 else 0,
                             "integral_k": len(model.spec.cls_heads), "fixed_bn": sorted(int(i) for i in model.spec.fixed_bn)}
        if self.bf16:              # a default checkpoint has no such key: it reads as False
            self._fingerprint["bf16"] = True
        self.method = method
        if method != "sgd" or o.lr_decay != 0:      # likewise: a missing key reads as sgd with lr_decay 0
            self._fingerprint["optim"] = {k: getattr(o, k) for k, _ in CTrainOptim._fields_ if k != "method"}
            self._fingerprint["optim"]["method"] = method

    @property
    def _n_states(self) -> int:
        """the method's state tensors per trained tensor: adam's m, v and adamax's m, u; one for the others"""
        return 2 if self.method in ("adam", "adamax") else 1

    def _each(self, fn: str, *args):
        """the library call fn(model, *args) on every replica"""
        for m in self.models:
            m.ctx.check(getattr(m.ctx.lib, fn)(m.h, *args), fn)

    def select_head(self, k: int):
        """the class head (0 .. K-1) that the following `step` calls train; head 0 until called"""
        self._each("mpn_model_train_select_head", int(k))
        self.head = int(k)

    def _trained_indices(self, trunk_from: int = None) -> List[int]:
        s = self.model.spec
        trunk_from = self.trunk_from if trunk_from is None else trunk_from
        out = []

        def layer(L):               # a fixed-batch-norm layer's bias is the constant b
            return [i for i in (L.weight, -1 if L.weight in s.fixed_bn else L.bias) if i >= 0]
        for t in s.towers:
            for L in t.layers:
                out += layer(L)
        for h in (*s.cls_heads, s.bbox_head):
            out += [i for i in (h.weight, h.bias) if i >= 0]
        if trunk_from > 0:
            for L in s.trunk_layers[trunk_from:]:
                out += layer(L)
        return out

    def step(self, images: Sequence[np.ndarray], rois_per_image: Sequence[np.ndarray], labels, bbox_targets) -> Tuple[float, float, float]:
        """one minibatch: images (transformed, 3 x H_i x W_i), per image its R_i x 4 ROIs in scaled-image coordinates,
        labels (R, 1..C), bbox_targets (R x 4C, normalised) -> (loss, cls_loss, bbox_loss)"""
        ims, rois, lab, tg = check_step(self.model.spec, self.model.limits, images, rois_per_image, labels, bbox_targets)
        n = len(ims)
        ptrs = (_vp * n)(*[im.ctypes.data for im in ims])
        hw = np.array([[im.shape[1], im.shape[2]] for im in ims], np.int32).reshape(-1)
        counts = np.array([np.asarray(r).reshape(-1, 4).shape[0] for r in rois_per_image], np.int32)
        losses = np.zeros(3, np.float32)
        if len(self.models) > 1:
            shard_plan(counts, len(self.models))
            self.ctx.check(self.ctx.lib.mpn_model_train_step_replicas(self._handles, len(self.models), n, ptrs, hw.ctypes.data_as(_i32p),
                                                                      counts.ctypes.data_as(_i32p), _ptr(rois), _ptr(lab), _ptr(tg),
                                                                      _ptr(losses)), "mpn_model_train_step_replicas")
            self._last_counts = counts
            self.steps += 1
            return float(losses[0]), float(losses[1]), float(losses[2])
        self.ctx.check(self.ctx.lib.mpn_model_train_step(self.model.h, n, ptrs, hw.ctypes.data_as(_i32p), counts.ctypes.data_as(_i32p),
                                                         _ptr(rois), _ptr(lab), _ptr(tg), _ptr(losses)), "mpn_model_train_step")
        self.steps += 1
        return float(losses[0]), float(losses[1]), float(losses[2])

    def step_batch(self, batch) -> Tuple[float, float, float]:
        """one minibatch that BatchProviderROI.sample left on the device (same ctx as the model) -> (loss, cls_loss,
        bbox_loss); the batch is used in place, nothing is copied to the host. An integral model trains head `batch.set`
        (and keeps it selected); its RoiDB must have one threshold set per class head."""
        max_rois, max_h, max_w = self.model.limits
        batch.check_current()
        if batch.roidb.ctx is not self.ctx:
            raise MpnError("step_batch: the batch was sampled on another context")
        K = len(self.model.spec.cls_heads)
        if K > 1 and len(batch.roidb.thresholds) != K:
            raise MpnError(f"step_batch: the RoiDB has {len(batch.roidb.thresholds)} threshold sets and the model {K} class heads; "
                           "an integral model trains head s on set s")
        if self.model.spec.num_classes != batch.num_classes:
            raise MpnError(f"step_batch: the model has {self.model.spec.num_classes} classes, the dataset {batch.num_classes - 1} + background")
        if not 0 < batch.R <= max_rois:
            raise MpnError(f"training step: R = {batch.R} out of range (0 < R <= max_rois = {max_rois})")
        for h, w in batch.image_hw:
            if h > max_h or w > max_w:
                raise MpnError(f"training step: image {h} x {w} is larger than max_h x max_w = {max_h} x {max_w}")
        losses = np.zeros(3, np.float32)
        if len(self.models) > 1:
            shard_plan(batch.rois_per_image, len(self.models))
            for m in self.models:
                if m.spec.num_classes != batch.num_classes:
                    raise MpnError(f"step_batch: a replica has {m.spec.num_classes} classes, the dataset {batch.num_classes - 1} + background")
            self.ctx.check(self.ctx.lib.mpn_model_train_step_batch_replicas(self._handles, len(self.models), batch.roidb.h, _ptr(losses)),
                           "mpn_model_train_step_batch_replicas")
            self._last_counts = np.asarray(batch.rois_per_image, np.int32)
        else:
            self.ctx.check(self.ctx.lib.mpn_model_train_step_batch(self.model.h, batch.roidb.h, _ptr(losses)), "mpn_model_train_step_batch")
        if K > 1:
            self.head = int(batch.set)
        self.steps += 1
        return float(losses[0]), float(losses[1]), float(losses[2])

    def set_phase2(self, lr: float = None):
        """switch a `Trainer(phase2=True)` run to phase 2 (train.lua:239-260, utils.vggSetPhase2_outer): from the next step
        the trunk layers from spec.phase2_from up train. lr: the new learning rate, and under sgd every momentum buffer is
        zeroed (phase2_learningRate >= 0; the other methods keep their state); None keeps both. The trunk tensors join
        with zero state and the ordinary update.
        Before the first step it starts the run in phase 2. phase2_step / phase2_decay stay the caller's schedule (`decay`)."""
        if not self.phase2:
            raise MpnError("set_phase2: the trainer was not made with phase2=True")
        self._each("mpn_model_train_phase2", -1.0 if lr is None else float(lr))
        if lr is not None:
            self.cfg.lr = float(lr)
        self.trunk_from = int(self.model.spec.phase2_from)
        self.phase = 2
        self.trained = sorted(self._trained_indices())

    def set_lr(self, lr: float):
        self._each("mpn_model_train_set_lr", float(lr))
        self.cfg.lr = float(lr)

    def decay(self, factor: float):
        """train.lua's onEndEpoch: lr and, under sgd, every momentum buffer times `factor` (the other methods' state is
        not the u.dfdx train.lua scales: only the rate changes)"""
        self._each("mpn_model_train_decay", float(factor))
        self.cfg.lr = float(np.float32(self.cfg.lr) * np.float32(factor))

    def _get(self, i: int, what: int) -> np.ndarray:
        shape = self.model.spec.weights[i].shape
        out = np.empty(shape, np.float32)
        self.ctx.check(self.ctx.lib.mpn_model_train_get(self.model.h, int(i), int(what), _ptr(out), out.size), "mpn_model_train_get")
        return out

    def weights(self) -> List[np.ndarray]:
        """every weight of the model in the spec's order and Torch layout (Cout x Cin x kh x kw, out x in): the trained ones
        read back from the device, the frozen trunk's (and fixed-batch-norm biases) as given. A fixed-batch-norm layer's
        weight is the folded W' = a * W, as the spec stores it."""
        return [self._get(i, 0) if i in self.trained else np.array(w, np.float32, copy=True)
                for i, w in enumerate(self.model.spec.weights)]

    def gradient(self, i: int) -> np.ndarray:
        """gradient of weight-table entry i from the last step (Torch layout); zero for the class heads it did not train.
        For a fixed-batch-norm layer, dL/dW' of the folded weight (dL/dW = a * dL/dW')."""
        return self._get(i, 1)

    def momentum_buffer(self, i: int) -> np.ndarray:
        """optim.sgd's buffer of entry i; for a fixed-batch-norm layer a * (the buffer of W), the buffer of W'"""
        return self._get(i, 2)

    def optim_state(self, i: int) -> Tuple[np.ndarray, ...]:
        """the optim method's state of entry i: (buf,) for sgd, (m, v) for adam, (m, u) for adamax, (s,) for adagrad, (m,)
        for rmsprop. For a fixed-batch-norm layer, sgd's buffer is that of W'; the other methods' state is that of W."""
        return tuple(self._get(i, 2 + k) for k in range(self._n_states))

    def _rows(self, fn: str, tower: int, layer: int) -> np.ndarray:
        """a per-row test hook (dropout mask, ReLU gate) of every replica, the rows joined in replica order"""
        outs = []
        cout = self.model.spec.towers[tower].layers[layer].cout
        for m in self.models:
            n = C.c_int64()
            m.ctx.check(getattr(m.ctx.lib, fn)(m.h, tower, layer, None, 0, C.byref(n)), fn)
            out = np.empty((n.value // cout, cout), np.uint8)
            m.ctx.check(getattr(m.ctx.lib, fn)(m.h, tower, layer, _ptr(out), out.size, C.byref(n)), fn)
            outs.append(out)
        return outs[0] if len(outs) == 1 else np.concatenate(outs, 0)

    def dropout_mask(self, tower: int, layer: int) -> np.ndarray:
        """the R x cout keep mask the last step applied after layer `layer` (index in the tower's layer list) of `tower`"""
        return self._rows("mpn_model_train_dropout_mask", tower, layer)

    def relu_gate(self, tower: int, layer: int) -> np.ndarray:
        """the last step's backward gate through the ReLU of layer `layer` of `tower` (stored output > 0, after dropout):
        rows (R x pixels) x cout"""
        return self._rows("mpn_model_train_relu_gate", tower, layer)

    def outputs(self):
        """the last step's raw logits (R x C, of the head it trained) and raw bbox deltas (R x 4C)"""
        cls_all, bbox_all = [], []
        for m in self.models:
            R, bins, ct = C.c_int64(), C.c_int32(), C.c_int32()       # R: the pooled tensor's row count
            m.ctx.check(m.ctx.lib.mpn_model_get_pooled(m.h, 0, 0, 0, None, 0, C.byref(R), C.byref(bins), C.byref(ct)), "get_pooled")
            cls = np.empty((R.value, m.C), np.float32)
            bbox = np.empty((R.value, 4 * m.C), np.float32)
            m.ctx.check(m.ctx.lib.mpn_model_train_outputs(m.h, _ptr(cls), _ptr(bbox)), "mpn_model_train_outputs")
            cls_all.append(cls)
            bbox_all.append(bbox)
        if len(self.models) == 1:
            return cls_all[0], bbox_all[0]
        return np.concatenate(cls_all, 0), np.concatenate(bbox_all, 0)

    def trunk_slot(self, image: int, slot: int) -> np.ndarray:
        """image `image`'s stored activation of trunk slot `slot` from the last step (C x H x W); kept are layer
        trunk_train_from's input and every slot written at or above it"""
        m = self.model
        if len(self.models) > 1 and getattr(self, "_last_counts", None) is not None:
            per = len(self._last_counts) // len(self.models)       # image `image` went to replica image // per
            m, image = self.models[int(image) // per], int(image) % per
        c, h, w = C.c_int32(), C.c_int32(), C.c_int32()
        lib = m.ctx.lib
        m.ctx.check(lib.mpn_model_train_trunk_slot(m.h, image, slot, None, 0, C.byref(c), C.byref(h), C.byref(w)), "trunk_slot")
        out = np.empty((c.value, h.value, w.value), np.float32)
        m.ctx.check(lib.mpn_model_train_trunk_slot(m.h, image, slot, _ptr(out), out.size, None, None, None), "trunk_slot")
        return out

    def allreduce_ms(self) -> float:
        """replica 0's device time of the last step's gradient reduction (MpnError with one replica: none runs)"""
        ms = np.zeros(1, np.float32)
        self.ctx.check(self.ctx.lib.mpn_model_train_allreduce_ms(self.model.h, ms.ctypes.data_as(_f32p)), "mpn_model_train_allreduce_ms")
        return float(ms[0])

    def _set(self, i: int, what: int, a) -> None:
        a = np.ascontiguousarray(a, np.float32)
        self._each("mpn_model_train_set", int(i), int(what), _ptr(a), a.size)

    def _zero_buffers(self) -> None:
        """every momentum buffer zeroed (train.lua:248-258 at the phase-2 epoch of a model without phase 2); train.lua
        zeroes u.dfdx, which only sgd's state has, so under the other methods nothing changes"""
        if self.method != "sgd":
            return
        for i in self.trained:
            self._set(i, 2, np.zeros(self.model.spec.weights[i].shape, np.float32))

    def state_dict(self) -> dict:
        """what resuming this training needs, as train.lua's checkpoint keeps it (model + optimState): the fingerprint of
        the spec and the trainer's setup, the config, the scalars (steps done, lr in force, class heads, phase 2) and the
        master and the optim state (momentum buffer, or the method's one or two states) of every trained tensor. `load_state_dict` on a fresh Trainer of the same spec and
        setup then continues bit for bit: the same losses, weights, buffers and dropout masks as an uninterrupted run."""
        st = CTrainState()
        self.ctx.check(self.ctx.lib.mpn_model_train_get_state(self.model.h, C.byref(st)), "mpn_model_train_get_state")
        return {"fingerprint": dict(self._fingerprint),
                "config": {k: getattr(self.cfg, k) for k, _ in CTrainConfig._fields_},
                "state": {"step": int(st.step), "lr": float(st.lr), "head": int(st.head), "last_head": int(st.last_head),
                          "phase2": int(st.phase2), "steps": int(self.steps)},
                "tensors": {int(i): (self._get(i, 0),) + self.optim_state(i) for i in self.trained}}

    def load_state_dict(self, d: dict) -> None:
        """apply a `state_dict`; MpnError (and nothing changed) on a fingerprint, config or tensor mismatch"""
        mine = bool(self._fingerprint.get("bf16", False))          # a missing key is the default numerics
        if bool(d["fingerprint"].get("bf16", False)) != mine:
            raise MpnError(f"load_state_dict: the checkpoint was trained with bf16={not mine}, this trainer has bf16={mine}")
        mine, theirs = self._fingerprint.get("optim"), d["fingerprint"].get("optim")     # missing: sgd, lr_decay 0
        if theirs != mine:
            raise MpnError(f"load_state_dict: the checkpoint's optim is {theirs or 'sgd with lr_decay 0'}, this trainer's "
                           f"{mine or 'sgd with lr_decay 0'}")
        for k, v in self._fingerprint.items():
            if d["fingerprint"].get(k) != v:
                raise MpnError(f"load_state_dict: the checkpoint's {k} is {d['fingerprint'].get(k)!r}, this trainer's {v!r}")
        for k, _ in CTrainConfig._fields_:
            if k != "lr" and d["config"].get(k) != getattr(self.cfg, k):
                raise MpnError(f"load_state_dict: the checkpoint's config {k} is {d['config'].get(k)!r}, this trainer's {getattr(self.cfg, k)!r}")
        s = d["state"]
        phase2 = bool(s["phase2"])
        if phase2 and not self.phase2:
            raise MpnError("load_state_dict: the checkpoint is in phase 2 and the trainer was not made with phase2=True")
        if self.phase == 2 and not phase2:
            raise MpnError("load_state_dict: the trainer is in phase 2 and the checkpoint in phase 1")
        trunk_from = int(self.model.spec.phase2_from) if phase2 else self.trunk_from
        want = sorted(self._trained_indices(trunk_from))
        if sorted(int(i) for i in d["tensors"]) != want:
            raise MpnError(f"load_state_dict: the checkpoint holds tensors {sorted(d['tensors'])}, the trainer trains {want}")
        for i, ts in d["tensors"].items():
            shape = tuple(self.model.spec.weights[int(i)].shape)
            if len(ts) != 1 + self._n_states:
                raise MpnError(f"load_state_dict: tensor {i} has {len(ts) - 1} optim states in the checkpoint, {self.method} keeps "
                               f"{self._n_states}")
            if any(tuple(np.shape(a)) != shape for a in ts):
                raise MpnError(f"load_state_dict: tensor {i} is {' / '.join(str(np.shape(a)) for a in ts)} in the checkpoint, {shape} here")
        st = CTrainState(int(s["step"]), float(s["lr"]), int(s["head"]), int(s["last_head"]), int(phase2))
        self._each("mpn_model_train_set_state", C.byref(st))
        if phase2:
            self.trunk_from, self.phase, self.trained = trunk_from, 2, want
        for i, ts in d["tensors"].items():
            for what, a in zip((0, 2, 3), ts):
                self._set(int(i), what, a)
        self.cfg.lr = float(s["lr"])
        self.head, self.steps = int(s["head"]), int(s["steps"])

    def close(self):
        for m in getattr(self, "models", [self.model]):
            if getattr(m, "h", None):
                m.ctx.check(m.ctx.lib.mpn_model_train_end(m.h), "mpn_model_train_end")


def save_checkpoint(path: str, trainer: Trainer, **extra) -> None:
    """trainer.state_dict() as one .npz: the tensors as arrays w<i> (master), b<i> (momentum buffer or the method's first
    state) and, for adam / adamax, c<i> (the second state), everything else,
    with `extra` (the training loop's own state: epoch, step / decay in force, the provider's bbox_regr mean / std ...,
    numpy arrays as lists), as one JSON string"""
    d = trainer.state_dict()
    tensors = d.pop("tensors")
    d["extra"] = {k: (v.tolist() if isinstance(v, np.ndarray) else v) for k, v in extra.items()}
    arrays = {"meta": np.array(json.dumps(d))}
    for i, ts in tensors.items():
        for key, a in zip("wbc", ts):
            arrays[f"{key}{i}"] = a
    with open(path, "wb") as f:
        np.savez(f, **arrays)


def load_checkpoint(path: str) -> dict:
    """a `save_checkpoint` file -> the state dict (for Trainer.load_state_dict) with its "extra" entry"""
    with np.load(path, allow_pickle=False) as z:
        d = json.loads(str(z["meta"]))
        idx = sorted(int(k[1:]) for k in z.files if k.startswith("w"))
        d["tensors"] = {i: (z[f"w{i}"], z[f"b{i}"]) + ((z[f"c{i}"],) if f"c{i}" in z.files else ()) for i in idx}
    return d

"""Torch-7 binary serialisation (`torch.save` / `torch.load`, torch7 File.lua) without Torch — SURVEY 8f-4.

The reference keeps its models and proposals in `.t7` files (`test_runner.lua:31`: `torch.load(opt.test_model)`;
proposals `{boxes, scores, images}`, `DataSetJSON.lua:124-239`). This module reads that format into plain Python / numpy
so real weights and proposals can be fed to the GPU path, and writes it (the subset below) so the reader can be tested
without Torch. PARITY UNPINNED: no `.t7` file and no Torch exist in the build image, so the format is restated from
torch7's public File.lua / Tensor / Storage `read`-`write` methods and pinned only by round trips through this module's
own writer (tests/test_t7_cpu.py); the first real file is the real test.

Format (little-endian, "binary" mode): every object starts with an int32 type tag
  0 nil | 1 number (float64) | 2 string (int32 length + bytes) | 3 table | 4 torch object | 5 boolean (int32)
  | 6/7/8 function (skipped: int32 size + bytecode + upvalue table).
Tables and torch objects are memoised: an int32 index follows the tag, and a repeated index means "the same object".
  table : int32 n, then n x (key object, value object)
  torch : version string "V 1" (int32 length + bytes), class name string, then the class payload:
          torch.*Tensor  : int32 ndim, int64 size[ndim], int64 stride[ndim], int64 storage offset (1-based), storage object
          torch.*Storage : int64 n, then n raw elements
          anything else (nn modules, ...): one object (a table) whose pairs become the fields — except classes with
          their own __write: nn.ModelParallelTable (ModelParallelTable.lua:607-628) and cunn's nn.DataParallelTable
          write the gpuAssignments table, the branch modules one by one, then the table of the remaining fields.
"""
from __future__ import annotations

import struct
from typing import Any, BinaryIO, Dict, List

import numpy as np

TYPE_NIL, TYPE_NUMBER, TYPE_STRING, TYPE_TABLE, TYPE_TORCH, TYPE_BOOLEAN, TYPE_FUNCTION, TYPE_LEGACY_RECUR_FUNCTION, TYPE_RECUR_FUNCTION = range(9)

_DTYPES = {"Float": np.float32, "Double": np.float64, "Long": np.int64, "Int": np.int32, "Short": np.int16,
           "Byte": np.uint8, "Char": np.int8, "CudaTensor": np.float32, "Cuda": np.float32, "Half": np.float16}


class T7Object:
    """A torch class instance that is not a tensor / storage (nn modules, ...): `typename` + its fields."""

    def __init__(self, typename: str, fields: Dict[Any, Any] = None):
        self.typename = typename
        self.fields = {} if fields is None else fields

    def __getattr__(self, k):
        f = self.__dict__.get("fields", {})
        if k in f:
            return f[k]
        raise AttributeError(f"{self.__dict__.get('typename')} has no field {k!r}")

    def get(self, k, default=None):
        return self.fields.get(k, default)

    def __repr__(self):
        return f"T7Object({self.typename}, fields={list(self.fields)})"


def _as_list_or_dict(d: Dict[Any, Any]):
    """A Lua table with keys 1..n (and nothing else) reads as a list, anything else as a dict."""
    n = len(d)
    if n and all(isinstance(k, float) and k == int(k) for k in d) and sorted(int(k) for k in d) == list(range(1, n + 1)):
        return [d[float(i)] for i in range(1, n + 1)]
    return {(int(k) if isinstance(k, float) and k == int(k) else k): v for k, v in d.items()}


class _Reader:
    def __init__(self, f: BinaryIO):
        self.f = f
        self.memo: Dict[int, Any] = {}

    def _read(self, fmt: str):
        size = struct.calcsize(fmt)
        b = self.f.read(size)
        if len(b) != size:
            raise EOFError("truncated .t7 file")
        return struct.unpack(fmt, b)

    def int32(self) -> int:
        return self._read("<i")[0]

    def int64(self) -> int:
        return self._read("<q")[0]

    def string(self) -> str:
        n = self.int32()
        b = self.f.read(n)
        if len(b) != n:
            raise EOFError("truncated .t7 string")
        return b.decode("latin-1")

    def obj(self):
        t = self.int32()
        if t == TYPE_NIL:
            return None
        if t == TYPE_NUMBER:
            return self._read("<d")[0]
        if t == TYPE_STRING:
            return self.string()
        if t == TYPE_BOOLEAN:
            return self.int32() != 0
        if t in (TYPE_FUNCTION, TYPE_LEGACY_RECUR_FUNCTION, TYPE_RECUR_FUNCTION):
            idx = self.int32() if t != TYPE_FUNCTION else None
            if idx is not None and idx in self.memo:
                return self.memo[idx]
            n = self.int32()
            self.f.read(n)                       # Lua bytecode: of no use here
            fn = T7Object("function")
            if idx is not None:
                self.memo[idx] = fn
            fn.fields["upvalues"] = self.obj()
            return fn
        if t == TYPE_TABLE:
            idx = self.int32()
            if idx in self.memo:
                return self.memo[idx]
            holder: Dict[Any, Any] = {}
            self.memo[idx] = holder              # cycles resolve to the raw dict
            n = self.int32()
            for _ in range(n):
                k = self.obj()
                holder[k] = self.obj()
            out = _as_list_or_dict(holder)
            self.memo[idx] = out
            return out
        if t == TYPE_TORCH:
            idx = self.int32()
            if idx in self.memo:
                return self.memo[idx]
            version = self.string()
            cls = self.string() if version.startswith("V ") else version
            if cls.startswith("torch.") and cls.endswith("Storage"):
                dt = _DTYPES[cls[len("torch."):-len("Storage")]]
                n = self.int64()
                raw = self.f.read(n * np.dtype(dt).itemsize)
                if len(raw) != n * np.dtype(dt).itemsize:
                    raise EOFError("truncated .t7 storage")
                a = np.frombuffer(raw, dtype=dt).copy()
                self.memo[idx] = a
                return a
            if cls.startswith("torch.") and cls.endswith("Tensor"):
                nd = self.int32()
                size = [self.int64() for _ in range(nd)]
                stride = [self.int64() for _ in range(nd)]
                off = self.int64() - 1
                storage = self.obj()
                key = cls[len("torch."):-len("Tensor")] or "Float"
                dt = _DTYPES.get(key, np.float32)
                if storage is None or nd == 0:
                    a = np.zeros((0,), dt)
                else:
                    item = storage.dtype.itemsize
                    a = np.lib.stride_tricks.as_strided(storage[off:], shape=size, strides=[s * item for s in stride]).copy()
                self.memo[idx] = a
                return a
            o = T7Object(cls)
            self.memo[idx] = o
            ver = int(version[2:]) if version.startswith("V ") and version[2:].strip().isdigit() else 0
            if cls.split(".")[-1] in _GPU_TABLES and ver >= 2:
                self._gpu_table(o)
                return o
            payload = self.obj()
            if isinstance(payload, dict):
                o.fields.update(payload)
            elif isinstance(payload, list):
                o.fields.update({i + 1: v for i, v in enumerate(payload)})
            if cls.endswith(".NoBackprop") and "modules" not in o.fields and "inner" in o.fields:
                o.fields["modules"] = [o.fields.pop("inner")]            # NoBackprop.lua:34-46, files older than version 2
            return o
        raise ValueError(f"unknown .t7 type tag {t}")


_GPU_TABLES = ("ModelParallelTable", "DataParallelTable", "DPParallelTable")


def _reader_gpu_table(self, o: T7Object):
    """Classes with their own __write (version >= 2). The reference's nn.ModelParallelTable writes (ModelParallelTable.lua:
    607-628, read back at :544-605): the gpuAssignments table, then every branch module as its own object, then a table
    of the remaining fields (without `modules` / `gpuAssignments`). cunn's nn.DataParallelTable (third-party, not in
    the reference; test_runner.lua:27 sets its `deserializeNGPUs`, the same scheme) writes gpuAssignments, then — depending
    on its version — the replicas or nothing, then the field table (which holds `modules` itself in newer versions).
    Both are read as: gpuAssignments, module objects until a plain table arrives, that table."""
    gpu = self.obj()
    gpu = [] if isinstance(gpu, dict) and not gpu else gpu
    if not isinstance(gpu, list):
        raise ValueError(f"{o.typename}: expected the gpuAssignments table first")
    mods: List[Any] = []
    while True:
        nxt = self.obj()
        if isinstance(nxt, T7Object) and nxt.typename != "function":
            mods.append(nxt)
            if len(mods) > max(len(gpu), 1):
                raise ValueError(f"{o.typename}: more branch modules than gpuAssignments")
            continue
        break
    if isinstance(nxt, dict):
        o.fields.update(nxt)
    elif isinstance(nxt, list):
        o.fields.update({i + 1: v for i, v in enumerate(nxt)})
    elif nxt is not None:
        raise ValueError(f"{o.typename}: expected the field table after the branches")
    o.fields["gpuAssignments"] = gpu
    if mods:
        o.fields["modules"] = mods


_Reader._gpu_table = _reader_gpu_table


def load(path_or_file) -> Any:
    """torch.load(path) -> numbers (float), str, bool, list / dict (Lua tables), numpy arrays (tensors, storages),
    T7Object (other torch classes, e.g. nn modules)."""
    if hasattr(path_or_file, "read"):
        return _Reader(path_or_file).obj()
    with open(path_or_file, "rb") as f:
        return _Reader(f).obj()


# ------------------------------------------------------------------------------------------ writer (tests, fixtures)
_TENSOR_NAMES = {np.dtype(np.float32): "Float", np.dtype(np.float64): "Double", np.dtype(np.int64): "Long",
                 np.dtype(np.int32): "Int", np.dtype(np.uint8): "Byte", np.dtype(np.int16): "Short", np.dtype(np.int8): "Char"}


class _Writer:
    def __init__(self, f: BinaryIO):
        self.f = f
        self.next_idx = 1
        self.seen: Dict[int, int] = {}

    def i32(self, v):
        self.f.write(struct.pack("<i", int(v)))

    def i64(self, v):
        self.f.write(struct.pack("<q", int(v)))

    def string(self, s: str):
        b = s.encode("latin-1")
        self.i32(len(b)); self.f.write(b)

    def _index(self, o) -> bool:
        """writes the memo index; True if the object was written before (nothing more to emit)"""
        if id(o) in self.seen:
            self.i32(self.seen[id(o)][0])
            return True
        self.seen[id(o)] = (self.next_idx, o)      # the entry keeps `o` alive: a freed temporary's id() could be reused within one save
        self.i32(self.next_idx)
        self.next_idx += 1
        return False

    def obj(self, o):
        if o is None:
            self.i32(TYPE_NIL)
        elif isinstance(o, bool):
            self.i32(TYPE_BOOLEAN); self.i32(1 if o else 0)
        elif isinstance(o, (int, float, np.integer, np.floating)):
            self.i32(TYPE_NUMBER); self.f.write(struct.pack("<d", float(o)))
        elif isinstance(o, str):
            self.i32(TYPE_STRING); self.string(o)
        elif isinstance(o, np.ndarray):
            self.i32(TYPE_TORCH)
            if self._index(o):
                return
            name = _TENSOR_NAMES[o.dtype]
            self.string("V 1"); self.string(f"torch.{name}Tensor")
            a = np.ascontiguousarray(o)
            self.i32(a.ndim)
            for s in a.shape:
                self.i64(s)
            for s in a.strides:
                self.i64(s // a.itemsize)
            self.i64(1)
            if a.ndim == 0 or a.size == 0:
                self.i32(TYPE_NIL)
            else:
                self.i32(TYPE_TORCH); self.i32(self.next_idx); self.next_idx += 1
                self.string("V 1"); self.string(f"torch.{name}Storage")
                self.i64(a.size); self.f.write(a.tobytes())
        elif isinstance(o, T7Object):
            self.i32(TYPE_TORCH)
            if self._index(o):
                return
            if o.typename.split(".")[-1] == "ModelParallelTable":           # ModelParallelTable.lua:607-628 (__version = 2)
                self.string("V 2"); self.string(o.typename)
                mods = list(o.fields.get("modules") or [])
                gpu = o.fields.get("gpuAssignments") or list(range(1, len(mods) + 1))
                self.obj(list(gpu))
                for m in mods:
                    self.obj(m)
                self._table({k: v for k, v in o.fields.items() if k not in ("modules", "gpuAssignments")}, fresh_index=True)
                return
            ver = 2 if o.typename.split(".")[-1] == "NoBackprop" else 1     # NoBackprop.lua:33
            self.string(f"V {ver}"); self.string(o.typename)
            self._table(o.fields, fresh_index=True)
        elif isinstance(o, (list, tuple)):
            self.i32(TYPE_TABLE)
            if self._index(o):
                return
            self.i32(len(o))
            for i, v in enumerate(o):
                self.obj(i + 1); self.obj(v)
        elif isinstance(o, dict):
            self.i32(TYPE_TABLE)
            if self._index(o):
                return
            self.i32(len(o))
            for k, v in o.items():
                self.obj(k); self.obj(v)
        else:
            raise TypeError(f"cannot serialise {type(o)} to .t7")

    def _table(self, d: dict, fresh_index: bool):
        self.i32(TYPE_TABLE)
        self.i32(self.next_idx); self.next_idx += 1
        self.i32(len(d))
        for k, v in d.items():
            self.obj(k); self.obj(v)


def save(path_or_file, obj) -> None:
    """torch.save(path, obj) for numbers, strings, booleans, lists / dicts, numpy arrays and T7Object."""
    if hasattr(path_or_file, "write"):
        _Writer(path_or_file).obj(obj)
        return
    with open(path_or_file, "wb") as f:
        _Writer(f).obj(obj)


# ------------------------------------------------------------------------------------------ nn graph -> ModelSpec
def _base(typename: str) -> str:
    return typename.split(".", 1)[-1]


def _children(m: T7Object) -> List[Any]:
    mods = m.get("modules")
    if mods is None and m.get("module") is not None:
        mods = [m.get("module")]
    if isinstance(mods, dict):
        mods = [mods[k] for k in sorted(mods)]
    return list(mods or [])


def flatten_sequential(m) -> List[T7Object]:
    """Depth-first list of the leaf modules of nested nn.Sequential / nn.NoBackprop / nn.DataParallelTable containers
    (utils.disableFeatureBackprop and makeDataParallel wrap parts of the trunk: model_utils.lua:95-103, vgg.lua:18-27)."""
    if not isinstance(m, T7Object):
        raise ValueError("not a torch object")
    b = _base(m.typename)
    if b in ("Sequential", "NoBackprop"):
        out: List[T7Object] = []
        for c in _children(m):
            out += flatten_sequential(c)
        return out
    if b in ("DataParallelTable", "DataParallel"):
        kids = _children(m)
        return flatten_sequential(kids[0]) if kids else []
    return [m]


def _leading_nobackprop(m):
    """the nn.NoBackprop a trunk starts with (utils.disableFeatureBackprop, model_utils.lua:95-103), reached through the
    first children of Sequential / DataParallelTable containers; None when the trunk does not start with one"""
    while isinstance(m, T7Object):
        b = _base(m.typename)
        if b == "NoBackprop":
            return m
        if b not in ("Sequential", "DataParallelTable", "DataParallel") or not _children(m):
            return None
        m = _children(m)[0]
    return None


def _linear_bias(m, cout: int, add) -> int:
    """the weight-table index of a tower Linear's bias: -1 for nn.LinearNB, the biasless first factor utils.SVDlinear
    (model_utils.lua:56-77) leaves behind; a zero vector for an nn.Linear whose bias was removed"""
    if _base(m.typename) == "LinearNB":
        return -1
    bias = m.get("bias")
    return add(np.zeros(cout, np.float32) if bias is None else _f32(bias).reshape(-1))


def _trunk_train_from(n_frozen: int, n_layers: int) -> int:
    """ModelSpec.trunk_train_from of a trunk whose first n_frozen layers sit under nn.NoBackprop: 0 (frozen) when the
    prefix is empty or covers the whole trunk (MultiPathNet's skip trunk, multipathnet.lua:60-62)"""
    return n_frozen if 0 < n_frozen < n_layers else 0


def _phase2_from(trunk, n_frozen: int, n_layers: int) -> int:
    """ModelSpec.phase2_from of a MultiPathNet skip trunk. utils.vggSetPhase2_outer (model_utils.lua:197-207) lifts the
    nn.NoBackprop around the whole skip trunk and wraps its first 10 modules instead (disableFeatureBackprop(skip, 10)).
    A phase-2 file already has that prefix: the count trunk_train_from takes. A phase-1 file (the skip trunk under
    nn.NoBackprop whole): the trunk layers its first 10 direct children make, when those are all plain convolutions,
    ReLUs and max pools (else the switch would wrap a branch: 0)."""
    if 0 < n_frozen < n_layers:
        return n_frozen
    if n_frozen != n_layers or _base(trunk.typename) != "NoBackprop" or not _children(trunk):
        return 0
    m = _children(trunk)[0]
    while _base(m.typename) in ("DataParallelTable", "DataParallel") and _children(m):
        m = _children(m)[0]
    kids = _children(m) if _base(m.typename) == "Sequential" else []
    plain = ("SpatialConvolution", "SpatialConvolutionMM", "ReLU", "SpatialMaxPooling")
    if len(kids) < 10 or any(_base(k.typename) not in plain for k in kids[:10]):
        return 0
    scratch: List[np.ndarray] = []

    def add(a):
        scratch.append(a)
        return len(scratch) - 1
    sub = _Layers(add, scratch, 3)
    v = 0
    for k in kids[:10]:
        v = sub.run(k, v)
    return len(sub.layers) if len(sub.layers) < n_layers else 0


def fast_rcnn_from_t7(model, num_classes: int = None, name: str = "t7"):
    """The graph `models/vgg.lua:23-31` (or alexnet / any trunk of conv / ReLU / max-pool) returns, as saved by train.lua,
    -> ModelSpec:  Sequential{ ParallelTable{trunk, Identity}, inn.ROIPooling(W,H,s), View, top (Linear/ReLU/Dropout...),
    ConcatTable{Linear cls, Linear bbox} [, BBoxNorm / SoftMax added at test time] }.
    Flat-list reader for this one graph; `model_from_t7` below evaluates the general table algebra (ResNet residual
    blocks, MultiPathNet towers). Grouped convolutions and LRN (CaffeNet) are refused here; model_from_t7 reads them."""
    from ._lib import Head, Layer, ModelSpec, Tower, MPN_LAYER_CONV, MPN_LAYER_FLATTEN, MPN_LAYER_MAXPOOL
    if not isinstance(model, T7Object) or _base(model.typename) != "Sequential":
        raise ValueError("expected the nn.Sequential detection model")
    top_mods = _children(model)
    if not top_mods or _base(top_mods[0].typename) != "ParallelTable":
        raise ValueError("expected nn.ParallelTable{trunk, Identity} first (vgg.lua:23-27)")
    trunk_mod = _children(top_mods[0])[0]
    trunk_mods = flatten_sequential(trunk_mod)
    frozen_mod = _leading_nobackprop(trunk_mod)
    n_frozen_leaves = len(flatten_sequential(frozen_mod)) if frozen_mod is not None else 0
    n_frozen = None                       # trunk layers made from the frozen leaves (ReLUs fuse into their convolution)
    arrays: List[np.ndarray] = []

    def add(a):
        arrays.append(np.ascontiguousarray(a, np.float32))
        return len(arrays) - 1

    trunk: List[Layer] = []
    slot, cin = 0, 3
    for mi, m in enumerate(trunk_mods):
        if mi == n_frozen_leaves:
            n_frozen = len(trunk)
        b = _base(m.typename)
        if b == "SpatialConvolution" or b == "SpatialConvolutionMM":
            if int(m.get("groups", 1) or 1) != 1:
                raise NotImplementedError("grouped convolution (CaffeNet) is not on the accelerated path")
            cout, cin_m = int(m.nOutputPlane), int(m.nInputPlane)
            kh, kw = int(m.kH), int(m.kW)
            if int(m.dW) != int(m.dH) or int(m.get("padW", 0)) != int(m.get("padH", 0)):
                raise NotImplementedError("anisotropic stride / padding")
            if cin_m != cin:
                raise ValueError(f"conv expects {cin_m} input planes, trunk has {cin}")
            w = np.asarray(m.weight, np.float32).reshape(cout, cin_m, kh, kw)
            trunk.append(Layer(MPN_LAYER_CONV, slot, slot + 1, cin=cin, cout=cout, kh=kh, kw=kw, stride=int(m.dW),
                               pad=int(m.get("padW", 0)), relu=0, weight=add(w), bias=add(np.asarray(m.bias, np.float32).reshape(cout))))
            cin = cout
            slot += 1
        elif b == "ReLU":
            if not trunk or trunk[-1].kind != MPN_LAYER_CONV or trunk[-1].out_slot != slot:
                raise NotImplementedError("ReLU that does not follow a convolution")
            trunk[-1].relu = 1
        elif b == "SpatialMaxPooling":
            if int(m.kW) != int(m.kH) or int(m.dW) != int(m.dH):
                raise NotImplementedError("anisotropic pooling")
            trunk.append(Layer(MPN_LAYER_MAXPOOL, slot, slot + 1, kh=int(m.kH), kw=int(m.kW), stride=int(m.dW),
                               pad=int(m.get("padW", 0)), ceil_mode=1 if m.get("ceil_mode", False) else 0))
            slot += 1
        elif b in ("Dropout", "Identity", "Copy"):
            continue
        else:
            raise NotImplementedError(f"trunk module {m.typename}")
    feat_slot, c5 = slot, cin
    if n_frozen is None:
        n_frozen = len(trunk)

    rest = top_mods[1:]
    if not rest or _base(rest[0].typename) != "ROIPooling":
        raise ValueError("expected inn.ROIPooling after the trunk (vgg.lua:28)")
    roi = rest[0]
    pw, ph, scale = int(roi.W), int(roi.H), float(roi.spatial_scale)
    tl = [Layer(MPN_LAYER_FLATTEN, 0, 1)]
    tslot, k_in = 1, c5 * pw * ph
    heads = None
    bbox_mean, bbox_std, has_norm = (0.0, 0.0, 0.0, 0.0), (0.1, 0.1, 0.2, 0.2), 0
    mods: List[T7Object] = []
    for m in rest[1:]:
        mods += flatten_sequential(m) if _base(m.typename) == "Sequential" else [m]
    for m in mods:
        b = _base(m.typename)
        if b in ("View", "Reshape", "Identity", "Copy"):
            continue
        if b == "Dropout":
            if m.get("v2", True) is False:
                raise NotImplementedError("nn.Dropout(v2=false) scales at test time")
            continue
        if b in ("Linear", "LinearNB") and heads is None:
            w = np.asarray(m.weight, np.float32)
            if w.shape[1] != k_in:
                raise ValueError(f"Linear expects {w.shape[1]} inputs, tower has {k_in}")
            tl.append(Layer(MPN_LAYER_CONV, tslot, tslot + 1, cin=k_in, cout=w.shape[0], relu=0, weight=add(w),
                            bias=_linear_bias(m, w.shape[0], add)))
            k_in = w.shape[0]
            tslot += 1
        elif b == "ReLU" and heads is None:
            tl[-1].relu = 1
        elif b == "ConcatTable":
            kids = _children(m)
            if len(kids) != 2 or any(_base(k.typename) != "Linear" for k in kids):
                raise NotImplementedError("expected ConcatTable{Linear cls, Linear bbox} (model_utils.lua:105-119)")
            heads = kids
        elif b == "ParallelTable" and heads is not None:
            for k in _children(m):        # test-time tail: {SoftMax, BBoxNorm} on {cls, bbox}
                kb = _base(k.typename)
                if kb == "BBoxNorm":
                    has_norm = 1
                    bbox_mean = tuple(float(x) for x in np.asarray(k.mean).reshape(-1)[:4])
                    bbox_std = tuple(float(x) for x in np.asarray(k.std).reshape(-1)[:4])
        elif b == "SoftMax":
            continue                      # detect() applies the softmax itself (ImageDetect.lua:186-190)
        elif b == "BBoxNorm":
            has_norm = 1
            bbox_mean = tuple(float(x) for x in np.asarray(m.mean).reshape(-1)[:4])
            bbox_std = tuple(float(x) for x in np.asarray(m.std).reshape(-1)[:4])
        else:
            raise NotImplementedError(f"head module {m.typename}")
    if heads is None:
        raise ValueError("no ConcatTable{cls, bbox} head found")
    wc, wb = np.asarray(heads[0].weight, np.float32), np.asarray(heads[1].weight, np.float32)
    C = wc.shape[0]
    if num_classes is not None and C != num_classes:
        raise ValueError(f"class head has {C} outputs, expected {num_classes}")
    if wb.shape[0] != 4 * C or wc.shape[1] != k_in or wb.shape[1] != k_in:
        raise ValueError("class / bbox head sizes do not match the tower")
    cls_head = Head(0, k_in, C, add(wc), add(np.asarray(heads[0].bias, np.float32).reshape(-1)))
    bbox_head = Head(0, k_in, 4 * C, add(wb), add(np.asarray(heads[1].bias, np.float32).reshape(-1)))
    tower = Tower(region=0, levels=[(feat_slot, scale)], pooled_w=pw, pooled_h=ph, normalize=0, layers=tl, out_slot=tslot)
    # ImageDetect applies SoftMax itself unless model.noSoftMax (ImageDetect.lua:186-190): a saved training graph has none
    return ModelSpec(name=name, trunk_layers=trunk, towers=[tower], cls_heads=[cls_head], bbox_head=bbox_head, num_classes=C,
                     weights=arrays, roi_variant=2, no_softmax=0, has_bbox_norm=has_norm,
                     bbox_mean=bbox_mean, bbox_std=bbox_std, transformer="ross", taps={"feat": feat_slot},
                     trunk_train_from=_trunk_train_from(n_frozen, len(trunk)))


def proposals_from_t7(obj) -> Dict[str, Any]:
    """A proposal file `{boxes = {[i] = N_i x 4 (y1, x1, y2, x2)}, scores = {...}, images = {...}}`
    (DataSetJSON.lua:124-239, utils.lua:305-372) -> {'boxes': [N_i x 4 float32 in x1,y1,x2,y2], 'scores': [...], 'images': [...]}."""
    if not isinstance(obj, dict) or "boxes" not in obj:
        raise ValueError("expected a table with a `boxes` field")
    boxes = obj["boxes"]
    if isinstance(boxes, dict):
        boxes = [boxes[k] for k in sorted(boxes)]
    out_boxes = []
    for b in boxes:
        b = np.asarray(b, np.float32).reshape(-1, 4)
        out_boxes.append(b[:, [1, 0, 3, 2]].copy())            # y1,x1,y2,x2 -> x1,y1,x2,y2
    res = {"boxes": out_boxes}
    for k in ("scores", "images"):
        if k in obj:
            v = obj[k]
            res[k] = [v[i] for i in sorted(v)] if isinstance(v, dict) else v
    return res


# ------------------------------------------------------------------------- general nn table algebra -> ModelSpec
# The MultiPathNet (models/multipathnet.lua:30-121) and ResNet (models/resnet.lua:28-50) graphs are not flat lists:
# residual blocks are ConcatTable{branch, shortcut} + CAddTable, the skip trunk returns a table {conv5, conv4, conv3}
# through ConcatTable / ParallelTable / FlattenTable. `_Layers` evaluates that table algebra symbolically: a value is a
# slot number or a (nested) list of values, leaf modules append Layer records.  PARITY UNPINNED like the rest of this file;
# the field names of third-party modules (nn.SpatialBatchNormalization running_mean / running_var | running_std,
# inn.ConstAffine a / b, nn.Narrow index / length, nn.Select index, nn.MulConstant constant_scalar) are recalled from
# torch/nn and imagine-nn, checked only against graphs this repo's tests assemble.
_PASS = ("Identity", "Copy", "Contiguous", "View", "Reshape", "Transpose", "Squeeze")
# cross-map LRN (CaffeNet's norm1 / norm2): nn.SpatialCrossMapLRN, cudnn.SpatialCrossMapLRN, inn.SpatialCrossResponseNormalization
_LRN = ("SpatialCrossMapLRN", "SpatialCrossResponseNormalization")


def _f32(a):
    return np.ascontiguousarray(np.asarray(a, np.float32))


class _Layers:
    def __init__(self, add, arrays, cin: int, hw=None, fixed_bn=None):
        from ._lib import Layer                                     # noqa: F401  (dataclass used below)
        self.add, self.arrays = add, arrays
        # fixed_bn: weight index -> inn.ConstAffine scale a, recorded for a bias-free convolution (ModelSpec.fixed_bn)
        self.fixed_bn = {} if fixed_bn is None else fixed_bn
        self.bias_free = set()
        self.layers: List[Any] = []
        self.n_frozen = 0                  # layers made inside the nn.NoBackprop the graph starts with
        self.next = 1
        self.shape = {0: (cin, None, None) if hw is None else (cin, hw[0], hw[1])}
        # where the map size is not known (the trunk), each axis' size as a function of the input's: (steps, offset), a
        # strided step (c, s, ceil) giving (x + c) // s + 1 (ceil: rounded up), then + offset; equal forms, equal sizes
        self.sig = {0: (((), 0), ((), 0))}

    # -- helpers
    def _slot(self, shape):
        s = self.next
        self.next += 1
        self.shape[s] = shape
        return s

    def _sized(self, o, s, kh, kw, st, ph, pw, ceil=0):
        """record slot o's size form: a k x k / stride / pad step (convolution or pooling) on slot s"""
        def step(f, k, p):
            ops, off = f
            return (ops, off + 2 * p - k + 1) if st == 1 and not ceil else (ops + ((off + 2 * p - k, st, ceil),), 1)
        if s in self.sig:
            self.sig[o] = (step(self.sig[s][0], kh, ph), step(self.sig[s][1], kw, pw))
        return o

    def _producer(self, slot):
        for L in reversed(self.layers):
            if L.out_slot == slot:
                return L
        return None

    @staticmethod
    def _need_slot(v, what):
        if not isinstance(v, int):
            raise NotImplementedError(f"{what} applied to a table")
        return v

    def _open_conv(self, slot, what):
        from ._lib import MPN_LAYER_CONV
        L = self._producer(slot)
        if L is None or L.kind != MPN_LAYER_CONV or L.relu or L.residual_slot >= 0 or L.out_c_total:
            raise NotImplementedError(f"{what} that does not directly follow a convolution / Linear")
        return L

    def _affine(self, slot, scale, shift, what):
        """y = scale[c] * x + shift[c] right after a convolution: fold into its weight and bias (inn.utils.foldBatchNorm)."""
        L = self._open_conv(slot, what)
        scale, shift = np.asarray(scale, np.float64).reshape(-1), np.asarray(shift, np.float64).reshape(-1)
        if scale.size != L.cout or shift.size != L.cout:
            raise ValueError(f"{what}: {scale.size} channels after a convolution with {L.cout}")
        w = self.arrays[L.weight].astype(np.float64)
        self.arrays[L.weight] = _f32(w * scale.reshape((-1,) + (1,) * (w.ndim - 1)))
        self.arrays[L.bias] = _f32(self.arrays[L.bias].astype(np.float64) * scale + shift)

    def _concat(self, m, b, v):
        """nn.Concat(2) / nn.DepthConcat(2) (inceptionv3.lua's Mixed blocks, nested): every branch runs on v, and the layers that
        write each branch's output are re-targeted to their channel slice of one slot (Layer.out_c_off / out_c_total)"""
        from ._lib import MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_CONV, MPN_LAYER_MAXPOOL
        s = self._need_slot(v, m.typename)
        d = int(m.get("dimension", 2))
        if d != 2:
            raise NotImplementedError(f"nn.{b} along dimension {d}: only the channel dimension (2) is concatenated")
        if any(_base(c.typename) == "Narrow" or (_base(c.typename) == "Sequential" and _children(c) and
                                                 _base(_children(c)[0].typename) == "Narrow") for c in _children(m)):
            raise NotImplementedError(f"nn.{b} of nn.Narrow branches (loadcaffe's form of a grouped convolution): convert it to "
                                      "cudnn.SpatialConvolution with groups")
        outs = [self.run(c, s) for c in _children(m)]
        if not outs or not all(isinstance(o, int) and o != s for o in outs):
            raise NotImplementedError(f"nn.{b} branch that is empty or returns a table")
        shapes = [self.shape[o] for o in outs]
        if len({sh[1:] for sh in shapes}) != 1 or (shapes[0][1] is None and len({self.sig.get(o) for o in outs}) != 1):
            why = "DepthConcat would zero-pad the smaller ones" if b == "DepthConcat" else "Concat needs equal sizes"
            raise NotImplementedError(f"nn.{b} of branches with different map sizes {[sh[1:] for sh in shapes]} ({why})")
        total = sum(sh[0] for sh in shapes)
        o = self._slot((total,) + shapes[0][1:])
        if outs[0] in self.sig:
            self.sig[o] = self.sig[outs[0]]
        off = 0
        for br, sh in zip(outs, shapes):
            writers = [L for L in self.layers if L.out_slot == br]
            if not writers or any(L.kind not in (MPN_LAYER_CONV, MPN_LAYER_MAXPOOL, MPN_LAYER_AVGPOOL_WIN) or L.residual_slot >= 0
                                  for L in writers) or any(L.in_slot == br or L.residual_slot == br for L in self.layers):
                raise NotImplementedError(f"nn.{b} branch that does not end in a convolution or a pooling written once")
            for L in writers:
                L.out_c_off, L.out_c_total, L.out_slot = off + (L.out_c_off if L.out_c_total else 0), total, o
            off += sh[0]
        return o

    # -- the evaluator
    def run(self, m, v):
        from ._lib import Layer, MPN_LAYER_AVGPOOL, MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_CONV, MPN_LAYER_FLATTEN, MPN_LAYER_LRN, MPN_LAYER_MAXPOOL
        if not isinstance(m, T7Object):
            raise ValueError("not a torch object")
        b = _base(m.typename)
        if b in ("Sequential", "NoBackprop"):
            start = len(self.layers)
            for c in _children(m):
                v = self.run(c, v)
            if b == "NoBackprop" and start == 0:
                self.n_frozen = max(self.n_frozen, len(self.layers))
            return v
        if b in ("DataParallelTable", "DataParallel"):
            kids = _children(m)
            return self.run(kids[0], v) if kids else v
        if b == "ConcatTable":
            return [self.run(c, v) for c in _children(m)]
        if b == "ParallelTable":
            kids = _children(m)
            if not isinstance(v, list) or len(v) != len(kids):
                raise ValueError("nn.ParallelTable arity does not match its input table")
            return [self.run(c, vi) for c, vi in zip(kids, v)]
        if b in ("Concat", "DepthConcat"):
            return self._concat(m, b, v)
        if b == "FlattenTable":
            def flat(x):
                return [y for e in x for y in flat(e)] if isinstance(x, list) else [x]
            return flat(v)
        if b == "SelectTable":
            i = int(m.index)
            if not isinstance(v, list):
                raise ValueError("nn.SelectTable on a tensor")
            return v[i - 1] if i > 0 else v[i]
        if b in _PASS:
            return v
        if b == "Dropout":
            if m.get("v2", True) is False:
                raise NotImplementedError("nn.Dropout(v2=false) scales at test time")
            return v
        if b == "CAddTable":
            if not isinstance(v, list) or len(v) != 2 or not all(isinstance(x, int) for x in v):
                raise NotImplementedError("nn.CAddTable of anything but two tensors")
            for main, other in ((v[0], v[1]), (v[1], v[0])):
                L = self._producer(main)
                if L is not None and L.kind == MPN_LAYER_CONV and not L.relu and L.residual_slot < 0 and self.shape[main] == self.shape[other]:
                    self.layers.remove(L)                      # the shortcut branch was emitted after it: run it last
                    self.layers.append(L)
                    L.residual_slot = other
                    return main
            raise NotImplementedError("residual add whose branches do not end in a bare convolution")
        s = self._need_slot(v, m.typename)
        c, h, w = self.shape[s]
        if b in ("SpatialConvolution", "SpatialConvolutionMM"):
            cout, cin, kh, kw = int(m.nOutputPlane), int(m.nInputPlane), int(m.kH), int(m.kW)
            g = int(m.get("groups", 1) or 1)
            if g != 1 and (g < 1 or cin % g or cout % g or (cin // g) % 8 or (cout // g) % 8):
                raise NotImplementedError(f"grouped convolution {cin} -> {cout} in {g} groups: each group must read and write a "
                                          "multiple of 8 channels (the engine's channel grid)")
            st, pw_ = int(m.get("dW", 1)), int(m.get("padW", 0) or 0)
            pd = int(m.get("padH", pw_) or 0)                  # a pad per axis: 1 x n / n x 1 kernels (inceptionv3.lua)
            if st != int(m.get("dH", st)):
                raise NotImplementedError(f"anisotropic stride ({m.get('dH')} x {st}): the engine strides both axes alike")
            if cin != c:
                raise ValueError(f"conv expects {cin} input planes, its input has {c}")
            bias = m.get("bias")
            o = self._slot((cout, None if h is None else (h + 2 * pd - kh) // st + 1, None if w is None else (w + 2 * pw_ - kw) // st + 1))
            self._sized(o, s, kh, kw, st, pd, pw_)
            self.layers.append(Layer(MPN_LAYER_CONV, s, o, cin=cin, cout=cout, kh=kh, kw=kw, stride=st, pad=pd, relu=0,
                                     pad_w=pw_ if pw_ != pd else -1, groups=g,
                                     weight=self.add(_f32(m.weight).reshape(cout, cin // g, kh, kw)),
                                     bias=self.add(np.zeros(cout, np.float32) if bias is None else _f32(bias).reshape(cout))))
            if bias is None:
                self.bias_free.add(self.layers[-1].weight)
            return o
        if b in _LRN:
            size, alpha, beta, k = int(m.get("size", 0)), float(m.get("alpha", 0)), float(m.get("beta", 0)), float(m.get("k", 1))
            if (size, alpha, beta, k) != (5, 1e-4, 0.75, 1.0):
                raise NotImplementedError(f"{m.typename}(size {size}, alpha {alpha}, beta {beta}, k {k}): only CaffeNet's LRN "
                                          "(size 5, alpha 1e-4, beta 0.75, k 1) runs on the device")
            if c % 8:
                raise NotImplementedError(f"{m.typename} over {c} channels: the LRN kernel takes a multiple of 8")
            o = self._slot((c, h, w))
            self._sized(o, s, 1, 1, 1, 0, 0)
            self.layers.append(Layer(MPN_LAYER_LRN, s, o))
            return o
        if b in ("Linear", "LinearNB"):
            wt = _f32(m.weight)
            if h is not None and h * w > 1:                     # View(-1):setNumInputDims(3) before the first Linear
                s2 = self._slot((c * h * w, 1, 1))
                self.layers.append(Layer(MPN_LAYER_FLATTEN, s, s2))
                s, c = s2, c * h * w
            if wt.shape[1] != c:
                raise ValueError(f"Linear expects {wt.shape[1]} inputs, its input has {c}")
            o = self._slot((wt.shape[0], 1, 1))
            self.layers.append(Layer(MPN_LAYER_CONV, s, o, cin=c, cout=wt.shape[0], relu=0, weight=self.add(wt),
                                     bias=_linear_bias(m, wt.shape[0], self.add)))
            return o
        if b in ("SpatialBatchNormalization", "BatchNormalization"):
            eps = float(m.get("eps", 1e-5))
            if m.get("running_var") is not None:
                inv = 1.0 / np.sqrt(np.asarray(m.running_var, np.float64) + eps)
            elif m.get("running_std") is not None:              # older nn: running_std already holds 1 / sqrt(var + eps)
                inv = np.asarray(m.running_std, np.float64)
            else:
                raise ValueError("batch normalisation without running statistics")
            g = np.asarray(m.weight, np.float64) if m.get("weight") is not None else np.ones_like(inv)
            beta = np.asarray(m.bias, np.float64) if m.get("bias") is not None else np.zeros_like(inv)
            scale = g * inv
            self._affine(s, scale, beta - np.asarray(m.running_mean, np.float64) * scale, m.typename)
            return s
        if b == "ConstAffine":                                  # inn.utils.BNtoFixed: y = a * x + b per channel
            a = m.get("a", m.get("weight"))
            sh = m.get("b", m.get("bias"))
            if a is None or sh is None:
                raise ValueError("inn.ConstAffine without a / b")
            self._affine(s, a, sh, m.typename)
            # a and b are constants (no gradWeight): after a bias-free convolution, the layer trains in the fixed-batch-norm
            # form. A convolution with its own bias would train that bias in the reference: no record.
            wi = self._producer(s).weight
            if wi in self.bias_free and wi not in self.fixed_bn:
                self.fixed_bn[wi] = _f32(a).reshape(-1)
            return s
        if b == "MulConstant":
            k = float(m.constant_scalar)
            self._affine(s, np.full(c, k), np.zeros(c), m.typename)
            return s
        if b in ("ReLU", "Threshold"):
            if b == "Threshold" and (float(m.get("threshold", 0)) != 0.0 or float(m.get("val", 0)) != 0.0):
                raise NotImplementedError("nn.Threshold other than ReLU")
            L = self._producer(s)
            if L is None or L.kind != MPN_LAYER_CONV or L.out_c_total:
                raise NotImplementedError("ReLU that does not follow a convolution / Linear / residual add")
            L.relu = 1
            return s
        if b == "SpatialMaxPooling":
            k, st, pd = int(m.kW), int(m.dW), int(m.get("padW", 0) or 0)
            if k != int(m.kH) or st != int(m.dH):
                raise NotImplementedError("anisotropic pooling")
            ceil = 1 if m.get("ceil_mode", False) else 0
            from .models import _pool_out
            o = self._slot((c, None if h is None else _pool_out(h, k, st, pd, ceil), None if w is None else _pool_out(w, k, st, pd, ceil)))
            self._sized(o, s, k, k, st, pd, pd, ceil)
            self.layers.append(Layer(MPN_LAYER_MAXPOOL, s, o, kh=k, kw=k, stride=st, pad=pd, ceil_mode=ceil))
            return o
        if b == "SpatialAveragePooling":
            k, st, pd = int(m.kW), int(m.get("dW", 1)), int(m.get("padW", 0) or 0)
            if h is not None and (int(m.kH), int(m.kW)) == (h, w) and pd == 0:
                o = self._slot((c, 1, 1))                          # the global pool that ends a ResNet (resnet.lua:39)
                self.layers.append(Layer(MPN_LAYER_AVGPOOL, s, o))
                return o
            if k != int(m.kH) or st != int(m.get("dH", st)) or pd != int(m.get("padH", pd) or 0):
                raise NotImplementedError("anisotropic average pooling")
            ceil = 1 if m.get("ceil_mode", False) else 0
            xp = 0 if m.get("count_include_pad", True) else 1   # setCountExcludePad
            from .models import _pool_out
            o = self._slot((c, None if h is None else _pool_out(h, k, st, pd, ceil), None if w is None else _pool_out(w, k, st, pd, ceil)))
            self._sized(o, s, k, k, st, pd, pd, ceil)
            self.layers.append(Layer(MPN_LAYER_AVGPOOL_WIN, s, o, kh=k, kw=k, stride=st, pad=pd, ceil_mode=ceil, exclude_pad=xp))
            return o
        raise NotImplementedError(f"module {m.typename}")


def _linear_heads(mods, width, add, narrows=None):
    """classAndBBoxLinear (model_utils.lua:105-119) and its integral-loss rewrite (:275-317):
    {Linear | ConcatTable{K x Linear}, Linear} fed by the whole tower output or by two nn.Narrow column ranges."""
    from ._lib import Head
    if len(mods) != 2:
        raise NotImplementedError("expected {class head(s), bbox head}")
    cols = narrows or [(0, width), (0, width)]
    cls_m = _children(mods[0]) if _base(mods[0].typename) == "ConcatTable" else [mods[0]]
    out = []
    for ms, (c0, cl) in ((cls_m, cols[0]), ([mods[1]], cols[1])):
        hs = []
        for m in ms:
            if _base(m.typename) != "Linear":
                raise NotImplementedError(f"head module {m.typename}")
            w = _f32(m.weight)
            if w.shape[1] != cl:
                raise ValueError(f"head Linear expects {w.shape[1]} inputs, its columns are {cl} wide")
            bias = m.get("bias")
            hs.append(Head(c0, cl, w.shape[0], add(w), add(np.zeros(w.shape[0], np.float32) if bias is None else _f32(bias).reshape(-1))))
        out.append(hs)
    return out[0], out[1][0]


def _parse_pool_level(seq, trunk_vals):
    """make1PoolingLayer (model_utils.lua:212-228): ParallelTable{SelectTable(idx), Identity}, inn.ROIPooling(7,7,s),
    then View / Normalize(2) / Contiguous / View  |  MulConstant(f)."""
    kids = _children(seq)
    if len(kids) < 2 or _base(kids[0].typename) != "ParallelTable" or _base(kids[1].typename) != "ROIPooling":
        raise NotImplementedError("pooling branch is not ParallelTable{SelectTable, Identity} + inn.ROIPooling")
    sel = _children(kids[0])[0]
    if _base(sel.typename) != "SelectTable":
        raise NotImplementedError("pooling branch does not select a trunk output")
    slot = trunk_vals[int(sel.index) - 1]
    roi = kids[1]
    norm, factor = False, 1.0
    for m in kids[2:]:
        b = _base(m.typename)
        if b == "Normalize":
            if float(m.get("p", 2)) != 2.0:
                raise NotImplementedError("nn.Normalize with p != 2")
            norm = True
        elif b == "MulConstant":
            factor *= float(m.constant_scalar)
        elif b not in _PASS:
            raise NotImplementedError(f"pooling branch module {m.typename}")
    return slot, (int(roi.W), int(roi.H), float(roi.spatial_scale)), norm, factor


def model_from_t7(model, name: str = "t7", transformer: str = None, num_classes: int = None):
    """Any of the detection graphs the reference's model files return (models/{vgg,alexnet,resnet,multipathnet}.lua), as
    torch.save'd by train.lua:195, -> ModelSpec.
      Sequential{ ParallelTable{trunk, Identity},
                  inn.ROIPooling, per-ROI modules                                   (vgg.lua:23-31, resnet.lua:41-50)
                | ParallelTable{Identity, Sequential{Foveal, View, Transpose}},
                  ModelParallelTable{ towers }, [ConcatTable{Narrow, Narrow}]        (multipathnet.lua:61-117)
                  ConcatTable | ParallelTable {class head(s), bbox head} [, ModeSwitch (integral loss)] [, SoftMax / BBoxNorm] }
    Batch normalisation (raw, or inn.ConstAffine after inn.utils.BNtoFixed) is folded into the preceding convolution, as
    inn.utils.foldBatchNorm does for the frozen layers (resnet.lua:33-36); per-level MulConstant factors of the
    un-normalised conv345Combine are folded into conv_mix's input columns (the mix is linear in them)."""
    from ._lib import Layer, ModelSpec, Tower, MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_CONV, MPN_LAYER_FLATTEN, MPN_LAYER_LRN
    if not isinstance(model, T7Object) or _base(model.typename) != "Sequential":
        raise ValueError("expected the nn.Sequential detection model")
    top = _children(model)
    if not top or _base(top[0].typename) != "ParallelTable" or len(_children(top[0])) != 2:
        raise ValueError("expected nn.ParallelTable{trunk, Identity} first (vgg.lua:23-27)")
    arrays: List[np.ndarray] = []

    def add(a):
        arrays.append(np.ascontiguousarray(a, np.float32))
        return len(arrays) - 1

    fixed_bn = {}
    tb = _Layers(add, arrays, 3, fixed_bn=fixed_bn)
    tv = tb.run(_children(top[0])[0], 0)
    trunk_vals = tv if isinstance(tv, list) else [tv]
    if not all(isinstance(x, int) for x in trunk_vals):
        raise NotImplementedError("trunk returns a nested table")
    has_res = any(L.residual_slot >= 0 for L in tb.layers)
    rest = top[1:]
    towers: List[Any] = []
    widths: List[int] = []
    i = 0
    phase2_from = 0
    if rest and _base(rest[0].typename) == "ROIPooling":
        roi = rest[0]
        pw, ph, sc = int(roi.W), int(roi.H), float(roi.spatial_scale)
        if len(trunk_vals) != 1:
            raise ValueError("inn.ROIPooling on a trunk that returns several maps")
        lb = _Layers(add, arrays, tb.shape[trunk_vals[0]][0], (ph, pw), fixed_bn=fixed_bn)
        v, i = 0, 1
        while i < len(rest) and _base(rest[i].typename) not in ("ConcatTable", "ParallelTable"):
            v = lb.run(rest[i], v)
            i += 1
        c, h, w = lb.shape[v]
        if h * w > 1:                                           # heads read a flat vector
            v2 = lb._slot((c * h * w, 1, 1))
            lb.layers.append(Layer(MPN_LAYER_FLATTEN, v, v2))
            v, c = v2, c * h * w
        if not lb.layers:
            raise NotImplementedError("no per-ROI layer between inn.ROIPooling and the heads")
        towers.append(Tower(region=0, levels=[(trunk_vals[0], sc)], pooled_w=pw, pooled_h=ph, normalize=0, layers=lb.layers, out_slot=v))
        widths.append(c)
    elif len(rest) >= 2 and _base(rest[0].typename) == "ParallelTable" and _base(rest[1].typename) == "ModelParallelTable":
        fov = flatten_sequential(_children(rest[0])[1])
        if not fov or _base(fov[0].typename) != "Foveal":
            raise NotImplementedError("expected nn.Foveal on the ROI branch (multipathnet.lua:65-69)")
        if int(rest[1].get("dimension", 2)) != 2:
            raise NotImplementedError("ModelParallelTable joining along a dimension other than 2")
        for t in _children(rest[1]):
            kids = _children(t)
            if len(kids) < 3 or _base(kids[0].typename) != "ParallelTable":
                raise NotImplementedError("tower is not {ParallelTable{Identity, Select}, conv345Combine, classifier}")
            sel = _children(kids[0])[1]
            if _base(sel.typename) != "Select" or int(sel.dimension) != 1:
                raise NotImplementedError("tower does not nn.Select(1, region) its ROIs")
            region = int(sel.index) - 1
            if not 0 <= region < 4:
                raise ValueError("nn.Foveal produces 4 regions")
            levels, shapes, norms, factors, post = [], [], [], [], 1.0
            mix_seen, lb, v = False, None, 0
            for m in _children(kids[1]):
                b = _base(m.typename)
                if b == "ConcatTable" and not levels:
                    for br in _children(m):
                        slot, (pw, ph, sc), nm, f = _parse_pool_level(br, trunk_vals)
                        levels.append((slot, sc)); shapes.append((pw, ph)); norms.append(nm); factors.append(f)
                elif b == "JoinTable":
                    if int(m.dimension) != 2:
                        raise NotImplementedError("levels are joined along channels (JoinTable(2), model_utils.lua:237)")
                elif b == "MulConstant" and not mix_seen:
                    post *= float(m.constant_scalar)
                elif b in ("SpatialConvolution", "SpatialConvolutionMM") and not mix_seen:
                    if len(set(shapes)) != 1 or len(set(norms)) != 1:
                        raise NotImplementedError("levels pooled to different sizes / mixed normalisation")
                    chans = [tb.shape[s][0] for s, _sc in levels]
                    lb = _Layers(add, arrays, sum(chans), (shapes[0][1], shapes[0][0]), fixed_bn=fixed_bn)
                    v = lb.run(m, 0)
                    col = np.concatenate([np.full(c, f, np.float64) for c, f in zip(chans, factors)])
                    col *= post / 1000.0 if norms[0] else post   # the kernel applies Normalize + MulConstant(1000) itself
                    if not np.all(col == 1.0):
                        L = lb.layers[0]
                        arrays[L.weight] = _f32(arrays[L.weight].astype(np.float64) * col.reshape(1, -1, 1, 1))
                    mix_seen = True
                elif b in _PASS:
                    continue
                else:
                    raise NotImplementedError(f"conv345Combine module {m.typename}")
            if not mix_seen:
                raise NotImplementedError("tower without conv_mix (model_utils.lua:242)")
            for m in kids[2:]:
                v = lb.run(m, v)
            c, h, w = lb.shape[v]
            if h * w > 1:
                raise NotImplementedError("tower output is not a vector")
            towers.append(Tower(region=region, levels=levels, pooled_w=shapes[0][0], pooled_h=shapes[0][1],
                                normalize=1 if norms[0] else 0, layers=lb.layers, out_slot=v))
            widths.append(c)
        i = 2
        if len(towers) > 1:
            phase2_from = _phase2_from(_children(top[0])[0], tb.n_frozen, len(tb.layers))
    else:
        raise NotImplementedError("expected inn.ROIPooling or the foveal ModelParallelTable after the trunk")

    total = sum(widths)
    narrows, cls_heads, bbox_head = None, None, None
    no_softmax = 1 if model.get("noSoftMax") else 0
    graph_softmax = False
    bbox_mean, bbox_std, has_norm = (0.0, 0.0, 0.0, 0.0), (0.1, 0.1, 0.2, 0.2), 0

    def norm_of(k):
        return 1, tuple(float(x) for x in np.asarray(k.mean).reshape(-1)[:4]), tuple(float(x) for x in np.asarray(k.std).reshape(-1)[:4])

    for m in rest[i:]:
        b = _base(m.typename)
        kids = _children(m)
        if b == "ConcatTable" and kids and all(_base(k.typename) == "Narrow" for k in kids) and cls_heads is None:
            if len(kids) != 2 or any(int(k.dimension) != 2 for k in kids):
                raise NotImplementedError("expected two nn.Narrow(2, ...) column ranges (multipathnet.lua:115)")
            narrows = [(int(k.index) - 1, int(k.length)) for k in kids]
            if any(c0 < 0 or c0 + cl > total for c0, cl in narrows):
                raise ValueError("nn.Narrow reaches past the tower outputs")
        elif b in ("ConcatTable", "ParallelTable") and cls_heads is None:
            if b == "ParallelTable" and narrows is None:
                raise NotImplementedError("ParallelTable heads without the Narrow split before them")
            cls_heads, bbox_head = _linear_heads(kids, total, add, narrows)
        elif b == "ModeSwitch" and cls_heads is not None:
            no_softmax = 1                                       # eval branch = mean of the K softmaxes (model_utils.lua:300-313)
        elif b == "ParallelTable" and cls_heads is not None:
            for k in kids:
                if _base(k.typename) == "BBoxNorm":
                    has_norm, bbox_mean, bbox_std = norm_of(k)
                elif _base(k.typename) == "SoftMax":
                    graph_softmax = True
        elif b == "BBoxNorm":
            has_norm, bbox_mean, bbox_std = norm_of(m)
        elif b == "SoftMax":
            graph_softmax = True
        elif b in _PASS:
            continue
        else:
            raise NotImplementedError(f"head module {m.typename}")
    if cls_heads is None:
        raise ValueError("no {class, bbox} head found")
    if graph_softmax and len(cls_heads) == 1:
        # a SoftMax inside the graph (test_add_nosoftmax, test_runner.lua:38-41): with model.noSoftMax the reference returns the
        # model's own softmax and ImageDetect adds none (ImageDetect.lua:189) = ONE softmax, which is what detect() applies
        # when no_softmax = 0; without noSoftMax the reference would apply it twice
        if not model.get("noSoftMax"):
            raise NotImplementedError("nn.SoftMax inside the graph without model.noSoftMax: the reference applies the softmax twice")
        no_softmax = 0
    C = cls_heads[0].cout
    if any(h.cout != C for h in cls_heads) or bbox_head.cout != 4 * C:
        raise ValueError("class / bbox head sizes disagree")
    if num_classes is not None and C != num_classes:
        raise ValueError(f"class head has {C} outputs, expected {num_classes}")
    if len(cls_heads) > 1:
        no_softmax = 1
    taps = {f"out{k + 1}": s for k, s in enumerate(trunk_vals)}
    for t in towers:
        for L in t.layers:
            if L.groups != 1 or L.kind == MPN_LAYER_LRN:
                raise NotImplementedError("a grouped convolution or an LRN in the per-ROI part: the device runs them in the trunk only")
    inception = any(L.out_c_total or L.kind == MPN_LAYER_AVGPOOL_WIN for L in tb.layers + [L for t in towers for L in t.layers])
    return ModelSpec(name=name, trunk_layers=tb.layers, towers=towers, cls_heads=cls_heads, bbox_head=bbox_head, num_classes=C,
                     weights=arrays, roi_variant=2, no_softmax=no_softmax, has_bbox_norm=has_norm, bbox_mean=bbox_mean,
                     bbox_std=bbox_std, transformer=transformer or ("inception" if inception else ("imagenet" if has_res else "ross")),
                     taps=taps,
                     trunk_train_from=_trunk_train_from(tb.n_frozen, len(tb.layers)), fixed_bn=fixed_bn, phase2_from=phase2_from)


# --------------------------------------------------------------------------------- ModelSpec -> nn graph (export)
def _m(name, **fields):
    return T7Object(name, fields)


def _seq_of(mods):
    return _m("nn.Sequential", modules=list(mods))


def _layers_to_modules(layers, weights, in_slot, out_slot):
    """A straight chain of Layer records (no residuals) -> nn modules, in order."""
    from ._lib import MPN_LAYER_AVGPOOL, MPN_LAYER_CONV, MPN_LAYER_FLATTEN, MPN_LAYER_LRN, MPN_LAYER_MAXPOOL
    mods, cur, flat = [], in_slot, False
    for L in layers:
        if L.in_slot != cur or L.residual_slot >= 0:
            raise NotImplementedError("only straight chains of layers can be exported")
        if L.kind == MPN_LAYER_CONV and not flat:
            g = L.groups
            mods.append(_m("cudnn.SpatialConvolution", nInputPlane=L.cin, nOutputPlane=L.cout, kW=L.kw, kH=L.kh, dW=L.stride, dH=L.stride,
                           padW=L.pad, padH=L.pad, groups=g, weight=_f32(weights[L.weight]).reshape(L.cout, L.cin // g, L.kh, L.kw),
                           bias=_f32(weights[L.bias]).reshape(L.cout)))
        elif L.kind == MPN_LAYER_LRN:
            mods.append(_m("inn.SpatialCrossResponseNormalization", size=5, alpha=1e-4, beta=0.75, k=1.0))
        elif L.kind == MPN_LAYER_CONV and L.bias < 0:           # the first factor of an SVD-compressed Linear
            mods.append(_m("nn.LinearNB", weight=_f32(weights[L.weight]).reshape(L.cout, L.cin)))
        elif L.kind == MPN_LAYER_CONV:
            mods.append(_m("nn.Linear", weight=_f32(weights[L.weight]).reshape(L.cout, L.cin), bias=_f32(weights[L.bias]).reshape(L.cout)))
        elif L.kind == MPN_LAYER_MAXPOOL:
            mods.append(_m("cudnn.SpatialMaxPooling", kW=L.kw, kH=L.kh, dW=L.stride, dH=L.stride, padW=L.pad, padH=L.pad, ceil_mode=bool(L.ceil_mode)))
        elif L.kind == MPN_LAYER_FLATTEN:
            mods.append(_m("nn.View", size=[-1], numInputDims=3))
            flat = True
        elif L.kind == MPN_LAYER_AVGPOOL:
            raise NotImplementedError("global average pool needs the pooled size: export ResNet graphs from Torch instead")
        else:
            raise NotImplementedError(f"layer kind {L.kind}")
        if L.kind == MPN_LAYER_CONV and L.relu:
            mods.append(_m("cudnn.ReLU", inplace=True))
        cur = L.out_slot
    if cur != out_slot:
        raise ValueError("layer chain does not end at the requested slot")
    return mods


def _layer_module(L, weights, hw):
    """one layer of a branching graph (Inception-v3) -> its nn modules; hw: the input map's (h, w), for a global average pool"""
    from ._lib import MPN_LAYER_AVGPOOL, MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_CONV, MPN_LAYER_MAXPOOL
    if L.residual_slot >= 0:
        raise NotImplementedError("residual adds are not exported inside a branching graph")
    if L.kind == MPN_LAYER_CONV:
        mods = [_m("cudnn.SpatialConvolution", nInputPlane=L.cin, nOutputPlane=L.cout, kW=L.kw, kH=L.kh, dW=L.stride, dH=L.stride,
                   padW=L.padw, padH=L.pad, groups=1, weight=_f32(weights[L.weight]).reshape(L.cout, L.cin, L.kh, L.kw),
                   bias=_f32(weights[L.bias]).reshape(L.cout))]
        return mods + ([_m("cudnn.ReLU", inplace=True)] if L.relu else [])
    if L.kind == MPN_LAYER_MAXPOOL:
        return [_m("cudnn.SpatialMaxPooling", kW=L.kw, kH=L.kh, dW=L.stride, dH=L.stride, padW=L.pad, padH=L.pad, ceil_mode=bool(L.ceil_mode))]
    if L.kind == MPN_LAYER_AVGPOOL_WIN:
        return [_m("cudnn.SpatialAveragePooling", kW=L.kw, kH=L.kh, dW=L.stride, dH=L.stride, padW=L.pad, padH=L.pad,
                   ceil_mode=bool(L.ceil_mode), count_include_pad=not L.exclude_pad)]
    if L.kind == MPN_LAYER_AVGPOOL:
        return [_m("cudnn.SpatialAveragePooling", kW=hw[1], kH=hw[0], dW=1, dH=1, padW=0, padH=0), _m("nn.View", size=[-1], numInputDims=3)]
    raise NotImplementedError(f"layer kind {L.kind} in a branching graph")


def _branching_to_modules(layers, weights, a, b, hw0):
    """the layers from slot a to slot b of a graph whose branches write channel slices of concatenation slots
    (Layer.out_c_total) -> nn modules, each concatenation an nn.Concat(2) of its branches, nested where branches share
    their first layers (inceptionv3.lua's Mixed blocks)"""
    from .models import _pool_out
    from ._lib import MPN_LAYER_AVGPOOL_WIN, MPN_LAYER_CONV, MPN_LAYER_MAXPOOL
    writers = {}
    for L in layers:
        writers.setdefault(L.out_slot, []).append(L)
    hw = {a: hw0}
    for L in layers:                                             # map sizes, for the global average pool's kernel
        if L.in_slot in hw and hw[L.in_slot] is not None:
            h, w = hw[L.in_slot]
            if L.kind == MPN_LAYER_CONV:
                hw[L.out_slot] = ((h + 2 * L.pad - L.kh) // L.stride + 1, (w + 2 * L.padw - L.kw) // L.stride + 1)
            elif L.kind in (MPN_LAYER_MAXPOOL, MPN_LAYER_AVGPOOL_WIN):
                hw[L.out_slot] = (_pool_out(h, L.kh, L.stride, L.pad, L.ceil_mode), _pool_out(w, L.kw, L.stride, L.pad, L.ceil_mode))
            else:
                hw[L.out_slot] = (1, 1)

    def path(L, stop):                                           # the layers from slot `stop` to L (a chain through unit inputs)
        out = [L]
        while out[0].in_slot != stop:
            ws = writers.get(out[0].in_slot, [])
            if len(ws) != 1 or ws[0].out_c_total:
                return None
            out.insert(0, ws[0])
        return out

    def unit(slot):
        """(input slot, modules) of what writes `slot`: one layer, or a concatenation of branches"""
        ws = writers.get(slot, [])
        if len(ws) == 1 and not ws[0].out_c_total:
            return ws[0].in_slot, _layer_module(ws[0], weights, hw.get(ws[0].in_slot))
        ws = sorted(ws, key=lambda L: L.out_c_off)
        # the block input: the nearest slot every writer's chain of inputs reaches
        def ancestors(L):
            out, cur = [], L.in_slot
            while True:
                out.append(cur)
                w = writers.get(cur, [])
                if cur == a or len(w) != 1 or w[0].out_c_total:
                    return out
                cur = w[0].in_slot
        anc = [ancestors(L) for L in ws]
        x = next((c for c in anc[0] if all(c in q for q in anc[1:])), None)
        paths = [path(L, x) for L in ws] if x is not None else [None]
        if any(p is None for p in paths):
            raise NotImplementedError("a concatenation whose branches do not start from one slot")

        def branches(ps):
            mods, i = [], 0
            while i < len(ps):
                j = i + 1
                while j < len(ps) and ps[j][0] is ps[i][0]:
                    j += 1
                g = ps[i:j]
                if any(ps[k][0] is ps[i][0] for k in range(j, len(ps))):
                    raise NotImplementedError("branches sharing a layer are not adjacent in the concatenation")
                if len(g) == 1:
                    mods.append(_seq_of([m for L in g[0] for m in _layer_module(L, weights, hw.get(L.in_slot))]))
                else:
                    pre = []
                    while all(len(p) > 1 for p in g) and all(p[0] is g[0][0] for p in g):
                        pre.append(g[0][0])
                        g = [p[1:] for p in g]
                    mods.append(_seq_of([m for L in pre for m in _layer_module(L, weights, hw.get(L.in_slot))] +
                                        [_m("nn.Concat", dimension=2, modules=branches(g))]))
                i = j
            return mods
        return x, [_m("nn.Concat", dimension=2, modules=branches(paths))]

    mods, cur = [], b
    while cur != a:
        cur, ms = unit(cur)
        mods = ms + mods
    return mods


def model_to_t7(spec):
    """ModelSpec -> the nn graph models/vgg.lua:23-31 (one tower, one trunk tap) or models/multipathnet.lua:30-121
    (skip trunk {conv5, conv4, conv3}, foveal towers, Narrow split) would build around the same weights, as T7Objects
    ready for `save`. The inverse of `model_from_t7` for straight-chain trunks (VGG-style); residual trunks are not
    exported. Lets weights produced or converted here go back to Torch, and gives the importer a full-depth round trip."""
    trunk = list(spec.trunk_layers)
    ident = lambda: _m("nn.Identity")
    par = lambda *ms: _m("nn.ParallelTable", modules=list(ms))
    cat = lambda *ms: _m("nn.ConcatTable", modules=list(ms))

    def chain(a, b):
        sel, cur = [], b
        for L in reversed(trunk):                               # walk back from b to a
            if L.out_slot == cur:
                sel.append(L)
                cur = L.in_slot
                if cur == a:
                    break
        if cur != a:
            raise NotImplementedError("trunk taps are not on one chain")
        return _layers_to_modules(list(reversed(sel)), spec.weights, a, b)

    tap_slots = []
    for t in spec.towers:
        for s, _sc in t.levels:
            if s not in tap_slots:
                tap_slots.append(s)
    order = {L.out_slot: i for i, L in enumerate(trunk)}
    tap_slots.sort(key=lambda s: -order[s])                      # deepest first: {conv5, conv4, conv3}
    heads_tail = []
    C = spec.num_classes
    lin = lambda h: _m("nn.Linear", weight=_f32(spec.weights[h.weight]).reshape(h.cout, h.col_len), bias=_f32(spec.weights[h.bias]).reshape(h.cout))
    cls_m = cat(*[lin(h) for h in spec.cls_heads]) if len(spec.cls_heads) > 1 else lin(spec.cls_heads[0])
    from ._lib import MPN_LAYER_AVGPOOL_WIN
    branching = any(L.out_c_total or L.kind == MPN_LAYER_AVGPOOL_WIN for L in trunk + [L for t in spec.towers for L in t.layers])
    if branching and len(spec.towers) == 1 and len(spec.towers[0].levels) == 1 and not spec.towers[0].normalize:
        t = spec.towers[0]                                       # models/inceptionv3.lua: concatenated branches
        feats = _branching_to_modules(trunk, spec.weights, 0, tap_slots[0], None)
        model = _seq_of([par(_seq_of(feats), ident()),
                         _m("inn.ROIPooling", W=t.pooled_w, H=t.pooled_h, spatial_scale=float(t.levels[0][1]), v2=True)]
                        + _branching_to_modules(t.layers, spec.weights, 0, t.out_slot, (t.pooled_h, t.pooled_w))
                        + [cat(cls_m, lin(spec.bbox_head))])
    elif len(spec.towers) == 1 and len(spec.towers[0].levels) == 1 and not spec.towers[0].normalize:
        t = spec.towers[0]
        k = spec.trunk_train_from
        feats = chain(0, tap_slots[0]) if k <= 0 else \
            [_m("nn.NoBackprop", modules=[_seq_of(chain(0, trunk[k - 1].out_slot))])] + chain(trunk[k - 1].out_slot, tap_slots[0])
        model = _seq_of([par(_seq_of(feats), ident()),
                         _m("inn.ROIPooling", W=t.pooled_w, H=t.pooled_h, spatial_scale=float(t.levels[0][1]), v2=True)]
                        + _layers_to_modules(t.layers, spec.weights, 0, t.out_slot) + [cat(cls_m, lin(spec.bbox_head))])
    else:
        if len(tap_slots) != 3:
            raise NotImplementedError("expected the three skip taps of multipathnet.lua")
        c5, c4, c3 = tap_slots
        skip = _seq_of(chain(0, c3) + [cat(_seq_of(chain(c3, c4)), ident()), par(cat(_seq_of(chain(c4, c5)), ident()), ident()),
                                       _m("nn.FlattenTable")])
        model = _seq_of([par(_m("nn.NoBackprop", modules=[skip]), ident()),
                         par(ident(), _seq_of([_m("nn.Foveal"), _m("nn.View", size=[-1, 4, 5]), _m("nn.Transpose", permutations=[[1, 2]])]))])
        regions = _m("nn.ModelParallelTable", dimension=2, modules=[], gpuAssignments=[])
        nchan = {s: next(L.cout for L in trunk if L.out_slot == s) for s in tap_slots}
        for t in spec.towers:
            pools = []
            for s, sc in t.levels:
                p = [par(_m("nn.SelectTable", index=tap_slots.index(s) + 1), ident()),
                     _m("inn.ROIPooling", W=t.pooled_w, H=t.pooled_h, spatial_scale=float(sc), v2=True)]
                if t.normalize:
                    n = nchan[s]
                    p += [_m("nn.View", size=[-1, n * t.pooled_w * t.pooled_h]), _m("nn.Normalize", p=2, eps=1e-10), _m("nn.Contiguous"),
                          _m("nn.View", size=[-1, n, t.pooled_h, t.pooled_w])]
                pools.append(_seq_of(p))
            join = [cat(*pools), _m("nn.JoinTable", dimension=2)] + ([_m("nn.MulConstant", constant_scalar=1000)] if t.normalize else [])
            rest = _layers_to_modules(t.layers, spec.weights, 0, t.out_slot)          # conv_mix, View, classifier
            nmix = 1 + (1 if rest[1].typename == "cudnn.ReLU" else 0)
            regions.fields["modules"].append(_seq_of([par(ident(), _m("nn.Select", dimension=1, index=t.region + 1)),
                                                      _seq_of(join + rest[:nmix + 1]), _seq_of(rest[nmix + 1:])]))
        model.fields["modules"].append(regions)
        hb, hc = spec.bbox_head, spec.cls_heads[0]
        model.fields["modules"].append(cat(_m("nn.Narrow", dimension=2, index=hc.col_begin + 1, length=hc.col_len),
                                           _m("nn.Narrow", dimension=2, index=hb.col_begin + 1, length=hb.col_len)))
        model.fields["modules"].append(par(cls_m, lin(hb)))
    if len(spec.cls_heads) > 1:                                  # model_utils.lua:275-317
        K = len(spec.cls_heads)
        sm = par(*[_seq_of([_m("nn.SoftMax"), _m("nn.View", size=[1, -1, C])]) for _ in range(K)])
        model.fields["modules"].append(_m("nn.ModeSwitch", train=False, modules=[
            par(_m("nn.SelectTable", index=1), ident()),
            _seq_of([par(_seq_of([sm, _m("nn.JoinTable", dimension=1), _m("nn.Mean", dimension=1)]), ident())])]))
        model.fields["noSoftMax"] = True
    elif spec.no_softmax:
        model.fields["noSoftMax"] = True
    if spec.has_bbox_norm:
        model.fields["modules"].append(par(ident(), _m("nn.BBoxNorm", mean=_f32(spec.bbox_mean).reshape(1, 4), std=_f32(spec.bbox_std).reshape(1, 4))))
    return model

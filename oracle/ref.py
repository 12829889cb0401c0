"""ctypes wrappers over oracle/libmpn_oracle.so (C restatement) and oracle/_ref/libnms_ref.so
(the LITERAL reference nms.c, compiled from the reference's own source by oracle/Makefile where it is present).
Where that build is absent, the literal functions answer from tests/golden/nms_literal_golden.npz: their outputs on
every fixed input the suite feeds them, recorded from the literal build (MPN_LITERAL_RECORD, see record_literal()).
TEST INFRASTRUCTURE — see oracle/__init__.py."""
from __future__ import annotations

import atexit
import ctypes as C
import hashlib
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_ORC = os.path.join(_HERE, "libmpn_oracle.so")
_REF = os.path.join(_HERE, "_ref", "libnms_ref.so")
_GOLD = os.path.join(os.path.dirname(_HERE), "tests", "golden", "nms_literal_golden.npz")


def build(quiet: bool = True):
    """compile the C restatement and (where the reference's source is present) the literal nms.c"""
    subprocess.run(["make", "-C", _HERE], check=True, stdout=subprocess.DEVNULL if quiet else None)


def _load(path):
    if not os.path.exists(path):
        build()
    return C.CDLL(path)


_orc = None
_ref = None
_fp = C.POINTER(C.c_float)


def orc():
    global _orc
    if _orc is None:
        _orc = _load(_ORC)
        _orc.orc_overlap.restype = C.c_float
        _orc.orc_nms.restype = C.c_long
        _orc.orc_nms_dense.restype = C.c_long
        _orc.orc_pool_out.restype = C.c_long
    return _orc


def ref_built() -> bool:
    """the literal nms.c itself is callable (not only its stored outputs)"""
    return os.path.exists(_REF)


def ref_available() -> bool:
    return ref_built() or os.path.exists(_GOLD)


_gold = None
_record = {} if os.environ.get("MPN_LITERAL_RECORD") else None


def _key(op, *arrays):
    h = hashlib.sha1(op.encode())
    for a in arrays:
        a = np.ascontiguousarray(a)
        h.update(str((a.dtype.str, a.shape)).encode())
        h.update(a.tobytes())
    return op + "_" + h.hexdigest()[:24]


def _literal(op, call, *arrays):
    """call() on the literal build, or its stored output for exactly these inputs"""
    global _gold
    key = _key(op, *arrays)
    if ref_built():
        out = call()
        if _record is not None:
            _record[key] = out
        return out
    if _gold is None:
        _gold = dict(np.load(_GOLD)) if os.path.exists(_GOLD) else {}
    if key not in _gold:
        raise LookupError(f"no stored output of the literal nms.c for this input ({key}): build oracle/_ref from the "
                          "reference's nms.c (oracle/Makefile) and record it (record_literal)")
    return _gold[key].copy()


@atexit.register
def record_literal():
    """MPN_LITERAL_RECORD=path: merge the literal outputs of this process into the .npz at path"""
    path = os.environ.get("MPN_LITERAL_RECORD")
    if not path or not _record:
        return
    old = dict(np.load(path)) if os.path.exists(path) else {}
    old.update(_record)
    np.savez_compressed(path, **old)


def ref():
    global _ref
    if _ref is None:
        _ref = _load(_REF)
        _ref.ref_nms.restype = C.c_long
    return _ref


def _f(a):
    return np.ascontiguousarray(a, dtype=np.float32)


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


# ---- literal reference (nms.c) ---------------------------------------------------------------
def ref_nms_rows(scored_boxes, thr):
    """utils.nms -> nms.c:NMS: returns the kept ROWS (K x 5) exactly as the reference does."""
    sb = _f(scored_boxes).reshape(-1, 5)

    def call():
        out = np.empty_like(sb)
        k = ref().ref_nms(_p(sb), C.c_long(sb.shape[0]), C.c_float(thr), _p(out)) if sb.shape[0] else 0
        return out[:k].copy()
    return _literal("nms", call, sb, np.float32(thr))


def ref_bbox_vote(nms_boxes, scored_boxes, thr):
    nb, sb = _f(nms_boxes).reshape(-1, 5), _f(scored_boxes).reshape(-1, 5)

    def call():
        res = np.zeros_like(nb)
        if nb.shape[0]:
            ref().ref_bbox_vote(_p(nb), C.c_long(nb.shape[0]), _p(sb), C.c_long(sb.shape[0]), C.c_float(thr), _p(res))
        return res
    return _literal("bbox_vote", call, nb, sb, np.float32(thr))


def ref_boxoverlap(a_n4, b4):
    a, b = _f(a_n4).reshape(-1, 4), _f(b4).reshape(4)

    def call():
        out = np.empty(a.shape[0], np.float32)
        ref().ref_boxoverlap(_p(a), C.c_long(a.shape[0]), _p(b), _p(out))
        return out
    return _literal("boxoverlap", call, a, b)


# ---- C restatement -----------------------------------------------------------------------------
def nms(scored_boxes, thr):
    sb = _f(scored_boxes).reshape(-1, 5)
    keep = np.empty(max(sb.shape[0], 1), np.int32)
    k = orc().orc_nms(_p(sb), C.c_long(sb.shape[0]), C.c_float(thr), _p(keep))
    return keep[:k].copy()


def nms_dense(scored_boxes, thr):
    sb = _f(scored_boxes).reshape(-1, 5)
    pick = np.empty(max(sb.shape[0], 1), np.int32)
    k = orc().orc_nms_dense(_p(sb), C.c_long(sb.shape[0]), C.c_float(thr), _p(pick))
    return pick[:k].copy()


def bbox_vote(nms_boxes, scored_boxes, thr):
    nb, sb = _f(nms_boxes).reshape(-1, 5), _f(scored_boxes).reshape(-1, 5)
    res = np.zeros_like(nb)
    orc().orc_bbox_vote(_p(nb), C.c_long(nb.shape[0]), _p(sb), C.c_long(sb.shape[0]), C.c_float(thr), _p(res))
    return res


def overlap(a4, b4):
    a, b = _f(a4), _f(b4)
    return float(orc().orc_overlap(_p(a), _p(b)))


def foveal(rois):
    r = _f(rois)
    out = np.empty((r.shape[0] * 4, 5), np.float32)
    orc().orc_foveal(_p(r), C.c_long(r.shape[0]), _p(out))
    return out


def context_region(rois, scale):
    r = _f(rois)
    out = np.empty_like(r)
    orc().orc_context_region(_p(r), C.c_long(r.shape[0]), C.c_float(scale), _p(out))
    return out


def bbox_norm(deltas, mean, std):
    d = _f(deltas).copy()
    m, s = _f(mean).reshape(4), _f(std).reshape(4)
    orc().orc_bbox_norm(_p(d), C.c_long(d.shape[0]), C.c_long(d.shape[1]), _p(m), _p(s))
    return d


def convert_from(deltas, boxes):
    d, b = _f(deltas), _f(boxes)
    out = np.empty_like(d)
    orc().orc_convert_from(_p(d), _p(b), C.c_long(d.shape[0]), C.c_long(d.shape[1] // 4), _p(out))
    return out


def convert_to_f64(bbox, tbox):
    b, t = np.ascontiguousarray(bbox, np.float64), np.ascontiguousarray(tbox, np.float64)
    out = np.empty(4, np.float64)
    orc().orc_convert_to_f64(_p(b), _p(t), _p(out))
    return out


def convert_from_f64(bbox, y):
    b, t = np.ascontiguousarray(bbox, np.float64), np.ascontiguousarray(y, np.float64)
    out = np.empty(4, np.float64)
    orc().orc_convert_from_f64(_p(b), _p(t), _p(out))
    return out


def clamp_boxes(bboxes, W0, H0):
    b = _f(bboxes).copy()
    orc().orc_clamp_boxes(_p(b), C.c_long(b.size // 4), C.c_float(W0), C.c_float(H0))
    return b


def softmax(x):
    x = _f(x)
    out = np.empty_like(x)
    orc().orc_softmax(_p(x), C.c_long(x.shape[0]), C.c_long(x.shape[1]), _p(out))
    return out


def project_rois(boxes, im_scale):
    b = _f(boxes)
    out = np.empty((b.shape[0], 5), np.float32)
    orc().orc_project_rois(_p(b), C.c_long(b.shape[0]), C.c_float(im_scale), _p(out))
    return out


def l2_normalize(x):
    x = _f(x).copy()
    orc().orc_l2_normalize(_p(x), C.c_long(x.shape[0]), C.c_long(x.shape[1]))
    return x


def roi_pool(fmap, rois, pw, ph, scale, variant=2, with_argmax=False):
    f, r = _f(fmap), _f(rois)
    n, c, h, w = f.shape
    out = np.empty((r.shape[0], c, ph, pw), np.float32)
    am = np.empty(out.shape, np.int32) if with_argmax else None
    orc().orc_roi_pool(_p(f), C.c_long(n), C.c_long(c), C.c_long(h), C.c_long(w), _p(r), C.c_long(r.shape[0]),
                       C.c_int(pw), C.c_int(ph), C.c_float(scale), C.c_int(variant), _p(out), _p(am) if with_argmax else None)
    return (out, am) if with_argmax else out


def pool_out(n, k, s, p, ceil_mode):
    return int(orc().orc_pool_out(C.c_long(n), C.c_int(k), C.c_int(s), C.c_int(p), C.c_int(ceil_mode)))


# ---- getImages (SURVEY 8f-1): ImageTransformer + image.scale, "parity unpinned" (third-party `image` package) --------
_HD = os.path.join(_HERE, "libhd_shim.so")
_hd = None
_TRANSFORMERS = {  # model_utils.lua:138-155: (mean, std, scale, swap)
    "ross": ((102.9801, 115.9465, 122.7717), None, 255.0, (3, 2, 1)),
    "imagenet": ((0.48462227599918, 0.45624044862054, 0.40588363755159),
                 (0.22889466674951, 0.22446679341259, 0.22495548344775), 1.0, (1, 2, 3)),
}


def transformer_params(kind):
    return _TRANSFORMERS[kind]


def get_images_size(H0, W0, scale, max_size):
    """ImageDetect.lua:31-39 -> (h, w, im_scale)"""
    h, w, s = C.c_long(), C.c_long(), C.c_double()
    orc().orc_get_images_size(C.c_long(H0), C.c_long(W0), C.c_double(scale), C.c_double(max_size), C.byref(h), C.byref(w), C.byref(s))
    return int(h.value), int(w.value), float(s.value)


def image_transform(im, kind):
    im = _f(im)
    mean, std, scale, swap = _TRANSFORMERS[kind]
    out = np.empty_like(im)
    m = _f(mean); sd = _f(std) if std is not None else None
    sw = (C.c_int * 3)(*swap)
    orc().orc_image_transform(_p(im), C.c_long(im.shape[1]), C.c_long(im.shape[2]), sw, C.c_float(scale), _p(m),
                              _p(sd) if sd is not None else None, _p(out))
    return out


def image_scale(im, h, w):
    """image.scale(im, w, h), 'bilinear': two passes with an fp32 temporary, as the original"""
    im = _f(im)
    out = np.empty((im.shape[0], h, w), np.float32)
    orc().orc_image_scale(_p(im), C.c_long(im.shape[0]), C.c_long(im.shape[1]), C.c_long(im.shape[2]), _p(out), C.c_long(h), C.c_long(w))
    return out


def get_images(im, kind, scale=600, max_size=1000):
    """getImages for the single test scale -> (3 x h x w image, im_scale)"""
    h, w, s = get_images_size(im.shape[1], im.shape[2], scale, max_size)
    return image_scale(image_transform(im, kind), h, w), s


def hd_get_images(im, kind, h, w):
    """the product's per-pixel __host__ __device__ arithmetic (csrc/image_scale.cuh), run on the host"""
    global _hd
    if _hd is None:
        _hd = _load(_HD)
    im = _f(im)
    mean, std, scale, swap = _TRANSFORMERS[kind]
    m = _f(mean); sd = _f(std) if std is not None else None
    out = np.empty((3, h, w), np.float32)
    _hd.hd_get_images(_p(im), C.c_int(im.shape[1]), C.c_int(im.shape[2]), (C.c_int * 3)(*swap), C.c_float(scale), _p(m),
                      _p(sd) if sd is not None else None, C.c_int(h), C.c_int(w), _p(out))
    return out


def hd_get_images_u8(im_hwc_u8, kind, h, w, use_lut=True):
    """the same per-pixel code fed with the decoder's uint8 H0 x W0 x 3 bytes, with or without the byte -> float table"""
    global _hd
    if _hd is None:
        _hd = _load(_HD)
    im = np.ascontiguousarray(im_hwc_u8, np.uint8)
    mean, std, scale, swap = _TRANSFORMERS[kind]
    m = _f(mean); sd = _f(std) if std is not None else None
    out = np.empty((3, h, w), np.float32)
    _hd.hd_get_images_u8(im.ctypes.data_as(C.c_void_p), C.c_int(im.shape[0]), C.c_int(im.shape[1]), (C.c_int * 3)(*swap), C.c_float(scale), _p(m),
                         _p(sd) if sd is not None else None, C.c_int(h), C.c_int(w), C.c_int(1 if use_lut else 0), _p(out))
    return out

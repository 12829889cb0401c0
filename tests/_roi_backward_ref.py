"""Reference for the inn.ROIPooling backward (imagine-nn's updateGradInput as recalled, source absent: "parity unpinned").

A plain scatter: zero grad_data, then for r, c, ph, pw ascending add grad_out into the cell the forward's argmax names
(-1, an empty bin, adds nothing). np.add.at applies the additions one by one in index order, in the array's dtype
(fp32), so per cell this is the summation order of the library's gather kernel (ascending r, ph, pw from +0), reached
by a different algorithm. imagine-nn adds with atomics (order unspecified): it agrees up to the rounding of the sum."""
import numpy as np


def roi_pool_backward(grad_out, argmax, rois, data_shape):
    """grad_out / argmax R x C x PH x PW, rois R x 5 (1-based batch index in column 0) -> grad_data of data_shape"""
    g = np.ascontiguousarray(grad_out, np.float32)
    am = np.ascontiguousarray(argmax, np.int32)
    r = np.asarray(rois, np.float32).reshape(-1, 5)
    N, C, H, W = (int(s) for s in data_shape)
    assert g.ndim == 4 and g.shape == am.shape and g.shape[:2] == (r.shape[0], C)
    n = r[:, 0].astype(np.int64) - 1                     # (int)roi[0] - 1, as the forward converts it
    plane = (n[:, None] * C + np.arange(C)[None, :]) * (H * W)
    flat = plane[:, :, None, None] + am.astype(np.int64)
    sel = (am >= 0) & ((n >= 0) & (n < N))[:, None, None, None]   # a batch index out of range matches no image
    out = np.zeros(N * C * H * W, np.float32)
    np.add.at(out, flat[sel], g[sel])                    # boolean selection keeps the (r, c, ph, pw) C order
    return out.reshape(N, C, H, W)

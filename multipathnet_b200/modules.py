"""nn.Module mirrors of the reference's region / bbox modules, backed by the C ABI.

Same constructor arguments, same input checks (the reference asserts become ValueError), same
eval/train behaviour where the reference defines it:
  nn.Foveal (modules/Foveal.lua), nn.ContextRegion (modules/ContextRegion.lua),
  nn.BBoxNorm (modules/BBoxNorm.lua), inn.ROIPooling(W,H,scale) (call sites vgg.lua:28 ...),
  fbcoco.ImageTransformer (modules/ImageTransformer.lua; host-side, stays on the CPU like the reference).
"""
from __future__ import annotations

import numpy as np

from ._lib import Context
from . import workloads


class _Module:
    def __init__(self, ctx: Context):
        self.ctx = ctx
        self.train = True
        self.output = None

    def training(self):
        self.train = True
        return self

    def evaluate(self):
        self.train = False
        return self

    def forward(self, x):
        self.output = self.updateOutput(x)
        return self.output

    def clearState(self):
        self.output = None
        return self


def _check_rois(x):
    x = np.asarray(x, dtype=np.float32)
    if x.ndim != 2 or x.shape[1] != 5:                       # Foveal.lua:16-17, ContextRegion.lua:27-28
        raise ValueError("expected an R x 5 tensor of [id,x1,y1,x2,y2]")
    return x


class Foveal(_Module):
    def updateOutput(self, input):
        return self.ctx.foveal(_check_rois(input))

    def updateGradInput(self, input, gradOutput):
        return None                                          # Foveal.lua defines no gradient


class ContextRegion(_Module):
    def __init__(self, ctx: Context, scale: float):
        super().__init__(ctx)
        self.scale = float(scale)

    def updateOutput(self, input):
        return self.ctx.context_region(_check_rois(input), self.scale)

    def updateGradInput(self, input, gradOutput):
        return np.zeros_like(np.asarray(input, np.float32))   # ContextRegion.lua:34-37

    def __repr__(self):
        return f"nn.ContextRegion({self.scale})"


class BBoxNorm(_Module):
    def __init__(self, ctx: Context, mean, std):
        if mean is None or std is None:
            raise ValueError("BBoxNorm needs mean and std")   # BBoxNorm.lua:12
        super().__init__(ctx)
        self.mean = np.asarray(mean, np.float32).reshape(4)
        self.std = np.asarray(std, np.float32).reshape(4)

    def updateOutput(self, input):
        x = np.asarray(input, np.float32)
        if x.ndim != 2 or x.shape[1] % 4 != 0:                # BBoxNorm.lua:19
            raise ValueError("BBoxNorm: input must be 2-D with size(2) % 4 == 0")
        if self.train:
            return x                                          # identity in training mode (BBoxNorm.lua:20-21)
        return self.ctx.bbox_norm(x, self.mean, self.std)

    def updateGradInput(self, input, gradOutput):
        if not self.train:
            raise RuntimeError("cannot updateGradInput in evaluate mode")   # BBoxNorm.lua:35
        return gradOutput


class ROIPooling(_Module):
    """inn.ROIPooling(W, H, spatial_scale); forward({data N x C x H x W, rois R x 5})."""

    def __init__(self, ctx: Context, W: int, H: int, spatial_scale: float = 1.0, v2: bool = True):
        super().__init__(ctx)
        self.W, self.H, self.spatial_scale, self.v2 = int(W), int(H), float(spatial_scale), bool(v2)
        self.indices = None

    def setSpatialScale(self, s: float):
        self.spatial_scale = float(s)
        return self

    def updateOutput(self, input):
        data, rois = input
        out, am = self.ctx.roi_pool(np.asarray(data, np.float32), _check_rois(rois), self.W, self.H, self.spatial_scale,
                                    2 if self.v2 else 1, with_argmax=True)
        self.indices = am
        return out

    def updateGradInput(self, input, gradOutput):
        """(grad_data, zeros like rois) from the argmax of the last forward; grad_data is summed per cell in ascending
        (roi, ph, pw) order, so it is deterministic (imagine-nn's atomics agree up to the rounding of that sum)"""
        if self.indices is None:
            raise RuntimeError("ROIPooling:updateGradInput needs a forward first (it uses the forward's argmax)")
        data, rois = input
        data, rois = np.asarray(data, np.float32), _check_rois(rois)
        grad_data = self.ctx.roi_pool_backward(gradOutput, self.indices, rois, data.shape, self.W, self.H, self.spatial_scale,
                                               2 if self.v2 else 1)
        self.gradInput = (grad_data, np.zeros_like(rois))
        return self.gradInput


class SelectBoxes:
    """nn.SelectBoxes (modules/SelectBoxes.lua:26-56), forward only: input {classes R x C, boxes R x 4C} -> for every row
    the 4 values of its arg-max class (first maximum, like torch.max), optionally de-normalised with std / mean
    (SelectBoxes.lua:45-52). Host side (numpy): R x C is tiny, and the reference only uses it between two detect() calls
    of the iterative localisation (Tester_FRCNN.lua:82-89)."""

    def __init__(self, mean=None, std=None):
        self.mean = None if mean is None else np.asarray(mean, np.float32).reshape(1, 4)
        self.std = None if std is None else np.asarray(std, np.float32).reshape(1, 4)
        self.output = None

    def forward(self, input):
        classes, ys = input
        classes = np.asarray(classes, np.float32)
        ys = np.asarray(ys, np.float32)
        if classes.ndim != 2 or ys.ndim != 2 or ys.shape[0] != classes.shape[0] or ys.shape[1] != 4 * classes.shape[1]:
            raise ValueError("SelectBoxes: expected {R x C, R x 4C}")
        maxids = np.argmax(classes, axis=1)                       # first maximum on ties
        cols = maxids[:, None] * 4 + np.arange(4)[None, :]
        out = np.take_along_axis(ys, cols, axis=1)
        if self.std is not None:
            out = out * self.std + self.mean
        self.output = out.astype(np.float32)
        return self.output

    def updateGradInput(self, input, gradOutput):
        raise RuntimeError("SelectBoxes: training is out of scope here")


class ImageTransformer:
    """fbcoco.ImageTransformer (host side). kind: 'ross' = RossTransformer, 'imagenet' = ImagenetTransformer,
    'inception' = ImageTransformer({1,1,1}, nil, 2) of inceptionv3.lua (2 x - 1)."""

    def __init__(self, kind: str = "ross"):
        self.kind = kind

    def forward(self, im_chw):
        im = np.asarray(im_chw, np.float32)
        if im.ndim != 3:
            raise ValueError("ImageTransformer expects a 3 x H x W image")   # ImageTransformer.lua:20
        return workloads.transform(im, self.kind)

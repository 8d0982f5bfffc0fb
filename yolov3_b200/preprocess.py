"""Device-side image pre-processing (SURVEY §8(f) row f1) with the reference's call shapes:

``letterbox(im, new_shape, color, auto, scaleFill, scaleup, stride)`` — utils/augmentations.py:104-134 on a CUDA uint8 HWC
image (returns ``(im, ratio, (dw, dh))`` exactly like the reference, the image staying on the device), and ``preprocess`` — what
``LoadImages.__next__`` hands to the model (utils/dataloaders.py:305-310: letterbox, HWC->CHW, BGR->RGB, contiguous) written
straight into a CHW uint8 tensor such as an engine's input buffer; ``im.float() / 255`` (detect.py:187-191) is applied by the
first conv kernel.  One launch of ``y3_letterbox_u8``, whose per-pixel routine the validation loader's batched letterbox
shares; the resize is OpenCV's 8-bit INTER_LINEAR bit for bit (csrc/y3_resize.cuh, csrc/y3_augment.cu)."""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import _lib
from .tensors import _stream


def letterbox_geometry(shape, new_shape=(640, 640), auto=True, scaleFill=False, scaleup=True, stride=32):
    """Scalar part of letterbox (utils/augmentations.py:104-132): (new_unpad (w, h), ratio, (dw, dh), top, bottom, left, right)."""
    if isinstance(new_shape, int):
        new_shape = (new_shape, new_shape)
    r = min(new_shape[0] / shape[0], new_shape[1] / shape[1])
    if not scaleup:  # only scale down (better val mAP)
        r = min(r, 1.0)
    ratio = r, r
    new_unpad = round(shape[1] * r), round(shape[0] * r)
    dw, dh = new_shape[1] - new_unpad[0], new_shape[0] - new_unpad[1]
    if auto:  # minimum rectangle
        dw, dh = np.mod(dw, stride), np.mod(dh, stride)
    elif scaleFill:  # stretch
        dw, dh = 0.0, 0.0
        new_unpad = (new_shape[1], new_shape[0])
        ratio = new_shape[1] / shape[1], new_shape[0] / shape[0]
    dw /= 2
    dh /= 2
    top, bottom = round(dh - 0.1), round(dh + 0.1)
    left, right = round(dw - 0.1), round(dw + 0.1)
    return new_unpad, ratio, (dw, dh), top, bottom, left, right


def _launch(im: torch.Tensor, new_unpad, top, left, out: torch.Tensor, chw: bool, swap_rb: bool, color):
    assert im.is_cuda and im.dtype == torch.uint8 and im.dim() == 3 and im.shape[2] == 3 and im.stride(2) == 1 and im.stride(1) == 3, \
        "image: CUDA uint8 [h, w, 3] with packed pixels (yolov3_b200 has no CPU path)"
    assert out.is_cuda and out.dtype == torch.uint8 and out.is_contiguous()
    d = _lib.LetterboxDesc()
    d.src, d.src_h, d.src_w, d.src_pitch = im.data_ptr(), im.shape[0], im.shape[1], im.stride(0)
    d.new_w, d.new_h, d.top, d.left = int(new_unpad[0]), int(new_unpad[1]), int(top), int(left)
    d.dst = out.data_ptr()
    d.out_h, d.out_w = (out.shape[1], out.shape[2]) if chw else (out.shape[0], out.shape[1])
    d.out_chw, d.swap_rb = int(chw), int(swap_rb)
    for c in range(3):
        d.pad[c] = int(color[c])
    _lib.check(_lib.lib().y3_letterbox_u8(C.byref(d), _stream()), "y3_letterbox_u8")
    return out


def letterbox(im: torch.Tensor, new_shape=(640, 640), color=(114, 114, 114), auto=True, scaleFill=False, scaleup=True, stride=32):
    """Drop-in for utils/augmentations.py:104 on a CUDA uint8 HWC image; returns (letterboxed HWC image, ratio, (dw, dh))."""
    new_unpad, ratio, (dw, dh), top, bottom, left, right = letterbox_geometry(im.shape[:2], new_shape, auto, scaleFill, scaleup, stride)
    out = torch.empty(new_unpad[1] + top + bottom, new_unpad[0] + left + right, 3, dtype=torch.uint8, device=im.device)
    _launch(im, new_unpad, top, left, out, chw=False, swap_rb=False, color=color)
    return out, ratio, (dw, dh)


def preprocess(im0: torch.Tensor, img_size=640, stride=32, auto=True, out: torch.Tensor | None = None):
    """LoadImages.__next__ (utils/dataloaders.py:305-310) on the device: BGR HWC uint8 frame -> letterboxed RGB CHW uint8
    (``out``: an existing [3, H, W] uint8 tensor of the right size, e.g. one image of an engine's input batch).
    Returns (im, ratio, (dw, dh))."""
    new_unpad, ratio, (dw, dh), top, bottom, left, right = letterbox_geometry(im0.shape[:2], img_size, auto, False, True, stride)
    hh, ww = new_unpad[1] + top + bottom, new_unpad[0] + left + right
    if out is None:
        out = torch.empty(3, hh, ww, dtype=torch.uint8, device=im0.device)
    assert tuple(out.shape) == (3, hh, ww), f"preprocess: out must be [3, {hh}, {ww}], got {tuple(out.shape)}"
    _launch(im0, new_unpad, top, left, out, chw=True, swap_rb=True, color=(114, 114, 114))
    return out, ratio, (dw, dh)

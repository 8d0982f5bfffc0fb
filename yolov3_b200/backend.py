"""``DetectMultiBackend`` — the reference's own backend-plugin point (models/common.py:435-476, ``pt`` branch; callers
detect.py:166,183,196, val.py:293,324,364, hubconf.py:63) with the GPU ``Model`` behind it: same constructor arguments,
same attributes (``stride names pt jit engine fp16 device triton model nhwc``), ``forward(im, augment, visualize)``,
``warmup(imgsz)`` and ``from_numpy``.  Only the PyTorch (``pt``) role exists here; there is no CPU device."""
from __future__ import annotations

from pathlib import Path

import numpy as np
import torch

from .model import Model


ALLOW_PICKLED_CHECKPOINTS = False  # opt-in: reference-pickled modules run arbitrary code in torch.load


def _load(weights, device, cfg=None) -> Model:
    if isinstance(weights, Model):
        return weights.to(device)
    if isinstance(weights, (list, tuple)):
        assert len(weights) == 1, "_load takes one checkpoint; several -> tta.attempt_load builds an Ensemble"
        weights = weights[0]
    ckpt = weights
    if isinstance(weights, (str, Path)):
        # a checkpoint written by this package: {"cfg": yaml name / path / dict, "state_dict": reference-named tensors}.
        # Reference *.pt files pickle the reference's nn.Module classes; with the reference importable they load too
        # (ckpt["ema"] or ckpt["model"], models/experimental.py:87-101).
        try:  # this package's own checkpoints hold only tensors / dicts / lists / strings: no pickle execution needed
            ckpt = torch.load(str(weights), map_location="cpu", weights_only=True)
        except Exception as e:
            if not ALLOW_PICKLED_CHECKPOINTS:
                raise RuntimeError(f"{weights}: not a tensors-only checkpoint ({type(e).__name__}).  Reference *.pt files pickle "
                                   "whole nn.Modules (train.py:445-462) and execute code on load; set "
                                   "yolov3_b200.backend.ALLOW_PICKLED_CHECKPOINTS = True to load a file you trust") from e
            ckpt = torch.load(str(weights), map_location="cpu", weights_only=False)
    if isinstance(ckpt, dict) and "state_dict" in ckpt:
        m = Model(ckpt.get("cfg", cfg or "yolov3.yaml"), device=device)
        m.load_state_dict(ckpt["state_dict"])
        if "names" in ckpt:
            m.names = ckpt["names"]
        return m
    ref = (ckpt.get("ema") or ckpt["model"]) if isinstance(ckpt, dict) else ckpt  # a reference DetectionModel object
    m = Model(ref.yaml, device=device)
    m.load_state_dict({k: v.float() for k, v in ref.float().state_dict().items()})
    m.names = getattr(ref, "names", m.names)
    return m


def save_checkpoint(model: Model, path) -> None:
    """Write the checkpoint format ``DetectMultiBackend`` / ``_load`` read: the YAML dict, reference-named fp32 tensors,
    class names (the reference pickles whole nn.Modules instead, train.py:445-462)."""
    # state_dict() reads the device masters while they exist: no mode flip, a mid-epoch save leaves training undisturbed
    torch.save({"cfg": model.yaml, "state_dict": {k: v.detach().float().cpu() for k, v in model.state_dict().items()},
                "names": list(model.names)}, str(path))


class DetectMultiBackend:
    def __init__(self, weights="yolov3.pt", device=torch.device("cuda"), dnn=False, data=None, fp16=False, fuse=True):  # noqa: B008
        device = torch.device(device)
        if device.type != "cuda":
            raise RuntimeError("yolov3_b200 has no CPU path: DetectMultiBackend needs a CUDA (H100) device")
        if dnn:
            raise NotImplementedError("only the PyTorch ('pt') role of DetectMultiBackend is accelerated")
        if isinstance(weights, (list, tuple)) and len(weights) > 1:  # models/common.py:471: attempt_load(weights list) -> Ensemble
            from .tta import attempt_load

            model = attempt_load(list(weights), device=device, inplace=True, fuse=fuse)
        else:
            model = _load(weights, device)
            model.eval()
            if fuse:
                model.fuse()
        self.model = model
        self.stride = max(int(model.stride.max()), 32)
        self.names = model.names
        self.device, self.fp16, self.data = device, bool(fp16), data
        self.pt, self.nhwc = True, False
        self.jit = self.onnx = self.xml = self.engine = self.coreml = self.saved_model = self.pb = self.tflite = False
        self.edgetpu = self.tfjs = self.paddle = self.triton = self.dnn = False

    def forward(self, im, augment=False, visualize=False):
        """Returns what the wrapped model returns (models/common.py:655-656): ``(z, [p3, p4, p5])``; with ``fp16`` the
        outputs are cast to half like the reference's half model (the kernels always store bf16 / accumulate fp32)."""
        if im.dtype == torch.float16:
            im = im.float()
        y = self.model(im, augment=augment, visualize=visualize) if augment or visualize else self.model(im)
        if self.fp16:
            y = tuple(t.half() if isinstance(t, torch.Tensor) else [u.half() for u in t] for t in y)
        return y

    __call__ = forward

    def from_numpy(self, x):
        return torch.from_numpy(x).to(self.device) if isinstance(x, np.ndarray) else x

    def warmup(self, imgsz=(1, 3, 640, 640)):
        """One forward on an empty batch of shape ``imgsz``: builds (lowers, packs, allocates) the engine for that shape."""
        im = torch.empty(*imgsz, dtype=torch.half if self.fp16 else torch.float, device=self.device)
        self.forward(im)

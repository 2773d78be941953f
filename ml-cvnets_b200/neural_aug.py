"""RangeAugment (arXiv 2212.10553): learned brightness / contrast / noise ranges in front of the stem.

Host-side mirror of ``cvnets/neural_augmentor`` (neural_aug.py, utils/neural_aug_utils.py): same class names, constructor signatures, child
tree and ``state_dict`` keys (``neural_augmentor.{brightness,contrast,noise}._{low,high}``, 0-dim).  ``forward`` runs the fused kernels of
csrc/neural_aug.cu through ``functional.NeuralAugmentFn``: the order of the augmentations, the sample subsets, the magnitudes and the noise are
drawn on the device from the dropout generator (``ops.rng_next``), so a captured training step draws fresh values at every replay.
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Any, Optional

import torch
from torch import Tensor, nn

from . import functional as Fn

# (min_fn, max_fn) bounds of DistributionNeuralAugmentor's samplers (neural_aug.py:263-290); csrc/neural_aug.cu holds the same constants
_BOUNDS = {"brightness": ((0.1, 0.9), (1.1, 10.0)), "contrast": ((0.1, 0.9), (1.1, 10.0)), "noise": ((0.0, 0.00005), (0.0001, 1.0))}
_INIT = {"brightness": (0.5, 1.5), "contrast": (0.5, 1.5), "noise": (0.0, 0.1)}


class Clip(nn.Module):
    """neural_aug_utils.py:Clip: ``sigmoid(x) * (max - min) + min`` (soft clip)."""

    def __init__(self, min_val: float, max_val: float, hard_clip: Optional[bool] = False, *args, **kwargs) -> None:
        super().__init__()
        if hard_clip:
            raise NotImplementedError("Clip(hard_clip=True): no RangeAugment recipe uses it")
        self.min_val, self.max_val, self.hard_clip = min_val, max_val, hard_clip

    def forward(self, x: Any) -> Any:
        return torch.sigmoid(x) * (self.max_val - self.min_val) + self.min_val

    def __repr__(self):
        return "{}(min={}, max={}, clipping=soft)".format(self.__class__.__name__, self.min_val, self.max_val)


class UniformSampler(nn.Module):
    """neural_aug_utils.py:UniformSampler: learnable 0-dim ``_low`` / ``_high``; ``low`` / ``high`` through ``min_fn`` / ``max_fn``.  Drawing
    happens inside the fused augmentor kernels, so ``forward`` is not available on its own."""

    def __init__(self, low: float, high: float, min_fn: Optional[nn.Module] = None, max_fn: Optional[nn.Module] = None, *args, **kwargs):
        super().__init__()
        self._low = nn.Parameter(torch.tensor(low, dtype=torch.float))
        self._high = nn.Parameter(torch.tensor(high, dtype=torch.float))
        self.min_fn = min_fn
        self.max_fn = max_fn

    @property
    def low(self):
        return self.min_fn(self._low) if self.min_fn is not None else self._low

    @property
    def high(self):
        return self.max_fn(self._high) if self.max_fn is not None else self._high

    def forward(self, *args, **kwargs) -> Tensor:
        raise NotImplementedError("UniformSampler draws inside DistributionNeuralAugmentor's kernels; call the augmentor")


class DistributionNeuralAugmentor(nn.Module):
    """neural_aug.py:DistributionNeuralAugmentor.  ``forward(x)``: x fp32 [B, 3, H, W] in [0, 1] on CUDA -> the augmented image, clipped to
    [0, 1].  Inside ``engine.TrainStep`` the image is mixed first (``TrainStep.set_mix``), as the reference mixes before the model."""

    def __init__(self, opts, *args, **kwargs) -> None:
        super().__init__()
        self.opts = opts
        self.lr_multiplier = getattr(opts, "model.learn_augmentation.lr_multiplier", 1.0)
        if self.lr_multiplier != 1.0:
            raise NotImplementedError(f"model.learn_augmentation.lr_multiplier = {self.lr_multiplier}: only 1.0 (every recipe's value) is implemented")
        self.brightness = self.contrast = self.noise = None
        enabled = 0
        for k, name in enumerate(("brightness", "contrast", "noise")):
            if getattr(opts, f"model.learn_augmentation.{name}", False):
                (lo_min, lo_max), (hi_min, hi_max) = _BOUNDS[name]
                setattr(self, name, UniformSampler(low=_INIT[name][0], high=_INIT[name][1], min_fn=Clip(min_val=lo_min, max_val=lo_max),
                                                   max_fn=Clip(min_val=hi_min, max_val=hi_max)))
                enabled |= 1 << k
        if not enabled:
            raise ValueError("DistributionNeuralAugmentor needs at least one of model.learn_augmentation.{brightness,contrast,noise}")
        self._cfg = SimpleNamespace(enabled=enabled)

    def raw_parameters(self):
        """The enabled samplers' (_low, _high) in brightness, contrast, noise order (the kernels' order)."""
        return [p for s in (self.brightness, self.contrast, self.noise) if s is not None for p in (s._low, s._high)]

    def forward_with_sq(self, x: Tensor):
        """(x_aug, sq): sq fp64 [B, 3] holds sum over (h, w) of (x_aug - x_mix)^2 per (sample, channel), the input of the PSNR loss."""
        if not x.is_cuda:
            raise RuntimeError(f"DistributionNeuralAugmentor: ml-cvnets_b200 runs on CUDA (sm_90a) only and has no CPU fallback; got a {x.device} tensor")
        self._cfg.ws = getattr(self, "_ws", None)
        y, sq = Fn.NeuralAugmentFn.apply(x, self._cfg, *self.raw_parameters())
        y._cvb_premixed = True  # the stem must not mix it again
        return y, sq

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        y, sq = self.forward_with_sq(x)
        y._cvb_sq = sq  # engine.NeuralAugmentationLoss reads the squared errors from here instead of re-reading both images
        return y

    def __repr__(self):
        parts = [f"\n\t{n}={getattr(self, n)}, " for n in ("brightness", "contrast", "noise") if getattr(self, n) is not None]
        return "{}({})".format(self.__class__.__name__, "".join(parts))


def build_neural_augmentor(opts, *args, **kwargs) -> Optional[DistributionNeuralAugmentor]:
    """neural_aug.py:build_neural_augmentor, reading ``model.learn_augmentation.mode``."""
    mode = (getattr(opts, "model.learn_augmentation.mode", None) or "none").lower()
    if mode == "distribution":
        return DistributionNeuralAugmentor(opts=opts, *args, **kwargs)
    if mode == "basic":
        raise NotImplementedError("model.learn_augmentation.mode = 'basic' (BasicNeuralAugmentor) is not implemented; no recipe uses it")
    return None


def augmented_forward(model: nn.Module, x: Tensor):
    """BaseImageEncoder.forward with an augmentor (base_image_encoder.py:282-298)."""
    if model.training:
        x_aug = model.neural_augmentor(x)
        return {"augmented_tensor": x_aug, "logits": model.forward_classifier(x_aug)}
    return {"augmented_tensor": None, "logits": model.forward_classifier(x)}

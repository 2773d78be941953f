"""fp32 restatement of RangeAugment (cvnets/neural_augmentor/neural_aug.py DistributionNeuralAugmentor, utils/neural_aug_utils.py) and its PSNR
loss (loss_fn/neural_augmentation.py), pinned to tests/golden/range_augment_fp32.pt.

The random draws are INPUTS, like the dropout masks of the oracle: ``draws`` = {"order": [names], name: {"idx": LongTensor [n], "u": [n],
"eps": [n, 3, H, W] (noise only)}}.  ``draws_from_kernels`` reads the same structure out of the kernels' draw table and noise field."""
import math
from typing import Dict

import torch
import torch.nn.functional as F
from torch import Tensor

NAMES = ("brightness", "contrast", "noise")
AUG_KEYS = [f"neural_augmentor.{n}._{s}" for n in NAMES for s in ("low", "high")]
INIT = {"brightness": (0.5, 1.5), "contrast": (0.5, 1.5), "noise": (0.0, 0.1)}
BOUNDS = {"brightness": ((0.1, 0.9), (1.1, 10.0)), "contrast": ((0.1, 0.9), (1.1, 10.0)), "noise": ((0.0, 0.00005), (0.0001, 1.0))}


def low_high(name: str, raw_low: Tensor, raw_high: Tensor):
    (a, b), (c, d) = BOUNDS[name]
    return torch.sigmoid(raw_low) * (b - a) + a, torch.sigmoid(raw_high) * (d - c) + c


def augment(x: Tensor, raw: Dict[str, tuple], draws: Dict) -> Tensor:
    """raw[name] = (_low, _high) 0-dim tensors (differentiable); x [B, 3, H, W] fp32 (already mixed)."""
    for name in draws["order"]:
        d = draws[name]
        idx = d["idx"].to(x.device)
        lo, hi = low_high(name, *raw[name])
        m = (lo + d["u"].to(x) * (hi - lo)).view(-1, 1, 1, 1)
        xa = torch.index_select(x, 0, idx)
        if name == "brightness":
            xa = xa * m
        elif name == "contrast":
            xa = (1.0 - m) * torch.mean(xa, dim=[-1, -2], keepdim=True) + xa * m
        else:
            xa = xa + d["eps"].to(x) * m
        x = torch.index_copy(x, 0, idx, xa)
    return torch.clip(x, min=0.0, max=1.0)


def psnr_to_mse(psnr: float) -> float:
    return 10.0 ** ((20.0 * math.log10(255.0) - psnr) / 10.0)


def na_loss(x_aug: Tensor, x: Tensor, target_mse: float, alpha: float = 100.0) -> Tensor:
    pred_mse = torch.mean(((x_aug - x) * 255.0) ** 2, dim=[1, 2, 3])
    return F.smooth_l1_loss(pred_mse, torch.full_like(pred_mse, target_mse), reduction="mean") * (alpha / 65025.0)


def mixed(x: Tensor, mix) -> Tensor:
    """The batch mixing of cvb_stem_im2col_mix: mix = (mode, lam, x1, y1, x2, y2), partner x.roll(1, 0)."""
    mode, lam, x1, y1, x2, y2 = [float(v) for v in mix]
    xp = x.roll(1, 0)
    if mode == 1:
        return lam * x + (1.0 - lam) * xp
    if mode == 2:
        out = x.clone()
        out[:, :, int(y1):int(y2), int(x1):int(x2)] = xp[:, :, int(y1):int(y2), int(x1):int(x2)]
        return out
    return x


def draws_from_kernels(tab: Tensor, eps_field: Tensor) -> Dict:
    """The kernels' draw table (cvb_na_plan layout) and noise field (cvb_na_noise) as ``augment``'s draws."""
    tab = tab.float().cpu()
    B = eps_field.shape[0]
    cnt = int(tab[3])
    out = {"order": [NAMES[int(tab[p])] for p in range(cnt)]}
    for k, name in enumerate(NAMES):
        row = tab[4 + k * B: 4 + (k + 1) * B]
        idx = torch.nonzero(row >= 0).flatten()
        if idx.numel():
            out[name] = {"idx": idx, "u": row[idx], "eps": eps_field.float().cpu()[idx]}
    return out


def seeded_aug_params(seed: int) -> Dict[str, Tensor]:
    """The six 0-dim sampler parameters (state_dict keys of a model with an augmentor) near their initial values, deterministic in ``seed``."""
    g = torch.Generator().manual_seed(seed)
    return {f"neural_augmentor.{n}._{s}": torch.tensor(INIT[n][i] + 0.3 * float(torch.randn((), generator=g)))
            for n in NAMES for i, s in enumerate(("low", "high"))}


def raw_from(P: Dict[str, Tensor]) -> Dict[str, tuple]:
    return {n: (P[f"neural_augmentor.{n}._low"], P[f"neural_augmentor.{n}._high"]) for n in NAMES if f"neural_augmentor.{n}._low" in P}


def mixed_targets(y: Tensor, n_classes: int, mix) -> Tensor:
    """lam * onehot(y) + (1 - lam) * onehot(y.roll(1, 0)): the targets of a mixed batch (mode 0: plain one-hot)."""
    lam = float(mix[1]) if float(mix[0]) != 0 else 1.0
    return F.one_hot(y, n_classes).float() * lam + F.one_hot(y.roll(1, 0), n_classes).float() * (1.0 - lam)

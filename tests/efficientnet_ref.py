"""fp32 restatement of EfficientNet (cvnets/models/classification/efficientnet.py, config/efficientnet.py) and EfficientNetBlock
(cvnets/modules/efficientnet.py), built from the oracle's pieces (oracle/cvnets_oracle.py) and pinned to tests/golden/efficientnet_fp32.pt.

``efficientnet_block`` takes the stochastic-depth factor as an INPUT (``drop_mask``: one multiplicative factor per sample, 0 or 1 / (1 - p)),
like the oracle's ``transformer_encoder(drop_masks=...)``: no two generators draw the same Bernoulli samples, so the parity tests hand it the
factors the kernel under test used."""
import math
from typing import Dict, Optional

import torch
import torch.nn.functional as F
from torch import Tensor

from oracle import cvnets_oracle as O

# mode: (width_mult, depth_mult); block groups (expand_ratio, kernel, stride, in, out, num_layers) before scaling
COMPOUND_SCALING = {"b0": (1.0, 1.0), "b1": (1.0, 1.1), "b2": (1.1, 1.2), "b3": (1.2, 1.4), "b4": (1.4, 1.8), "b5": (1.6, 2.2), "b6": (1.8, 2.6),
                    "b7": (2.0, 3.1)}
BLOCKS = {"layer_1": [(1, 3, 1, 32, 16, 1)], "layer_2": [(6, 3, 2, 16, 24, 2)], "layer_3": [(6, 5, 2, 24, 40, 2)],
          "layer_4": [(6, 3, 2, 40, 80, 3), (6, 5, 1, 80, 112, 3)], "layer_5": [(6, 5, 2, 112, 192, 4), (6, 3, 1, 192, 320, 1)]}


def efficientnet_layout(mode: str = "b0", stochastic_depth_prob: float = 0.0):
    """[(prefix, expand_ratio, kernel, stride, cin, cout, sd_prob)] of every block, plus (stem channels, last channels)."""
    wm, dm = COMPOUND_SCALING[mode]
    groups = {n: [(e, k, s, O.make_divisible(ci * wm, 8), O.make_divisible(co * wm, 8), int(math.ceil(n_ * dm))) for e, k, s, ci, co, n_ in g]
              for n, g in BLOCKS.items()}
    total = sum(g[5] for gs in groups.values() for g in gs)
    out, prev = [], 0
    for name, gs in groups.items():
        count = 0
        for e, k, s, ci, co, n in gs:
            for i in range(n):
                out.append((f"{name}.{count}", e, k, s if i == 0 else 1, ci, co, round(stochastic_depth_prob * float(prev + count) / total, 4)))
                count += 1
                ci = co
        prev += count
    return out, groups["layer_1"][0][3], 4 * groups["layer_5"][-1][4]


def efficientnet_block_shapes(P: Dict, pre: str, cin: int, cout: int, expand_ratio: int, kernel_size: int):
    O.inverted_residual_se_shapes(P, pre, cin, cout, expand_ratio, use_se=True, kernel_size=kernel_size, squeeze_factor=expand_ratio * 4)


def efficientnet_shapes(mode: str = "b0", n_classes: int = 1000) -> Dict[str, Tensor]:
    blocks, c0, last = efficientnet_layout(mode)
    P = {}
    O._conv_bn(P, "conv_1", 3, c0, 3)
    for pre, e, k, _, ci, co, _ in blocks:
        efficientnet_block_shapes(P, pre, ci, co, e, k)
    O._conv_bn(P, "conv_1x1_exp", blocks[-1][5], last, 1)
    P["classifier.classifier_fc.weight"] = torch.empty(n_classes, last)
    P["classifier.classifier_fc.bias"] = torch.empty(n_classes)
    return P


def efficientnet_block(P, pre: str, x: Tensor, *, stride: int, training: bool = True, drop_mask: Optional[Tensor] = None) -> Tensor:
    """EfficientNetBlock.forward: InvertedResidualSE's block (swish, SE with swish fc1 and sigmoid scale), then with a residual
    x + StochasticDepth(block(x)); ``drop_mask`` [B] = per-sample factor (None: eval mode / p = 0, the identity)."""
    cout = P[pre + ".block.red_1x1.block.conv.weight"].shape[0]
    res = stride == 1 and x.shape[1] == cout
    y = O.inverted_residual_se(P, pre, x, stride=stride, act="swish", se_scale="sigmoid", fc_act="swish", training=training)
    if not res:
        return y
    y = y - x  # inverted_residual_se already added the residual
    if drop_mask is not None:
        y = y * drop_mask.view(-1, 1, 1, 1)
    return x + y


def efficientnet_forward(P, x: Tensor, *, mode: str = "b0", training: bool = True) -> Tensor:
    blocks, _, _ = efficientnet_layout(mode)
    h = O.conv_layer_2d(P, "conv_1", x, stride=2, training=training)
    for pre, _, _, s, _, _, _ in blocks:
        h = efficientnet_block(P, pre, h, stride=s, training=training)
    h = O.conv_layer_2d(P, "conv_1x1_exp", h, training=training)
    return F.linear(h.mean(dim=(2, 3)), P["classifier.classifier_fc.weight"], P["classifier.classifier_fc.bias"])

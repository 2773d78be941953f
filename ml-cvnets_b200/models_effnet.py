"""EfficientNet assembler -- mirror of cvnets/models/classification/efficientnet.py + config/efficientnet.py, modes b0 .. b7.  Same attribute
names / ``state_dict`` keys as the reference: conv_1, layer_1 .. layer_5 (EfficientNetBlock), conv_1x1_exp,
classifier.{global_pool, [classifier_dropout,] classifier_fc}.  Host code only: the stem, the blocks' stand-alone layers, the depthwise
3x3 / 5x5 walk kernels, SE, stochastic depth and the head are the library's kernels.

The recipes (examples/range_augment/classification/efficientnet_b{0..3}.yaml) train with SGD + Nesterov: ``TrainStep(model, optimizer="sgd")``.
"""
from __future__ import annotations

import argparse
import math
from typing import Dict, List, Optional, Tuple, Union

from torch import Tensor, nn

from .layers import ConvLayer2d, Dropout, GlobalPool, LinearLayer, norm_layers_tuple
from .modules import EfficientNetBlock, _require_cuda, make_divisible
from .neural_aug import augmented_forward, build_neural_augmentor

# mode: (width_mult, depth_mult, train_resolution)
_COMPOUND_SCALING = {"b0": (1.0, 1.0, 224), "b1": (1.0, 1.1, 240), "b2": (1.1, 1.2, 260), "b3": (1.2, 1.4, 300), "b4": (1.4, 1.8, 380),
                     "b5": (1.6, 2.2, 456), "b6": (1.8, 2.6, 528), "b7": (2.0, 3.1, 600)}
# (expand_ratio, kernel, stride, in_channels, out_channels, num_layers) per block group, before compound scaling
_BLOCKS = {"layer_1": [(1, 3, 1, 32, 16, 1)], "layer_2": [(6, 3, 2, 16, 24, 2)], "layer_3": [(6, 5, 2, 24, 40, 2)],
           "layer_4": [(6, 3, 2, 40, 80, 3), (6, 5, 1, 80, 112, 3)], "layer_5": [(6, 5, 2, 112, 192, 4), (6, 3, 1, 192, 320, 1)]}
LAYERS = ["layer_1", "layer_2", "layer_3", "layer_4", "layer_5"]


def default_effnet_opts(mode: str = "b0", n_classes: int = 1000, **extra) -> argparse.Namespace:
    """Model section of examples/range_augment/classification/efficientnet_b0.yaml (swish, batch_norm momentum 0.1, no stochastic depth, no
    classifier dropout)."""
    opts = argparse.Namespace()
    kv = {
        "model.classification.name": "efficientnet", "model.classification.n_classes": n_classes, "model.classification.efficientnet.mode": mode,
        "model.classification.efficientnet.stochastic_depth_prob": 0.0, "model.classification.classifier_dropout": 0.0,
        "model.normalization.name": "batch_norm", "model.normalization.momentum": 0.1, "model.activation.name": "swish",
        "model.layer.global_pool": "mean", "model.layer.conv_init": "kaiming_normal", "model.layer.linear_init": "normal",
        "model.layer.linear_init_std_dev": 0.01,
    }
    kv.update(extra)
    for k, v in kv.items():
        setattr(opts, k, v)
    return opts


def get_effnet_configuration(opts) -> Dict:
    """config/efficientnet.py:get_configuration: per layer a list of (expand_ratio, kernel, stride, in_channels, out_channels, num_layers)
    after width / depth scaling, ``last_channels`` and ``total_layers``."""
    mode = (getattr(opts, "model.classification.efficientnet.mode", None) or "").lower()
    if mode not in _COMPOUND_SCALING:
        raise NotImplementedError(f"EfficientNet modes are b0 .. b7, got {mode!r}")
    wm, dm, _ = _COMPOUND_SCALING[mode]
    cfg = {}
    for name, groups in _BLOCKS.items():
        cfg[name] = [(e, k, s, int(make_divisible(ci * wm, 8)), int(make_divisible(co * wm, 8)), int(math.ceil(n * dm)))
                     for e, k, s, ci, co, n in groups]
    cfg["last_channels"] = 4 * cfg["layer_5"][-1][4]
    cfg["total_layers"] = sum(g[5] for name in LAYERS for g in cfg[name])
    return cfg


class EfficientNet(nn.Module):
    def __init__(self, opts, *args, **kwargs) -> None:
        super().__init__()
        num_classes = getattr(opts, "model.classification.n_classes", 1000)
        classifier_dropout = getattr(opts, "model.classification.classifier_dropout", 0.0)
        sd_prob = getattr(opts, "model.classification.efficientnet.stochastic_depth_prob", 0.2)
        cfg = get_effnet_configuration(opts)
        self.opts, self.dilation = opts, 1
        c = cfg["layer_1"][0][3]
        self.neural_augmentor = build_neural_augmentor(opts)  # before conv_1: its parameters come first (base_image_encoder.py:50)
        self.conv_1 = ConvLayer2d(opts=opts, in_channels=3, out_channels=c, kernel_size=3, stride=2, use_norm=True, use_act=True)
        prev = 0
        for name in LAYERS:
            layer, prev = self._make_layer(opts, cfg[name], sd_prob, prev, cfg["total_layers"])
            setattr(self, name, layer)
        c, last = cfg["layer_5"][-1][4], cfg["last_channels"]
        self.conv_1x1_exp = ConvLayer2d(opts=opts, in_channels=c, out_channels=last, kernel_size=1, use_act=True, use_norm=True)
        self.classifier = nn.Sequential()
        self.classifier.add_module(name="global_pool", module=GlobalPool(pool_type=getattr(opts, "model.layer.global_pool", "mean"), keep_dim=False))
        if 0.0 < classifier_dropout < 1.0:
            self.classifier.add_module(name="classifier_dropout", module=Dropout(p=classifier_dropout, inplace=True))
        self.classifier.add_module(name="classifier_fc", module=LinearLayer(in_features=last, out_features=num_classes, bias=True))
        self.reset_parameters(opts)

    @staticmethod
    def _make_layer(opts, groups: List[Tuple], sd_prob: float, prev: int, total: int) -> Tuple[nn.Sequential, int]:
        block, count = [], 0
        for e, k, s, ci, co, n in groups:
            for i in range(n):
                p = round(sd_prob * float(prev + count) / total, 4)  # efficientnet.py:_make_layer
                block.append(EfficientNetBlock(stochastic_depth_prob=p, opts=opts, in_channels=ci, out_channels=co, kernel_size=k,
                                               stride=s if i == 0 else 1, expand_ratio=e, dilation=1, use_se=True, squeeze_factor=e * 4,
                                               act_fn_name="swish", se_scale_fn_name="sigmoid"))
                count += 1
                ci = co
        return nn.Sequential(*block), prev + count

    @classmethod
    def build_model(cls, opts, *args, **kwargs):
        return cls(opts, *args, **kwargs)

    def reset_parameters(self, opts) -> None:
        """cvnets/misc/init_utils.py with the recipe's kaiming_normal convs / normal(0.01) linear."""
        lin_std = getattr(opts, "model.layer.linear_init_std_dev", 0.01)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                nn.init.kaiming_normal_(m.weight, mode="fan_out")
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, norm_layers_tuple):
                if m.weight is not None:
                    nn.init.ones_(m.weight)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, LinearLayer):
                nn.init.normal_(m.weight, mean=0.0, std=lin_std)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    def extract_features(self, x: Tensor, *args, **kwargs) -> Tensor:
        x = self.conv_1(x)
        for name in LAYERS:
            x = getattr(self, name)(x)
        return self.conv_1x1_exp(x)

    def extract_end_points_all(self, x: Tensor, use_l5: Optional[bool] = True, use_l5_exp: Optional[bool] = False, *args, **kwargs) -> Dict[str, Tensor]:
        """base_image_encoder.py:extract_end_points_all."""
        _require_cuda(x, "EfficientNet")
        out = {}
        x = self.layer_1(self.conv_1(x))
        out["out_l1"] = x
        x = self.layer_2(x)
        out["out_l2"] = x
        x = self.layer_3(x)
        out["out_l3"] = x
        x = self.layer_4(x)
        out["out_l4"] = x
        if use_l5:
            x = self.layer_5(x)
            out["out_l5"] = x
            if use_l5_exp:
                out["out_l5_exp"] = self.conv_1x1_exp(x)
        return out

    def forward_classifier(self, x: Tensor, *args, **kwargs) -> Tensor:
        _require_cuda(x, "EfficientNet")
        x = self.classifier.global_pool(self.extract_features(x))
        if hasattr(self.classifier, "classifier_dropout"):
            x = self.classifier.classifier_dropout(x)
        return self.classifier.classifier_fc(x)

    def forward(self, x: Tensor, *args, **kwargs) -> Union[Tensor, Dict[str, Optional[Tensor]]]:
        if self.neural_augmentor is not None:
            return augmented_forward(self, x)
        return self.forward_classifier(x)

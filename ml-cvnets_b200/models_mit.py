"""MobileViT (v1) assembler -- mirror of cvnets/models/classification/mobilevit.py:19-300 + config/mobilevit.py:14-200 (SURVEY.md 8a rows a9,
a15; BASELINE.json configs[0]: MobileViT-XXS forward at 1x3x256x256).  Same attribute names / ``state_dict`` keys as the reference:
conv_1, layer_1 .. layer_5, conv_1x1_exp, classifier.{global_pool, [dropout,] fc}.  Host code only; every kernel is the library's.
"""
from __future__ import annotations

import argparse
from typing import Dict, Optional, Tuple, Union

from torch import Tensor, nn

from .layers import ConvLayer2d, Dropout, GlobalPool, LinearLayer, norm_layers_tuple
from .modules import InvertedResidual, MobileViTBlock, _require_cuda
from .neural_aug import augmented_forward, build_neural_augmentor


def default_mit_opts(mode: str = "xx_small", n_classes: int = 1000, **extra) -> argparse.Namespace:
    """config/classification/imagenet/mobilevit.yaml model section (dropout 0.1 / attn_dropout 0 / classifier_dropout 0.1, swish)."""
    opts = argparse.Namespace()
    kv = {
        "model.classification.name": "mobilevit", "model.classification.n_classes": n_classes, "model.classification.mit.mode": mode,
        "model.classification.classifier_dropout": 0.1, "model.classification.mit.dropout": 0.1, "model.classification.mit.ffn_dropout": 0.0,
        "model.classification.mit.attn_dropout": 0.0, "model.classification.mit.number_heads": 4, "model.classification.mit.head_dim": None,
        "model.classification.mit.no_fuse_local_global_features": False, "model.classification.mit.conv_kernel_size": 3,
        "model.normalization.name": "batch_norm", "model.normalization.momentum": 0.1, "model.activation.name": "swish",
        "model.layer.global_pool": "mean", "model.layer.conv_init": "kaiming_normal", "model.layer.linear_init": "trunc_normal",
        "model.layer.linear_init_std_dev": 0.02,
    }
    kv.update(extra)
    for k, v in kv.items():
        setattr(opts, k, v)
    return opts


def get_mit_configuration(opts) -> Dict:
    """cvnets/models/classification/config/mobilevit.py:14-200."""
    mode = getattr(opts, "model.classification.mit.mode", "small").lower()
    head_dim = getattr(opts, "model.classification.mit.head_dim", None)
    num_heads = getattr(opts, "model.classification.mit.number_heads", 4)
    table = {  # mode: (mv2 expand, layer1 out, layer2 out, [(out, transformer dim, ffn dim, blocks)] x 3)
        "xx_small": (2, 16, 24, [(48, 64, 128, 2), (64, 80, 160, 4), (80, 96, 192, 3)]),
        "x_small": (4, 32, 48, [(64, 96, 192, 2), (80, 120, 240, 4), (96, 144, 288, 3)]),
        "small": (4, 32, 64, [(96, 144, 288, 2), (128, 192, 384, 4), (160, 240, 480, 3)]),
    }
    if mode not in table:
        raise NotImplementedError(f"MobileViT mode {mode}")
    e, c1, c2, mits = table[mode]
    cfg = {"layer1": {"out_channels": c1, "expand_ratio": e, "num_blocks": 1, "stride": 1, "block_type": "mv2"},
           "layer2": {"out_channels": c2, "expand_ratio": e, "num_blocks": 3, "stride": 2, "block_type": "mv2"},
           "last_layer_exp_factor": 4}
    for i, (co, d, f, n) in enumerate(mits):
        cfg[f"layer{3 + i}"] = {"out_channels": co, "transformer_channels": d, "ffn_dim": f, "transformer_blocks": n, "patch_h": 2, "patch_w": 2,
                                "stride": 2, "mv_expand_ratio": e, "head_dim": head_dim, "num_heads": num_heads, "block_type": "mobilevit"}
    return cfg


class MobileViT(nn.Module):
    def __init__(self, opts, *args, **kwargs) -> None:
        super().__init__()
        num_classes = getattr(opts, "model.classification.n_classes", 1000)
        classifier_dropout = getattr(opts, "model.classification.classifier_dropout", 0.0)
        cfg = get_mit_configuration(opts)
        self.opts, self.dilation = opts, 1
        self.neural_augmentor = build_neural_augmentor(opts)  # before conv_1: its parameters come first (base_image_encoder.py:50)
        self.conv_1 = ConvLayer2d(opts=opts, in_channels=3, out_channels=16, kernel_size=3, stride=2, use_norm=True, use_act=True)
        c = 16
        for li in range(1, 6):
            layer, c = self._make_layer(opts, c, cfg[f"layer{li}"])
            setattr(self, f"layer_{li}", layer)
        exp_channels = min(cfg["last_layer_exp_factor"] * c, 960)
        self.conv_1x1_exp = ConvLayer2d(opts=opts, in_channels=c, out_channels=exp_channels, kernel_size=1, stride=1, use_act=True, use_norm=True)
        self.classifier = nn.Sequential()
        self.classifier.add_module(name="global_pool", module=GlobalPool(pool_type=getattr(opts, "model.layer.global_pool", "mean"), keep_dim=False))
        if 0.0 < classifier_dropout < 1.0:
            self.classifier.add_module(name="dropout", module=Dropout(p=classifier_dropout, inplace=True))
        self.classifier.add_module(name="fc", module=LinearLayer(in_features=exp_channels, out_features=num_classes, bias=True))
        self.reset_parameters(opts)

    def _make_layer(self, opts, input_channel: int, cfg: Dict) -> Tuple[nn.Sequential, int]:
        if cfg.get("block_type", "mobilevit").lower() != "mobilevit":
            block, out_c = [], cfg["out_channels"]
            for i in range(cfg.get("num_blocks", 2)):
                block.append(InvertedResidual(opts=opts, in_channels=input_channel, out_channels=out_c, stride=cfg.get("stride", 1) if i == 0 else 1,
                                              expand_ratio=cfg.get("expand_ratio", 4)))
                input_channel = out_c
            return nn.Sequential(*block), input_channel
        block = []
        if cfg.get("stride", 1) == 2:
            block.append(InvertedResidual(opts=opts, in_channels=input_channel, out_channels=cfg["out_channels"], stride=2,
                                          expand_ratio=cfg.get("mv_expand_ratio", 4), dilation=1))
            input_channel = cfg["out_channels"]
        d = cfg["transformer_channels"]
        head_dim = cfg.get("head_dim") or d // (cfg.get("num_heads") or 4)
        block.append(MobileViTBlock(
            opts=opts, in_channels=input_channel, transformer_dim=d, ffn_dim=cfg["ffn_dim"], n_transformer_blocks=cfg.get("transformer_blocks", 1),
            patch_h=cfg.get("patch_h", 2), patch_w=cfg.get("patch_w", 2), dropout=getattr(opts, "model.classification.mit.dropout", 0.1),
            ffn_dropout=getattr(opts, "model.classification.mit.ffn_dropout", 0.0), attn_dropout=getattr(opts, "model.classification.mit.attn_dropout", 0.1),
            head_dim=head_dim, no_fusion=getattr(opts, "model.classification.mit.no_fuse_local_global_features", False),
            conv_ksize=getattr(opts, "model.classification.mit.conv_kernel_size", 3)))
        return nn.Sequential(*block), input_channel

    @classmethod
    def build_model(cls, opts, *args, **kwargs):
        return cls(opts, *args, **kwargs)

    def reset_parameters(self, opts) -> None:
        lin_std = getattr(opts, "model.layer.linear_init_std_dev", 0.02)
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
                nn.init.trunc_normal_(m.weight, mean=0.0, std=lin_std)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    def extract_features(self, x: Tensor, *args, **kwargs) -> Tensor:
        x = self.conv_1(x)
        for li in range(1, 6):
            x = getattr(self, f"layer_{li}")(x)
        return self.conv_1x1_exp(x)

    def forward(self, x: Tensor, *args, **kwargs) -> Union[Tensor, Dict[str, Optional[Tensor]]]:
        if self.neural_augmentor is not None:
            return augmented_forward(self, x)
        return self.forward_classifier(x)

    def forward_classifier(self, x: Tensor, *args, **kwargs) -> Tensor:
        _require_cuda(x, "MobileViT")
        x = self.extract_features(x)
        x = self.classifier.global_pool(x)
        if hasattr(self.classifier, "dropout"):
            x = self.classifier.dropout(x)  # classifier_dropout 0.1 of the recipe (mobilevit.py:110-113): hashed-mask kernel in training, identity in eval
        return self.classifier.fc(x)

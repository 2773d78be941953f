"""MobileViTv2 assembler (mirror of cvnets/models/classification/mobilevit_v2.py:19-226 + base_image_encoder.py:261-301).

The assembler is host code the reference keeps in Python; it instantiates the drop-in modules and owns nothing else.
With the reference importable, ``register.register_with_cvnets()`` exposes the same class to ``get_model()``
(INTEGRATION.md); standalone (GPU box, no reference) it is constructed directly: ``MobileViTv2(default_opts())``.
"""
from __future__ import annotations

import argparse
from types import SimpleNamespace
from typing import Dict, List, Optional, Tuple, Union

import torch
from torch import Tensor, nn

from . import functional as Fn
from .layers import ConvLayer2d, GlobalPool, Identity, LinearLayer, _bind, _need_cuda, norm_layers_tuple
from .modules import InvertedResidual, MobileViTBlockv2, make_divisible
from .neural_aug import augmented_forward, build_neural_augmentor
from .ops import PreparedWeights as PW


def default_opts(width_multiplier: float = 1.0, n_classes: int = 1000, **extra) -> argparse.Namespace:
    """The subset of the reference's flat dotted-key namespace the hot path reads (options/utils.py:34-42)."""
    opts = argparse.Namespace()
    kv = {
        "model.classification.name": "mobilevit_v2",
        "model.classification.n_classes": n_classes,
        "model.classification.mitv2.width_multiplier": width_multiplier,
        "model.classification.mitv2.attn_norm_layer": "layer_norm_2d",
        "model.classification.mitv2.dropout": 0.0,
        "model.classification.mitv2.attn_dropout": 0.0,
        "model.classification.mitv2.ffn_dropout": 0.0,
        "model.normalization.name": "batch_norm",
        "model.normalization.momentum": 0.1,
        "model.activation.name": "swish",
        "model.layer.global_pool": "mean",
        "model.layer.conv_init": "kaiming_normal",
        "model.layer.linear_init": "trunc_normal",
        "model.layer.linear_init_std_dev": 0.02,
    }
    kv.update(extra)
    for k, v in kv.items():
        setattr(opts, k, v)
    return opts


def get_configuration(opts) -> Dict:
    """cvnets/models/classification/config/mobilevit_v2.py:11-77."""
    wm = getattr(opts, "model.classification.mitv2.width_multiplier", 1.0)
    layer_0_dim = int(make_divisible(max(16, min(64, 32 * wm)), divisor=8, min_value=16))

    def mit(c, d, n):
        return {"out_channels": int(make_divisible(c * wm, divisor=8)), "attn_unit_dim": int(make_divisible(d * wm, divisor=8)),
                "ffn_multiplier": 2, "attn_blocks": n, "patch_h": 2, "patch_w": 2, "stride": 2, "mv_expand_ratio": 2,
                "block_type": "mobilevit"}

    return {
        "layer0": {"img_channels": 3, "out_channels": layer_0_dim},
        "layer1": {"out_channels": int(make_divisible(64 * wm, divisor=16)), "expand_ratio": 2, "num_blocks": 1, "stride": 1, "block_type": "mv2"},
        "layer2": {"out_channels": int(make_divisible(128 * wm, divisor=8)), "expand_ratio": 2, "num_blocks": 2, "stride": 2, "block_type": "mv2"},
        "layer3": mit(256, 128, 2), "layer4": mit(384, 192, 4), "layer5": mit(512, 256, 3),
        "last_layer_exp_factor": 4,
    }


class MobileViTv2(nn.Module):
    """Same attribute names / state_dict keys as the reference model: conv_1, layer_1..layer_5, conv_1x1_exp, classifier."""

    def __init__(self, opts, *args, **kwargs) -> None:
        super().__init__()
        num_classes = getattr(opts, "model.classification.n_classes", 1000)
        pool_type = getattr(opts, "model.layer.global_pool", "mean")
        cfg = get_configuration(opts)
        self.opts = opts
        # segmentation heads (DeepLabv3 / PSPNet) ask for output_stride 8 / 16: the stride of layer_4 / layer_5 becomes dilation
        # (base_image_encoder.py:38-47)
        self.dilation = 1
        output_stride = kwargs.get("output_stride", None)
        self.dilate_l4, self.dilate_l5 = output_stride == 8, output_stride in (8, 16)
        self.output_stride = output_stride
        self.model_conf_dict = dict()
        c0 = cfg["layer0"]["out_channels"]
        self.neural_augmentor = build_neural_augmentor(opts)  # before conv_1: its parameters come first (base_image_encoder.py:50)
        self.conv_1 = ConvLayer2d(opts=opts, in_channels=cfg["layer0"]["img_channels"], out_channels=c0, kernel_size=3, stride=2,
                                  use_norm=True, use_act=True)
        self.model_conf_dict["conv1"] = {"in": 3, "out": c0}
        in_c = c0
        for li in range(1, 6):
            layer, out_c = self._make_layer(opts=opts, input_channel=in_c, cfg=cfg[f"layer{li}"],
                                            dilate={4: self.dilate_l4, 5: self.dilate_l5}.get(li, False))
            setattr(self, f"layer_{li}", layer)
            self.model_conf_dict[f"layer{li}"] = {"in": in_c, "out": out_c}
            in_c = out_c
        self.conv_1x1_exp = Identity()
        self.model_conf_dict["exp_before_cls"] = {"in": in_c, "out": in_c}
        self.classifier = nn.Sequential(GlobalPool(pool_type=pool_type, keep_dim=False),
                                        LinearLayer(in_features=in_c, out_features=num_classes, bias=True))
        self._head = None
        self.reset_parameters(opts)
        # lazy module boundaries (functional.LazyBN): a module whose successor in THIS chain is a hot-path module without a residual on its
        # input hands over its output pre-BatchNorm; the successor normalises on load.  Active only inside extract_features().
        self.fuse_boundaries = True
        chain = [self.conv_1] + [m for li in range(1, 6) for m in getattr(self, f"layer_{li}")]
        for prod, cons in zip(chain[:-1], chain[1:]):
            takes_lazy = isinstance(cons, MobileViTBlockv2) or (isinstance(cons, InvertedResidual) and not cons.use_res_connect)
            object.__setattr__(prod, "_lazy_out", bool(takes_lazy))
        self._chain = chain

    # ---- construction (mobilevit_v2.py:137-226)
    def _make_layer(self, opts, input_channel, cfg: Dict, dilate: Optional[bool] = False) -> Tuple[nn.Sequential, int]:
        if cfg.get("block_type", "mobilevit").lower() == "mobilevit":
            return self._make_mit_layer(opts=opts, input_channel=input_channel, cfg=cfg, dilate=dilate)
        return self._make_mobilenet_layer(opts=opts, input_channel=input_channel, cfg=cfg)

    @staticmethod
    def _make_mobilenet_layer(opts, input_channel: int, cfg: Dict) -> Tuple[nn.Sequential, int]:
        output_channels = cfg.get("out_channels")
        block = []
        for i in range(cfg.get("num_blocks", 2)):
            stride = cfg.get("stride", 1) if i == 0 else 1
            block.append(InvertedResidual(opts=opts, in_channels=input_channel, out_channels=output_channels, stride=stride,
                                          expand_ratio=cfg.get("expand_ratio", 4)))
            input_channel = output_channels
        return nn.Sequential(*block), input_channel

    def _make_mit_layer(self, opts, input_channel, cfg: Dict, dilate: Optional[bool] = False) -> Tuple[nn.Sequential, int]:
        prev_dilation = self.dilation
        block = []
        stride = cfg.get("stride", 1)
        if stride == 2:
            if dilate:  # mobilevit_v2.py:183-186
                self.dilation *= 2
                stride = 1
            block.append(InvertedResidual(opts=opts, in_channels=input_channel, out_channels=cfg.get("out_channels"), stride=stride,
                                          expand_ratio=cfg.get("mv_expand_ratio", 4), dilation=prev_dilation))
            input_channel = cfg.get("out_channels")
        block.append(MobileViTBlockv2(
            opts=opts, in_channels=input_channel, attn_unit_dim=cfg["attn_unit_dim"], ffn_multiplier=cfg.get("ffn_multiplier"),
            n_attn_blocks=cfg.get("attn_blocks", 1), patch_h=cfg.get("patch_h", 2), patch_w=cfg.get("patch_w", 2),
            dropout=getattr(opts, "model.classification.mitv2.dropout", 0.0),
            ffn_dropout=getattr(opts, "model.classification.mitv2.ffn_dropout", 0.0),
            attn_dropout=getattr(opts, "model.classification.mitv2.attn_dropout", 0.0), conv_ksize=3,
            attn_norm_layer=getattr(opts, "model.classification.mitv2.attn_norm_layer", "layer_norm_2d"), dilation=self.dilation))
        return nn.Sequential(*block), input_channel

    @classmethod
    def build_model(cls, opts, *args, **kwargs):
        return cls(opts, *args, **kwargs)

    # ---- weight init (cvnets/misc/init_utils.py:110-150, called from base_model.py:69-71)
    def reset_parameters(self, opts) -> None:
        conv_init = getattr(opts, "model.layer.conv_init", "kaiming_normal")
        lin_init = getattr(opts, "model.layer.linear_init", "normal")
        lin_std = getattr(opts, "model.layer.linear_init_std_dev", 0.01)
        for m in self.modules():
            if isinstance(m, nn.Conv2d):
                if conv_init == "kaiming_normal":
                    nn.init.kaiming_normal_(m.weight, mode="fan_out")
                elif conv_init == "kaiming_uniform":
                    nn.init.kaiming_uniform_(m.weight, mode="fan_out")
                else:
                    nn.init.xavier_uniform_(m.weight)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, norm_layers_tuple):
                if m.weight is not None:
                    nn.init.ones_(m.weight)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)
            elif isinstance(m, LinearLayer):
                if lin_init == "trunc_normal":
                    nn.init.trunc_normal_(m.weight, mean=0.0, std=lin_std)
                elif lin_init == "normal":
                    nn.init.normal_(m.weight, mean=0.0, std=lin_std)
                else:
                    nn.init.xavier_uniform_(m.weight)
                if m.bias is not None:
                    nn.init.zeros_(m.bias)

    # ---- optimizer grouping (cvnets/misc/common.py:122-176 via base_model.py:92-123)
    def get_trainable_parameters(self, weight_decay: Optional[float] = 0.0, no_decay_bn_filter_bias: Optional[bool] = False,
                                 *args, **kwargs) -> Tuple[List[Dict], List[float]]:
        with_decay, without_decay = [], []
        for p in self.parameters():
            if not p.requires_grad:
                continue
            (without_decay if (no_decay_bn_filter_bias and p.dim() == 1) else with_decay).append(p)
        groups = [{"params": with_decay, "weight_decay": weight_decay}]
        if without_decay:
            groups.append({"params": without_decay, "weight_decay": 0.0})
        return groups, [1.0] * len(groups)

    # ---- forward (base_image_encoder.py:261-301)
    def extract_features(self, x: Tensor, *args, **kwargs) -> Tensor:
        for m in self._chain:
            object.__setattr__(m, "_lazy_active", bool(self.fuse_boundaries))
        try:
            x = self.conv_1(x)
            x = self.layer_1(x)
            x = self.layer_2(x)
            x = self.layer_3(x)
            x = self.layer_4(x)
            x = self.layer_5(x)
        finally:
            for m in self._chain:
                object.__setattr__(m, "_lazy_active", False)
        return self.conv_1x1_exp(x)

    # ---- feature maps for down-stream heads (base_image_encoder.py:206-276); every returned map is materialised (no lazy boundaries)
    def extract_end_points_all(self, x: Tensor, use_l5: Optional[bool] = True, use_l5_exp: Optional[bool] = False, *args, **kwargs) -> Dict[str, Tensor]:
        _need_cuda(x, "MobileViTv2")
        out_dict = {}
        x = self.layer_1(self.conv_1(x))
        out_dict["out_l1"] = x
        x = self.layer_2(x)
        out_dict["out_l2"] = x
        x = self.layer_3(x)
        out_dict["out_l3"] = x
        x = self.layer_4(x)
        out_dict["out_l4"] = x
        if use_l5:
            x = self.layer_5(x)
            out_dict["out_l5"] = x
            if use_l5_exp:
                out_dict["out_l5_exp"] = self.conv_1x1_exp(x)
        return out_dict

    def extract_end_points_l4(self, x: Tensor, *args, **kwargs) -> Dict[str, Tensor]:
        return self.extract_end_points_all(x, use_l5=False)

    def forward_classifier(self, x: Tensor, *args, **kwargs) -> Tensor:
        x = self.extract_features(x)
        lin = self.classifier[1]
        if self._head is None:
            prep = PW()
            npad = (lin.out_features + 7) // 8 * 8
            self._head = SimpleNamespace(prep=prep,
                                         i_w=prep.add(lin.weight, PW.KIND_ROWMAJOR, dst_rows=npad),
                                         i_wt=prep.add(lin.weight, PW.KIND_TRANSPOSED, ldd=npad),
                                         i_b=prep.add(lin.bias, PW.KIND_VECTOR_F32, dst_rows=npad))
        head = _bind(self, self._head, [lin.weight, lin.bias])
        return Fn.PoolLinearFn.apply(Fn.to_bf16_cl(x), head, lin.weight, lin.bias)

    def forward(self, x: Tensor, *args, **kwargs) -> Union[Tensor, Dict[str, Optional[Tensor]]]:
        _need_cuda(x, "MobileViTv2")
        if self.neural_augmentor is not None:
            return augmented_forward(self, x)
        return self.forward_classifier(x)

"""MobileViTv2 assembler (mirror of cvnets/models/classification/mobilevit_v2.py:19-226 + base_image_encoder.py:261-301).

The assembler is host code the reference keeps in Python; it instantiates the drop-in modules and owns nothing else.
With the reference importable, ``register.register_with_cvnets()`` exposes the same class to ``get_model()``
(INTEGRATION.md); standalone (GPU box, no reference) it is constructed directly: ``MobileViTv2(default_opts())``.
"""
from __future__ import annotations

import argparse
from types import SimpleNamespace
from typing import Dict, Optional, Tuple

from torch import Tensor, nn

from . import functional as Fn
from .layers import ConvLayer2d, GlobalPool, Identity, LinearLayer, _bind
from .models_base import ImageEncoder, extract_end_points_all, init_weights, make_mobilenet_layer
from .modules import InvertedResidual, MobileViTBlockv2, make_divisible
from .ops import PreparedWeights as PW


def default_opts(width_multiplier: float = 1.0, n_classes: int = 1000, **extra) -> argparse.Namespace:
    """The subset of the reference's flat dotted-key namespace the hot path reads (options/utils.py:34-42)."""
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
    return argparse.Namespace(**{**kv, **extra})


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


class MobileViTv2(ImageEncoder):
    """Same attribute names / state_dict keys as the reference model: conv_1, layer_1..layer_5, conv_1x1_exp, classifier."""

    def __init__(self, opts, *args, **kwargs) -> None:
        super().__init__(opts)
        num_classes = getattr(opts, "model.classification.n_classes", 1000)
        pool_type = getattr(opts, "model.layer.global_pool", "mean")
        cfg = get_configuration(opts)
        # segmentation heads (DeepLabv3 / PSPNet) ask for output_stride 8 / 16: the stride of layer_4 / layer_5 becomes dilation
        # (base_image_encoder.py:38-47)
        self.dilation = 1
        output_stride = kwargs.get("output_stride", None)
        self.dilate_l4, self.dilate_l5 = output_stride == 8, output_stride in (8, 16)
        self.output_stride = output_stride
        self.model_conf_dict = dict()
        c0 = cfg["layer0"]["out_channels"]
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
        return make_mobilenet_layer(opts=opts, input_channel=input_channel, cfg=cfg)

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

    # ---- weight init (cvnets/misc/init_utils.py:110-150, called from base_model.py:69-71)
    def reset_parameters(self, opts) -> None:
        init_weights(self.modules(), getattr(opts, "model.layer.conv_init", "kaiming_normal"), getattr(opts, "model.layer.linear_init", "normal"),
                     getattr(opts, "model.layer.linear_init_std_dev", 0.01))

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

    extract_end_points_all = extract_end_points_all

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

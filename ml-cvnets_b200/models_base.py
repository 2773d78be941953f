"""What the image classifiers share (mirror of cvnets/models/classification/base_image_encoder.py and cvnets/misc/init_utils.py:110-150):
the base class ``ImageEncoder`` (augmentor, ``build_model``, optimizer groups, the RangeAugment forward), the weight init, the feature
pyramid of the conv backbones and the MobileNetV2 stage.  Host code only."""
from __future__ import annotations

from typing import Dict, List, Optional, Tuple, Union

from torch import Tensor, nn

from .layers import LinearLayer, _need_cuda, norm_layers_tuple
from .modules import InvertedResidual
from .neural_aug import build_neural_augmentor


def init_weights(modules, conv_init: str, linear_init: str, linear_std: float) -> None:
    """init_utils.py:110-150: Conv2d by ``conv_init``, norm layers to (1, 0), LinearLayer by ``linear_init`` with std ``linear_std``, biases
    to zero; an unknown method is xavier_uniform."""
    for m in modules:
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
            if linear_init == "trunc_normal":
                nn.init.trunc_normal_(m.weight, mean=0.0, std=linear_std)
            elif linear_init == "normal":
                nn.init.normal_(m.weight, mean=0.0, std=linear_std)
            else:
                nn.init.xavier_uniform_(m.weight)
            if m.bias is not None:
                nn.init.zeros_(m.bias)


def make_mobilenet_layer(opts, input_channel: int, cfg: Dict) -> Tuple[nn.Sequential, int]:
    """A MobileNetV2 stage of ``cfg["num_blocks"]`` InvertedResiduals, the first with ``cfg["stride"]`` (mobilevit_v2.py:151-171,
    mobilevit.py:207-227)."""
    output_channels = cfg.get("out_channels")
    block = []
    for i in range(cfg.get("num_blocks", 2)):
        stride = cfg.get("stride", 1) if i == 0 else 1
        block.append(InvertedResidual(opts=opts, in_channels=input_channel, out_channels=output_channels, stride=stride,
                                      expand_ratio=cfg.get("expand_ratio", 4)))
        input_channel = output_channels
    return nn.Sequential(*block), input_channel


def extract_end_points_all(self, x: Tensor, use_l5: Optional[bool] = True, use_l5_exp: Optional[bool] = False, *args,
                           **kwargs) -> Dict[str, Tensor]:
    """Feature maps for down-stream heads (base_image_encoder.py:206-276); every returned map is materialised (no lazy boundaries).  A
    class attribute of the conv backbones (conv_1, layer_1 .. layer_5, conv_1x1_exp), not of ImageEncoder: ViT's version differs."""
    _need_cuda(x, type(self).__name__)
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


class ImageEncoder(nn.Module):
    """base_image_encoder.py:BaseImageEncoder.  Subclasses build their children after ``super().__init__(opts)`` and provide
    ``forward_classifier``."""

    def __init__(self, opts) -> None:
        super().__init__()
        self.opts = opts
        self.neural_augmentor = build_neural_augmentor(opts)  # the first child: its parameters come first (base_image_encoder.py:50)

    @classmethod
    def build_model(cls, opts, *args, **kwargs):
        return cls(opts, *args, **kwargs)

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

    def forward(self, x: Tensor, *args, **kwargs) -> Union[Tensor, Dict[str, Optional[Tensor]]]:
        """Logits; with a RangeAugment augmentor the reference's {"augmented_tensor", "logits"} (base_image_encoder.py:282-298),
        augmented_tensor None in eval mode."""
        _need_cuda(x, type(self).__name__)
        if self.neural_augmentor is None:
            return self.forward_classifier(x)
        if self.training:
            x_aug = self.neural_augmentor(x)
            return {"augmented_tensor": x_aug, "logits": self.forward_classifier(x_aug)}
        return {"augmented_tensor": None, "logits": self.forward_classifier(x)}

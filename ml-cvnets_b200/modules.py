"""Host-side mirror of ``cvnets.modules`` for the hot path (drop-in ``nn.Module``s, see layers.py for the contract).

``InvertedResidual`` (cvnets/modules/mobilenetv2.py:141-246), ``LinearAttnFFN`` (cvnets/modules/transformer.py:159-264)
and ``MobileViTBlockv2`` (cvnets/modules/mobilevit_block.py:329-667): identical constructor signatures, child tree and
``state_dict`` keys; ``forward`` dispatches to the autograd Functions in functional.py (hand-written sm_90a kernels).
"""
from __future__ import annotations

from types import SimpleNamespace
from typing import Optional, Sequence, Tuple, Union

import numpy as np
import torch
from torch import Tensor, nn

from . import functional as Fn
from .layers import (AdaptiveAvgPool2d, ConvLayer2d, Dropout, Identity, LinearLayer, LinearSelfAttention, MultiHeadAttention, StochasticDepth,
                     _bind, _need_cuda, build_activation_layer, get_normalization_layer)
from .ops import PreparedWeights as PW


def make_divisible(v, divisor: int = 8, min_value=None):
    """utils/math_utils.py:9-30."""
    if min_value is None:
        min_value = divisor
    new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
    if new_v < 0.9 * v:
        new_v += divisor
    return new_v


class BaseModule(nn.Module):
    """cvnets/modules/base_module.py:12-22."""

    def __init__(self, *args, **kwargs) -> None:
        super().__init__()

    def forward(self, x, *args, **kwargs):
        raise NotImplementedError


# ------------------------------------------------------------------------------------------------ lazy module boundaries
def _lazy_out(module) -> bool:
    """True while the model assembler runs its own chain and has marked this module's consumer as one of ours (functional.LazyBN)."""
    return bool(getattr(module, "_lazy_out", False) and getattr(module, "_lazy_active", False))


def _tag(out: Tensor, cfg) -> Tensor:
    if cfg.lazy_out:
        out._cvb_lazy = cfg.last_lazy  # the tensor is PRE-BatchNorm; only the next hot-path module may consume it
    return out


def _lazy_in(x: Tensor):
    return getattr(x, "_cvb_lazy", None)


# -------------------------------------------------------------------------------------------------------------- stem
def _stem_forward(layer: ConvLayer2d, x: Tensor) -> Tensor:
    _need_cuda(x, "ConvLayer2d(stem)")
    if layer._stem is None:
        prep = PW()
        cfg = SimpleNamespace(prep=prep, i_w=prep.add(layer.block.conv.weight, PW.KIND_ROWMAJOR, ldd=32))
        layer._stem = cfg
    cfg = layer._stem
    cfg.bn = Fn.bn_cfg(layer.block.norm)
    cfg.lazy_out = _lazy_out(layer)
    _bind(layer, cfg, [layer.block.conv.weight, layer.block.norm.weight, layer.block.norm.bias])
    return _tag(Fn.StemFn.apply(x, cfg, *cfg.plist), cfg)


# ---------------------------------------------------------------------------------------------------- InvertedResidual
class InvertedResidual(BaseModule):
    def __init__(self, opts, in_channels: int, out_channels: int, stride: int, expand_ratio: Union[int, float], dilation: int = 1,
                 skip_connection: Optional[bool] = True, *args, **kwargs) -> None:
        assert stride in [1, 2]
        hidden_dim = make_divisible(int(round(in_channels * expand_ratio)), 8)
        super().__init__()
        block = nn.Sequential()
        if expand_ratio != 1:
            block.add_module("exp_1x1", ConvLayer2d(opts, in_channels=in_channels, out_channels=hidden_dim, kernel_size=1,
                                                    use_act=True, use_norm=True))
        block.add_module("conv_3x3", ConvLayer2d(opts, in_channels=hidden_dim, out_channels=hidden_dim, stride=stride, kernel_size=3,
                                                 groups=hidden_dim, use_act=True, use_norm=True, dilation=dilation))
        block.add_module("red_1x1", ConvLayer2d(opts, in_channels=hidden_dim, out_channels=out_channels, kernel_size=1,
                                                use_act=False, use_norm=True))
        self.block = block
        self.in_channels, self.out_channels, self.exp, self.dilation, self.stride = in_channels, out_channels, expand_ratio, dilation, stride
        self.hidden_dim = hidden_dim
        self.use_res_connect = self.stride == 1 and in_channels == out_channels and skip_connection
        self._cfg = None

    def _build_cfg(self):
        if self.exp == 1:
            raise NotImplementedError("InvertedResidual with expand_ratio == 1 (no exp_1x1) is not on the MobileViT hot path")
        if self.dilation != 1 and self.stride != 1:
            raise NotImplementedError("a dilated depthwise conv must have stride 1 (the reference dilates instead of striding, mobilevit_v2.py:183-186)")
        if self.in_channels % 8 or self.out_channels % 8 or self.hidden_dim % 8:
            raise NotImplementedError("channel counts must be multiples of 8 (16-byte channel vectors)")
        b = self.block
        prep = PW()
        cfg = SimpleNamespace(prep=prep, hid=self.hidden_dim, cout=self.out_channels, stride=self.stride, residual=self.use_res_connect,
                              dilation=int(self.dilation))
        cfg.i_w1 = prep.add(b.exp_1x1.block.conv.weight, PW.KIND_ROWMAJOR)
        cfg.i_w1t = prep.add(b.exp_1x1.block.conv.weight, PW.KIND_TRANSPOSED)
        cfg.i_wd = prep.add(b.conv_3x3.block.conv.weight, PW.KIND_TAPMAJOR_F32)
        cfg.i_w3 = prep.add(b.red_1x1.block.conv.weight, PW.KIND_ROWMAJOR)
        cfg.i_w3t = prep.add(b.red_1x1.block.conv.weight, PW.KIND_TRANSPOSED)
        self._cfg = cfg

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        _need_cuda(x, "InvertedResidual")
        if self._cfg is None:
            self._build_cfg()
        cfg, b = self._cfg, self.block
        cfg.bn = [Fn.bn_cfg(b.exp_1x1.block.norm), Fn.bn_cfg(b.conv_3x3.block.norm), Fn.bn_cfg(b.red_1x1.block.norm)]
        cfg.lazy_in, cfg.lazy_out = _lazy_in(x), _lazy_out(self) and not self.use_res_connect
        _bind(self, cfg, [b.exp_1x1.block.conv.weight, b.exp_1x1.block.norm.weight, b.exp_1x1.block.norm.bias,
                          b.conv_3x3.block.conv.weight, b.conv_3x3.block.norm.weight, b.conv_3x3.block.norm.bias,
                          b.red_1x1.block.conv.weight, b.red_1x1.block.norm.weight, b.red_1x1.block.norm.bias])
        return _tag(Fn.InvertedResidualFn.apply(Fn.to_bf16_cl(x), cfg, *cfg.plist), cfg)

    def __repr__(self) -> str:
        return "{}(in_channels={}, out_channels={}, stride={}, exp={}, dilation={}, skip_conn={})".format(
            self.__class__.__name__, self.in_channels, self.out_channels, self.stride, self.exp, self.dilation, self.use_res_connect)


# ------------------------------------------------------------------------------- SqueezeExcitation / InvertedResidualSE
class SqueezeExcitation(BaseModule):
    """cvnets/modules/squeeze_excitation.py:16-91: ``x * scale_act(fc2(act(fc1(avg_pool(x)))))`` with the reference child tree
    ``se_layer.{global_pool, fc1, fc2, scale_act}`` (fc1 / fc2 are 1x1 ConvLayer2d with bias; fc1's activation is the model-wide
    ``model.activation.name``).  Pool, the two GEMMs, the activations and the channel scaling (cvb_se_scale_*) are library kernels."""

    def __init__(self, opts, in_channels: int, squeeze_factor: Optional[int] = 4, squeeze_channels: Optional[int] = None,
                 scale_fn_name: Optional[str] = "sigmoid", *args, **kwargs) -> None:
        if squeeze_channels is None:
            squeeze_channels = max(make_divisible(in_channels // squeeze_factor, 8), 32)
        super().__init__()
        self.se_layer = nn.Sequential()
        self.se_layer.add_module("global_pool", AdaptiveAvgPool2d(output_size=1))
        self.se_layer.add_module("fc1", ConvLayer2d(opts=opts, in_channels=in_channels, out_channels=squeeze_channels, kernel_size=1, stride=1, bias=True,
                                                    use_norm=False, use_act=True))
        self.se_layer.add_module("fc2", ConvLayer2d(opts=opts, in_channels=squeeze_channels, out_channels=in_channels, kernel_size=1, stride=1, bias=True,
                                                    use_norm=False, use_act=False))
        self.se_layer.add_module("scale_act", build_activation_layer(opts, act_type=scale_fn_name, inplace=True))
        self.in_channels, self.squeeze_factor, self.scale_fn = in_channels, squeeze_factor, scale_fn_name

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        _need_cuda(x, "SqueezeExcitation")
        x = Fn.to_bf16_cl(x)
        return Fn.SeScaleFn.apply(x, self.se_layer(x))

    def __repr__(self) -> str:
        return "{}(in_channels={}, squeeze_factor={}, scale_fn={})".format(self.__class__.__name__, self.in_channels, self.squeeze_factor, self.scale_fn)


class InvertedResidualSE(BaseModule):
    """cvnets/modules/mobilenetv2.py:16-138 (MobileNetv3-style block; SURVEY.md 8f row 4): exp_1x1 (1x1 + BN) -> act -> conv_3x3 (depthwise + BN)
    -> act -> [SqueezeExcitation] -> red_1x1 (1x1 + BN), residual iff stride 1 and Cin == Cout.  Same constructor, child tree and state_dict
    keys (``block.{exp_1x1, act_fn_1, conv_3x3, act_fn_2, se, red_1x1}``; the two act children are ONE module object, as in the reference).
    Composition of the stand-alone layer kernels; the residual add rides the red_1x1 BatchNorm-apply pass.  Depthwise kernel size 3 or 5."""

    def __init__(self, opts, in_channels: int, out_channels: int, expand_ratio: Union[int, float], dilation: Optional[int] = 1,
                 stride: Optional[int] = 1, use_se: Optional[bool] = False, act_fn_name: Optional[str] = "relu",
                 se_scale_fn_name: Optional[str] = "hard_sigmoid", kernel_size: Optional[int] = 3, squeeze_factor: Optional[int] = 4,
                 *args, **kwargs) -> None:
        hidden_dim = make_divisible(int(round(in_channels * expand_ratio)), 8)
        act_fn = build_activation_layer(opts, act_type=act_fn_name, inplace=True)
        super().__init__()
        block = nn.Sequential()
        if expand_ratio != 1:
            block.add_module("exp_1x1", ConvLayer2d(opts, in_channels=in_channels, out_channels=hidden_dim, kernel_size=1, use_act=False, use_norm=True))
            block.add_module("act_fn_1", act_fn)
        block.add_module("conv_3x3", ConvLayer2d(opts, in_channels=hidden_dim, out_channels=hidden_dim, stride=stride, kernel_size=kernel_size,
                                                 groups=hidden_dim, use_act=False, use_norm=True, dilation=dilation))
        block.add_module("act_fn_2", act_fn)
        if use_se:
            block.add_module("se", SqueezeExcitation(opts=opts, in_channels=hidden_dim, squeeze_factor=squeeze_factor, scale_fn_name=se_scale_fn_name))
        block.add_module("red_1x1", ConvLayer2d(opts, in_channels=hidden_dim, out_channels=out_channels, kernel_size=1, use_act=False, use_norm=True))
        self.block = block
        self.in_channels, self.out_channels, self.exp, self.dilation = in_channels, out_channels, expand_ratio, dilation
        self.use_se, self.stride, self.act_fn_name, self.kernel_size = use_se, stride, act_fn_name, kernel_size
        self.use_res_connect = self.stride == 1 and in_channels == out_channels

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        _need_cuda(x, "InvertedResidualSE")
        x = Fn.to_bf16_cl(x)
        y = x
        for name, m in self.block._modules.items():  # (named_children() would de-duplicate the shared activation module)
            if name == "red_1x1" and self.use_res_connect:
                y = m(y, residual=x)  # x + block(x): the residual is added in red_1x1's BatchNorm-apply pass
            else:
                y = m(y)
        return y

    def __repr__(self) -> str:
        return "{}(in_channels={}, out_channels={}, stride={}, exp={}, dilation={}, use_se={}, kernel_size={}, act_fn={})".format(
            self.__class__.__name__, self.in_channels, self.out_channels, self.stride, self.exp, self.dilation, self.use_se, self.kernel_size,
            self.act_fn_name)


class EfficientNetBlock(InvertedResidualSE):
    """cvnets/modules/efficientnet.py: InvertedResidualSE plus a row-mode ``stochastic_depth`` child (torchvision.ops.StochasticDepth) on the
    block output before the residual add.  Same constructor (``stochastic_depth_prob`` first) and state_dict.  In training with p > 0 the
    residual add and the per-sample mask run as one pass of the hashed-mask kernel (cvb_dropout_fwd with p_row = p, one sample = Ho*Wo rows)
    keyed from the device generator, so a captured step draws fresh masks on every replay; otherwise (eval, p = 0) the add rides red_1x1's
    BatchNorm-apply pass as in InvertedResidualSE."""

    def __init__(self, stochastic_depth_prob: float, *args, **kwargs) -> None:
        super().__init__(*args, **kwargs)
        self.stochastic_depth = StochasticDepth(p=stochastic_depth_prob, mode="row")

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        p = float(self.stochastic_depth.p)
        if not (self.use_res_connect and self.training and p > 0.0):
            return super().forward(x)
        _need_cuda(x, "EfficientNetBlock")
        x = Fn.to_bf16_cl(x)
        y = x
        for m in self.block._modules.values():
            y = m(y)
        return Fn.StochasticDepthAddFn.apply(y, x, p)

    def __repr__(self) -> str:
        return super().__repr__()[:-1] + f", stochastic_depth_prob={self.stochastic_depth.p})"


# -------------------------------------------------------------------------------------------------------- LinearAttnFFN
class LinearAttnFFN(BaseModule):
    """Parameter container with the reference tree (pre_norm_attn.{0,1,2}, pre_norm_ffn.{0,1,2,3,4}); executed inside
    MobileViTBlockv2Fn."""

    def __init__(self, opts, embed_dim: int, ffn_latent_dim: int, attn_dropout: Optional[float] = 0.0, dropout: Optional[float] = 0.1,
                 ffn_dropout: Optional[float] = 0.0, norm_layer: Optional[str] = "layer_norm_2d", *args, **kwargs) -> None:
        super().__init__()
        attn_unit = LinearSelfAttention(opts, embed_dim=embed_dim, attn_dropout=attn_dropout, bias=True)
        self.pre_norm_attn = nn.Sequential(
            get_normalization_layer(opts=opts, norm_type=norm_layer, num_features=embed_dim), attn_unit, Dropout(p=dropout))
        self.pre_norm_ffn = nn.Sequential(
            get_normalization_layer(opts=opts, norm_type=norm_layer, num_features=embed_dim),
            ConvLayer2d(opts=opts, in_channels=embed_dim, out_channels=ffn_latent_dim, kernel_size=1, stride=1, bias=True,
                        use_norm=False, use_act=True),
            Dropout(p=ffn_dropout),
            ConvLayer2d(opts=opts, in_channels=ffn_latent_dim, out_channels=embed_dim, kernel_size=1, stride=1, bias=True,
                        use_norm=False, use_act=False),
            Dropout(p=dropout))
        self.embed_dim, self.ffn_dim, self.ffn_dropout, self.std_dropout = embed_dim, ffn_latent_dim, ffn_dropout, dropout
        self.attn_fn_name, self.norm_name = attn_unit.__repr__(), norm_layer
        self.attn_dropout_p = attn_dropout

    def forward(self, x: Tensor, x_prev: Optional[Tensor] = None, *args, **kwargs) -> Tensor:
        """Stand-alone use on the unfolded tensor [B, d, P, N] (transformer.py:248-264), self- or cross-attention: the layers' own
        kernel paths composed, residual additions inside the out_proj / second FFN conv epilogues.  Inside MobileViTBlockv2 the unit runs
        in the block's fused function instead."""
        _need_cuda(x, "LinearAttnFFN")
        if self.std_dropout or self.ffn_dropout or self.attn_dropout_p:
            raise NotImplementedError("dropout > 0 is not implemented")
        norm1, attn = self.pre_norm_attn[0], self.pre_norm_attn[1]
        x = attn(norm1(x), x_prev, residual=x)      # x + LSA(GN(x)[, x_prev])   (:253 / :254-260)
        norm2, conv1, conv2 = self.pre_norm_ffn[0], self.pre_norm_ffn[1], self.pre_norm_ffn[3]
        return conv2(conv1(norm2(x)), residual=x)   # x + conv(act(conv(GN(x))))  (:263)

    def __repr__(self) -> str:
        return "{}(embed_dim={}, ffn_dim={}, dropout={}, ffn_dropout={}, attn_fn={}, norm_layer={})".format(
            self.__class__.__name__, self.embed_dim, self.ffn_dim, self.std_dropout, self.ffn_dropout, self.attn_fn_name, self.norm_name)


# ----------------------------------------------------------------------------------------------------- MobileViTBlockv2
class MobileViTBlockv2(BaseModule):
    def __init__(self, opts, in_channels: int, attn_unit_dim: int,
                 ffn_multiplier: Optional[Union[Sequence[Union[int, float]], int, float]] = 2.0, n_attn_blocks: Optional[int] = 2,
                 attn_dropout: Optional[float] = 0.0, dropout: Optional[float] = 0.0, ffn_dropout: Optional[float] = 0.0,
                 patch_h: Optional[int] = 8, patch_w: Optional[int] = 8, conv_ksize: Optional[int] = 3, dilation: Optional[int] = 1,
                 attn_norm_layer: Optional[str] = "layer_norm_2d", *args, **kwargs) -> None:
        cnn_out_dim = attn_unit_dim
        conv_3x3_in = ConvLayer2d(opts=opts, in_channels=in_channels, out_channels=in_channels, kernel_size=conv_ksize, stride=1,
                                  use_norm=True, use_act=True, dilation=dilation, groups=in_channels)
        conv_1x1_in = ConvLayer2d(opts=opts, in_channels=in_channels, out_channels=cnn_out_dim, kernel_size=1, stride=1,
                                  use_norm=False, use_act=False)
        super().__init__()
        self.local_rep = nn.Sequential(conv_3x3_in, conv_1x1_in)
        self.global_rep, attn_unit_dim = self._build_attn_layer(opts=opts, d_model=attn_unit_dim, ffn_mult=ffn_multiplier,
                                                               n_layers=n_attn_blocks, attn_dropout=attn_dropout, dropout=dropout,
                                                               ffn_dropout=ffn_dropout, attn_norm_layer=attn_norm_layer)
        self.conv_proj = ConvLayer2d(opts=opts, in_channels=cnn_out_dim, out_channels=in_channels, kernel_size=1, stride=1,
                                     use_norm=True, use_act=False)
        self.patch_h, self.patch_w, self.patch_area = patch_h, patch_w, patch_w * patch_h
        self.cnn_in_dim, self.cnn_out_dim, self.transformer_in_dim = in_channels, cnn_out_dim, attn_unit_dim
        self.dropout, self.attn_dropout, self.ffn_dropout = dropout, attn_dropout, ffn_dropout
        self.n_blocks, self.conv_ksize, self.dilation = n_attn_blocks, conv_ksize, dilation
        self.attn_norm_layer = attn_norm_layer
        self._cfg = None

    def _build_attn_layer(self, opts, d_model: int, ffn_mult, n_layers: int, attn_dropout: float, dropout: float, ffn_dropout: float,
                          attn_norm_layer: str, *args, **kwargs) -> Tuple[nn.Module, int]:
        if isinstance(ffn_mult, Sequence) and len(ffn_mult) == 2:
            ffn_dims = np.linspace(ffn_mult[0], ffn_mult[1], n_layers, dtype=float) * d_model
        elif isinstance(ffn_mult, Sequence) and len(ffn_mult) == 1:
            ffn_dims = [ffn_mult[0] * d_model] * n_layers
        elif isinstance(ffn_mult, (int, float)):
            ffn_dims = [ffn_mult * d_model] * n_layers
        else:
            raise NotImplementedError
        ffn_dims = [int((d // 16) * 16) for d in ffn_dims]
        global_rep = [LinearAttnFFN(opts=opts, embed_dim=d_model, ffn_latent_dim=ffn_dims[i], attn_dropout=attn_dropout, dropout=dropout,
                                    ffn_dropout=ffn_dropout, norm_layer=attn_norm_layer) for i in range(n_layers)]
        global_rep.append(get_normalization_layer(opts=opts, norm_type=attn_norm_layer, num_features=d_model))
        return nn.Sequential(*global_rep), d_model

    def _build_cfg(self):
        C, d = self.cnn_in_dim, self.cnn_out_dim
        if self.patch_h != 2 or self.patch_w != 2:
            raise NotImplementedError("only 2x2 patches (every MobileViTv2 config) are implemented")
        if self.conv_ksize != 3:
            raise NotImplementedError("local_rep must be a 3x3 depthwise conv")
        if self.attn_norm_layer not in ("layer_norm_2d", "layer_norm_nchw"):
            raise NotImplementedError("attn_norm_layer must be layer_norm_2d")
        if self.dropout or self.attn_dropout or self.ffn_dropout:
            raise NotImplementedError("dropout > 0 is not implemented (the MobileViTv2 recipes use 0)")
        ffns = {blk.ffn_dim for blk in list(self.global_rep)[:-1]}
        if len(ffns) != 1:
            raise NotImplementedError("per-block FFN widths must be equal")
        if C % 8 or d % 8:
            raise NotImplementedError("channel counts must be multiples of 8")
        prep = PW()
        cfg = SimpleNamespace(prep=prep, d=d, ffn=ffns.pop(), n_blocks=self.n_blocks, gn_eps=float(self.global_rep[-1].eps), dilation=int(self.dilation))
        cfg.i_wd0 = prep.add(self.local_rep[0].block.conv.weight, PW.KIND_TAPMAJOR_F32)
        cfg.i_wl = prep.add(self.local_rep[1].block.conv.weight, PW.KIND_ROWMAJOR)
        cfg.i_wlt = prep.add(self.local_rep[1].block.conv.weight, PW.KIND_TRANSPOSED)
        cfg.i_blk = []
        for i in range(self.n_blocks):
            blk = self.global_rep[i]
            attn = blk.pre_norm_attn[1]
            ix = SimpleNamespace()
            # qkv: reference row order [q, K(d), V(d)] -> kernel order [K, V, q, pad(7)]  (rot = 1)
            ix.wqkv = prep.add(attn.qkv_proj.block.conv.weight, PW.KIND_ROWMAJOR, rot=1, dst_rows=2 * d + 8)
            ix.wqkvt = prep.add(attn.qkv_proj.block.conv.weight, PW.KIND_TRANSPOSED, rot=1, ldd=2 * d + 8)
            ix.bqkv = prep.add(attn.qkv_proj.block.conv.bias, PW.KIND_VECTOR_F32, rot=1, dst_rows=2 * d + 8)
            ix.wo = prep.add(attn.out_proj.block.conv.weight, PW.KIND_ROWMAJOR)
            ix.wot = prep.add(attn.out_proj.block.conv.weight, PW.KIND_TRANSPOSED)
            ix.w1 = prep.add(blk.pre_norm_ffn[1].block.conv.weight, PW.KIND_ROWMAJOR)
            ix.w1t = prep.add(blk.pre_norm_ffn[1].block.conv.weight, PW.KIND_TRANSPOSED)
            ix.w2 = prep.add(blk.pre_norm_ffn[3].block.conv.weight, PW.KIND_ROWMAJOR)
            ix.w2t = prep.add(blk.pre_norm_ffn[3].block.conv.weight, PW.KIND_TRANSPOSED)
            cfg.i_blk.append(ix)
        cfg.i_wp = prep.add(self.conv_proj.block.conv.weight, PW.KIND_ROWMAJOR)
        cfg.i_wpt = prep.add(self.conv_proj.block.conv.weight, PW.KIND_TRANSPOSED)
        self._cfg = cfg

    def _params(self):
        lr = self.local_rep
        out = [lr[0].block.conv.weight, lr[0].block.norm.weight, lr[0].block.norm.bias, lr[1].block.conv.weight]
        for i in range(self.n_blocks):
            blk = self.global_rep[i]
            attn = blk.pre_norm_attn[1]
            out += [blk.pre_norm_attn[0].weight, blk.pre_norm_attn[0].bias,
                    attn.qkv_proj.block.conv.weight, attn.qkv_proj.block.conv.bias,
                    attn.out_proj.block.conv.weight, attn.out_proj.block.conv.bias,
                    blk.pre_norm_ffn[0].weight, blk.pre_norm_ffn[0].bias,
                    blk.pre_norm_ffn[1].block.conv.weight, blk.pre_norm_ffn[1].block.conv.bias,
                    blk.pre_norm_ffn[3].block.conv.weight, blk.pre_norm_ffn[3].block.conv.bias]
        gl = self.global_rep[self.n_blocks]
        out += [gl.weight, gl.bias, self.conv_proj.block.conv.weight, self.conv_proj.block.norm.weight, self.conv_proj.block.norm.bias]
        return out

    def forward_spatial(self, x: Tensor, *args, **kwargs) -> Tensor:
        _need_cuda(x, "MobileViTBlockv2")
        if x.shape[2] % self.patch_h or x.shape[3] % self.patch_w:
            raise NotImplementedError("H, W must be multiples of the patch size (the bilinear resize_input_if_needed path, "
                                      "mobilevit_block.py:595-603, never fires at 256x256 and is out of scope)")
        if self._cfg is None:
            self._build_cfg()
        cfg = self._cfg
        cfg.bn = [Fn.bn_cfg(self.local_rep[0].block.norm), Fn.bn_cfg(self.conv_proj.block.norm)]
        cfg.lazy_in, cfg.lazy_out = _lazy_in(x), _lazy_out(self)
        _bind(self, cfg, self._params())
        return _tag(Fn.MobileViTBlockv2Fn.apply(Fn.to_bf16_cl(x), cfg, *cfg.plist), cfg)

    def forward(self, x: Union[Tensor, Tuple[Tensor]], *args, **kwargs) -> Union[Tensor, Tuple[Tensor, Tensor]]:
        if isinstance(x, Tuple) and len(x) == 2:
            raise NotImplementedError("forward_temporal (video cross-attention, mobilevit_block.py:628-655) is out of scope")
        elif isinstance(x, Tensor):
            return self.forward_spatial(x)
        else:
            raise NotImplementedError


# ------------------------------------------------------------------------------------------------------- MobileViTBlock (v1)
class MobileViTBlock(BaseModule):
    """cvnets/modules/mobilevit_block.py:19-326 (SURVEY.md 8a row a9): dense 3x3 conv + 1x1 -> unfold to [B*P, N, d] tokens -> n x
    TransformerEncoder -> LayerNorm -> fold -> 1x1 conv -> cat(input, .) -> dense 3x3 fusion conv.  Same constructor, child tree
    (``local_rep.{conv_3x3,conv_1x1}``, ``global_rep.{i}``, ``conv_proj``, ``fusion``) and ``state_dict`` keys as the reference.

    Composition of the library's own layer functions (the block is <= 0.4 GMAC at XXS scale and not on the throughput metric): dense convs
    via im2col + GEMM, unfold / fold as one row-permutation kernel each, the encoders on the fused TransformerEncoderFn."""

    def __init__(self, opts, in_channels: int, transformer_dim: int, ffn_dim: int, n_transformer_blocks: Optional[int] = 2,
                 head_dim: Optional[int] = 32, attn_dropout: Optional[float] = 0.0, dropout: Optional[float] = 0.0, ffn_dropout: Optional[float] = 0.0,
                 patch_h: Optional[int] = 8, patch_w: Optional[int] = 8, transformer_norm_layer: Optional[str] = "layer_norm",
                 conv_ksize: Optional[int] = 3, dilation: Optional[int] = 1, no_fusion: Optional[bool] = False, *args, **kwargs) -> None:
        conv_3x3_in = ConvLayer2d(opts=opts, in_channels=in_channels, out_channels=in_channels, kernel_size=conv_ksize, stride=1, use_norm=True,
                                  use_act=True, dilation=dilation)
        conv_1x1_in = ConvLayer2d(opts=opts, in_channels=in_channels, out_channels=transformer_dim, kernel_size=1, stride=1, use_norm=False,
                                  use_act=False)
        conv_1x1_out = ConvLayer2d(opts=opts, in_channels=transformer_dim, out_channels=in_channels, kernel_size=1, stride=1, use_norm=True,
                                   use_act=True)
        conv_3x3_out = None
        if not no_fusion:
            conv_3x3_out = ConvLayer2d(opts=opts, in_channels=2 * in_channels, out_channels=in_channels, kernel_size=conv_ksize, stride=1,
                                       use_norm=True, use_act=True)
        super().__init__()
        self.local_rep = nn.Sequential()
        self.local_rep.add_module(name="conv_3x3", module=conv_3x3_in)
        self.local_rep.add_module(name="conv_1x1", module=conv_1x1_in)
        assert transformer_dim % head_dim == 0
        num_heads = transformer_dim // head_dim
        global_rep = [TransformerEncoder(opts=opts, embed_dim=transformer_dim, ffn_latent_dim=ffn_dim, num_heads=num_heads, attn_dropout=attn_dropout,
                                         dropout=dropout, ffn_dropout=ffn_dropout, transformer_norm_layer=transformer_norm_layer)
                      for _ in range(n_transformer_blocks)]
        global_rep.append(get_normalization_layer(opts=opts, norm_type=transformer_norm_layer, num_features=transformer_dim))
        self.global_rep = nn.Sequential(*global_rep)
        self.conv_proj = conv_1x1_out
        self.fusion = conv_3x3_out
        self.patch_h, self.patch_w, self.patch_area = patch_h, patch_w, patch_w * patch_h
        self.cnn_in_dim, self.cnn_out_dim, self.n_heads, self.ffn_dim = in_channels, transformer_dim, num_heads, ffn_dim
        self.dropout, self.attn_dropout, self.ffn_dropout = dropout, attn_dropout, ffn_dropout
        self.dilation, self.n_blocks, self.conv_ksize = dilation, n_transformer_blocks, conv_ksize

    def forward_spatial(self, x: Tensor) -> Tensor:
        _need_cuda(x, "MobileViTBlock")
        res = Fn.to_bf16_cl(x)
        fm = self.local_rep(res)
        B, _, H, W = fm.shape
        patches = Fn.UnfoldFn.apply(fm, self.patch_h, self.patch_w)           # [B*P, N, d]
        for layer in self.global_rep:
            patches = layer(patches)
        fm = Fn.FoldFn.apply(patches, B, H, W, self.patch_h, self.patch_w)
        fm = self.conv_proj(fm)
        if self.fusion is not None:
            fm = self.fusion(Fn.Concat2Fn.apply(res, fm))
        return fm

    def forward(self, x: Union[Tensor, Tuple[Tensor]], *args, **kwargs) -> Union[Tensor, Tuple[Tensor, Tensor]]:
        if isinstance(x, Tuple) and len(x) == 2:
            raise NotImplementedError("forward_temporal (video cross-attention, mobilevit_block.py:290-311) is out of scope")
        elif isinstance(x, Tensor):
            return self.forward_spatial(x)
        else:
            raise NotImplementedError


class TransformerEncoder(BaseModule):
    """cvnets/modules/transformer.py:26-156: pre-norm encoder, ``x = x + MHA(LN(x)); x = x + FFN(LN(x))``.

    Same constructor, child tree (``pre_norm_mha = [norm, MultiHeadAttention, Dropout]``, ``pre_norm_ffn = [norm, LinearLayer,
    act, Dropout, LinearLayer, Dropout]``) and ``state_dict`` keys as the reference; the forward is one fused autograd function
    (LayerNorm as a GEMM load mode, attention core in shared memory, residuals in the GEMM epilogues).  Not implemented (raises):
    ``num_heads == 1`` (SingleHeadAttention), dropout / stochastic depth > 0, cross-attention (``x_prev``), norms other than
    ``layer_norm``, activations other than swish / gelu."""

    def __init__(self, opts, embed_dim: int, ffn_latent_dim: int, num_heads: Optional[int] = 8, attn_dropout: Optional[float] = 0.0,
                 dropout: Optional[float] = 0.0, ffn_dropout: Optional[float] = 0.0, transformer_norm_layer: Optional[str] = "layer_norm",
                 stochastic_dropout: Optional[float] = 0.0, *args, **kwargs) -> None:
        super().__init__()
        if num_heads <= 1:
            raise NotImplementedError("SingleHeadAttention (num_heads == 1) is not on the GPU path")
        attn_unit = MultiHeadAttention(embed_dim, num_heads, attn_dropout=attn_dropout, bias=True)
        self.pre_norm_mha = nn.Sequential(get_normalization_layer(opts=opts, norm_type=transformer_norm_layer, num_features=embed_dim),
                                          attn_unit, Dropout(p=dropout))
        act_name = build_activation_layer(opts, num_parameters=1)
        self.pre_norm_ffn = nn.Sequential(get_normalization_layer(opts=opts, norm_type=transformer_norm_layer, num_features=embed_dim),
                                          LinearLayer(in_features=embed_dim, out_features=ffn_latent_dim, bias=True), act_name,
                                          Dropout(p=ffn_dropout),
                                          LinearLayer(in_features=ffn_latent_dim, out_features=embed_dim, bias=True), Dropout(p=dropout))
        self.drop_path = Identity()
        if stochastic_dropout > 0.0:
            if dropout > 0.0:
                raise ValueError("Stochastic dropout and dropout are mutually exclusive. Use either of them, but not both. "
                                 "Got: {} and {}".format(stochastic_dropout, dropout))  # transformer.py:98-104 (logger.error -> exit)
            self.drop_path = StochasticDepth(p=stochastic_dropout, mode="row")
        self.embed_dim, self.ffn_dim, self.ffn_dropout = embed_dim, ffn_latent_dim, ffn_dropout
        self.stochastic_dropout, self.std_dropout = stochastic_dropout, dropout
        self.attn_fn_name, self.act_fn_name, self.norm_type = attn_unit.__class__.__name__, act_name.__class__.__name__, transformer_norm_layer
        self._cfg = None

    def __repr__(self) -> str:
        return "{}(embed_dim={}, ffn_dim={}, dropout={}, ffn_dropout={}, stochastic_dropout={}, attn_fn={}, act_fn={}, norm_fn={})".format(
            self.__class__.__name__, self.embed_dim, self.ffn_dim, self.std_dropout, self.ffn_dropout, self.stochastic_dropout,
            self.attn_fn_name, self.act_fn_name, self.norm_type)

    def _build_cfg(self):
        from . import ops
        if self.norm_type not in ("layer_norm", "layer_norm_fp32"):
            raise NotImplementedError("transformer_norm_layer must be layer_norm or layer_norm_fp32")
        if self.embed_dim % 8 or self.ffn_dim % 8:
            raise NotImplementedError("embed_dim / ffn_latent_dim must be multiples of 8")
        prep = PW()
        cfg = self.pre_norm_mha[1].build_cfg(prep)
        cfg.prep, cfg.ffn, cfg.eps = prep, self.ffn_dim, float(self.pre_norm_mha[0].eps)
        cfg.act = ops.ACT_SILU if self.act_fn_name == "Swish" else ops.ACT_GELU
        cfg.i_w1 = prep.add(self.pre_norm_ffn[1].weight, PW.KIND_ROWMAJOR)
        cfg.i_w1t = prep.add(self.pre_norm_ffn[1].weight, PW.KIND_TRANSPOSED)
        cfg.i_w2 = prep.add(self.pre_norm_ffn[4].weight, PW.KIND_ROWMAJOR)
        cfg.i_w2t = prep.add(self.pre_norm_ffn[4].weight, PW.KIND_TRANSPOSED)
        self._cfg = cfg

    def forward(self, x: Tensor, x_prev: Optional[Tensor] = None, key_padding_mask: Optional[Tensor] = None,
                attn_mask: Optional[Tensor] = None, *args, **kwargs) -> Tensor:
        _need_cuda(x, "TransformerEncoder")
        if x_prev is not None:
            raise NotImplementedError("cross-attention (x_prev) is not implemented on the GPU path")
        if self.training and self.pre_norm_mha[1].attn_dropout.p:
            raise NotImplementedError("attention-probability dropout > 0 in training mode is not implemented (every recipe of the reference sets 0; "
                                      "it is the identity in eval mode, which works)")
        if x.dim() != 3:
            raise NotImplementedError("TransformerEncoder expects [N, S, C]")
        hd = self.pre_norm_mha[1].head_dim
        if x.shape[1] > 256 and hd != 64:
            raise NotImplementedError(f"TransformerEncoder: S = {x.shape[1]} > 256 needs head_dim 64 (the streaming attention kernels); "
                                      f"head_dim {hd} keeps a head in shared memory and supports S <= 256")
        if x.shape[1] == x.shape[2]:
            raise NotImplementedError("S == C: the reference's LayerNorm would take its channel-first branch (layer_norm.py:52-65)")
        if self._cfg is None:
            self._build_cfg()
        cfg = self._cfg
        cfg.masks = (attn_mask, key_padding_mask)
        # training-mode dropout after the attention / FFN branches, FFN-hidden dropout and stochastic depth (transformer.py:77-100, 139-156): hashed
        # masks folded into the residual adds (functional.TransformerEncoderFn); all three are the identity in eval mode
        p, pf, pr = float(self.pre_norm_mha[2].p), float(self.pre_norm_ffn[3].p), float(self.stochastic_dropout)
        cfg.drop = (p, pf, pr) if (self.training and (p > 0 or pf > 0 or pr > 0)) else None
        cfg.eps = float(self.pre_norm_mha[0].eps)  # VisionTransformer.update_layer_norm_eps rewrites it after construction (vit.py:204-208)
        n1, mha, n2 = self.pre_norm_mha[0], self.pre_norm_mha[1], self.pre_norm_ffn[0]
        l1, l2 = self.pre_norm_ffn[1], self.pre_norm_ffn[4]
        _bind(self, cfg, [n1.weight, n1.bias, mha.qkv_proj.weight, mha.qkv_proj.bias, mha.out_proj.weight, mha.out_proj.bias, n2.weight, n2.bias,
                          l1.weight, l1.bias, l2.weight, l2.bias])
        return Fn.TransformerEncoderFn.apply(x.to(torch.bfloat16).contiguous(), cfg, *cfg.plist)

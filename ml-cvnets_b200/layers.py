"""Host-side mirror of ``cvnets.layers`` for the hot path: SAME class names, constructor signatures, child-module tree
and ``state_dict`` keys as the reference (SURVEY.md 8b / Appendix B), so published checkpoints load unchanged and the
reference's isinstance/name based machinery (weight init, BN momentum annealing, weight-decay grouping, EMA deepcopy)
keeps working.  Parameters are ordinary ``nn.Parameter``s inside ordinary ``nn.Conv2d`` / ``nn.BatchNorm2d`` /
``nn.GroupNorm`` / ``nn.Linear`` children; only ``forward`` is ours and it runs hand-written sm_90a kernels.

There is deliberately NO PyTorch fallback.  Inside InvertedResidual / MobileViTBlockv2 / TransformerEncoder the layers are parameter
containers executed by the fused autograd functions; used on their own they run the stand-alone functions of functional.py (same
kernels, one layer per function).  What has no kernel path (dilated dense convs, dropout p > 0 in training) raises.
"""
from __future__ import annotations

import argparse
from typing import Optional, Tuple, Union

import torch
from torch import Tensor, nn


def _opt(opts, name: str, default):
    return getattr(opts, name, default) if opts is not None else default


class BaseLayer(nn.Module):
    """cvnets/layers/base_layer.py:14-63."""

    def __init__(self, *args, **kwargs) -> None:
        super().__init__()

    @classmethod
    def add_arguments(cls, parser: argparse.ArgumentParser):
        return parser


class Identity(BaseLayer):
    """cvnets/layers/identity.py."""

    def forward(self, x: Tensor) -> Tensor:
        return x


class Dropout(nn.Dropout):
    """cvnets/layers/dropout.py: nn.Dropout.  Training mode with p > 0 on a CUDA tensor runs the library's hashed-mask kernel (cvb_dropout_fwd);
    eval mode / p == 0 is the identity.  Inside TransformerEncoder the module is only a parameter-free marker: its p is folded into the
    block's residual adds."""

    def __init__(self, p: Optional[float] = 0.5, inplace: Optional[bool] = False, *args, **kwargs) -> None:
        super().__init__(p=p, inplace=inplace)

    def forward(self, x: Tensor) -> Tensor:
        if not self.training or self.p == 0.0:
            return x
        from . import functional as Fn
        _need_cuda(x, "Dropout")
        if self.p >= 1.0:
            raise NotImplementedError("Dropout: 0 <= p < 1")
        if x.dim() == 4:  # [B, C, H, W] maps live channels-last: the kernel sees the [B*H*W, C] matrix
            xc = Fn.to_bf16_cl(x)
            B, C, H, W = xc.shape
            if C % 8:
                raise NotImplementedError("Dropout: channel count must be a multiple of 8")
            return Fn.to_4d(Fn.DropoutFn.apply(Fn.as_2d(xc), float(self.p)), B, H, W)
        if x.shape[-1] % 8:
            raise NotImplementedError("Dropout: the last dimension must be a multiple of 8 (16-byte channel vectors)")
        return Fn.DropoutFn.apply(x, float(self.p))


class StochasticDepth(nn.Module):
    """cvnets/layers/stochastic_depth.py == torchvision.ops.StochasticDepth: parameter-free marker child ``drop_path`` of TransformerEncoder; its
    per-sample mask is folded into the block's residual adds (cvb_dropout_fwd, p_row)."""

    def __init__(self, p: float, mode: str) -> None:
        super().__init__()
        if mode != "row":
            raise NotImplementedError("StochasticDepth: mode='row' is what the reference uses (transformer.py:105)")
        self.p, self.mode = p, mode

    def forward(self, x: Tensor) -> Tensor:
        raise NotImplementedError("StochasticDepth runs fused inside TransformerEncoder")

    def __repr__(self) -> str:
        return "{}(p={}, mode={})".format(self.__class__.__name__, self.p, self.mode)


class Swish(nn.SiLU):
    """cvnets/layers/activation/swish.py:13-20."""

    def __init__(self, inplace: Optional[bool] = False, *args, **kwargs) -> None:
        super().__init__(inplace=inplace)

    def forward(self, x: Tensor) -> Tensor:
        """Stand-alone use on a CUDA tensor (the activations of InvertedResidualSE / EfficientNetBlock) is one pass of cvb_act_fwd (bf16 out);
        inside the fused blocks the module is only a marker."""
        if not x.is_cuda:
            return super().forward(x)
        from . import functional as Fn
        from . import ops
        return Fn.ActFn.apply(Fn.to_bf16_cl(x) if x.dim() == 4 else x.to(torch.bfloat16).contiguous(), ops.ACT_SILU)


class BatchNorm2d(nn.BatchNorm2d):
    """cvnets/layers/normalization/batch_norm.py:14-49."""

    def __init__(self, num_features: int, eps: Optional[float] = 1e-5, momentum: Optional[float] = 0.1,
                 affine: Optional[bool] = True, track_running_stats: Optional[bool] = True, *args, **kwargs) -> None:
        super().__init__(num_features=num_features, eps=eps, momentum=momentum, affine=affine,
                         track_running_stats=track_running_stats)


class LayerNorm2D_NCHW(nn.GroupNorm):
    """cvnets/layers/normalization/layer_norm.py:75-108 (``layer_norm_2d``): GroupNorm with one group."""

    def __init__(self, num_features: int, eps: Optional[float] = 1e-5, elementwise_affine: Optional[bool] = True,
                 *args, **kwargs) -> None:
        super().__init__(num_channels=num_features, eps=eps, affine=elementwise_affine, num_groups=1)
        self.num_channels = num_features

    def forward(self, x: Tensor) -> Tensor:
        """Stand-alone use (inside MobileViTBlockv2 the norm is a load mode of the consuming GEMM)."""
        from types import SimpleNamespace
        from . import functional as Fn
        _need_cuda(x, "LayerNorm2D_NCHW")
        if x.dim() != 4 or x.shape[1] % 8 or not self.affine:
            raise NotImplementedError("LayerNorm2D_NCHW: expects [B, C, H, W] with C % 8 == 0 and affine=True")
        cfg = getattr(self, "_cfg", None)
        if cfg is None:  # ONE cfg object per module: its id keys the module's slice of the step workspace
            cfg = self._cfg = SimpleNamespace()
        cfg.eps = float(self.eps)
        _bind(self, cfg, [self.weight, self.bias])
        return Fn.GroupNorm1Fn.apply(Fn.to_bf16_cl(x), cfg, self.weight, self.bias)

    def __repr__(self):
        return "{}(num_channels={}, eps={}, affine={})".format(self.__class__.__name__, self.num_channels, self.eps, self.affine)


class LayerNorm(nn.LayerNorm):
    """cvnets/layers/normalization/layer_norm.py:14-72 (``layer_norm``): nn.LayerNorm over the last dimension of [N, S, C].
    Runs fused: per-token statistics (cvb_ln_stats / a producer epilogue) + the normalising load mode of the consuming GEMM."""

    def __init__(self, normalized_shape, eps: Optional[float] = 1e-5, elementwise_affine: Optional[bool] = True, *args, **kwargs):
        super().__init__(normalized_shape=normalized_shape, eps=eps, elementwise_affine=elementwise_affine)

    def forward(self, x: Tensor) -> Tensor:
        """Stand-alone use on [..., C] (inside TransformerEncoder the norm is a load mode of the consuming GEMM)."""
        from types import SimpleNamespace
        from . import functional as Fn
        _need_cuda(x, self.__class__.__name__)
        C = self.normalized_shape[0]
        if len(self.normalized_shape) != 1 or x.shape[-1] != C or C % 8 or C > 1024 or not self.elementwise_affine:
            raise NotImplementedError("LayerNorm: last-dimension normalisation with C % 8 == 0, C <= 1024 and affine weights is implemented")
        if x.dim() > 2 and x.shape[1] == C:
            raise NotImplementedError("LayerNorm on a channel-first tensor (x.shape[1] == C, layer_norm.py:52-65) is not implemented")
        cfg = getattr(self, "_cfg", None)
        if cfg is None:
            cfg = self._cfg = SimpleNamespace()
        cfg.eps = float(self.eps)
        _bind(self, cfg, [self.weight, self.bias])
        return Fn.LayerNormFn.apply(x, cfg, self.weight, self.bias)


class LayerNormFP32(LayerNorm):
    """cvnets/layers/normalization/layer_norm.py:111-137 (``layer_norm_fp32``, the ViT-B recipe's norm): the reference upcasts the
    input to fp32 around nn.LayerNorm.  Here every LayerNorm already computes its statistics and the normalisation in fp32 from the
    bf16 activation, so the two classes share one kernel path; the class exists for the registry name / isinstance checks."""


class GELU(nn.GELU):
    """cvnets/layers/activation/gelu.py."""

    def __init__(self, *args, **kwargs) -> None:
        super().__init__()


norm_layers_tuple = (nn.BatchNorm2d, nn.GroupNorm, nn.LayerNorm)


class _KernelAct(nn.Module):
    """Stand-alone activation modules of the MobileNetv3-style blocks (cvnets/layers/activation/{relu,hard_swish,hard_sigmoid,sigmoid}.py): one
    element-wise pass of the kernel library (cvb_act_fwd / cvb_act_bwd).  ``inplace`` is accepted and ignored (outputs are always new tensors)."""
    kind = -1

    def __init__(self, inplace: Optional[bool] = False, *args, **kwargs) -> None:
        super().__init__()
        self.inplace = inplace

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        from . import functional as Fn
        _need_cuda(x, self.__class__.__name__)
        return Fn.ActFn.apply(Fn.to_bf16_cl(x) if x.dim() == 4 else x.to(torch.bfloat16).contiguous(), self.kind)


class ReLU(_KernelAct):
    kind = 2


class Hardswish(_KernelAct):
    kind = 3


class Hardsigmoid(_KernelAct):
    kind = 4


class Sigmoid(_KernelAct):
    kind = 5


class AdaptiveAvgPool2d(nn.Module):
    """cvnets/layers/pooling.py: nn.AdaptiveAvgPool2d; output_size = 1 (the squeeze of SqueezeExcitation, squeeze_excitation.py:67-69) is the
    global mean-pool kernel with keep_dim."""

    def __init__(self, output_size=1, *args, **kwargs) -> None:
        super().__init__()
        if output_size not in (1, (1, 1)):
            raise NotImplementedError("AdaptiveAvgPool2d: output_size = 1 is on the GPU hot path")
        self.output_size = output_size

    def forward(self, x: Tensor) -> Tensor:
        from . import functional as Fn
        _need_cuda(x, "AdaptiveAvgPool2d")
        if x.dim() != 4 or x.shape[1] % 8:
            raise NotImplementedError("AdaptiveAvgPool2d: expects [B, C, H, W] with C % 8 == 0")
        return Fn.GlobalPoolFn.apply(Fn.to_bf16_cl(x), True)


_ACT_CLASSES = {}


def _need_cuda(x: Tensor, who: str):
    if not x.is_cuda:
        raise RuntimeError(f"{who}: ml-cvnets_b200 runs on CUDA (sm_90a) only and has no CPU fallback; got a {x.device} tensor")


def _bind(module: nn.Module, cfg, plist):
    """Ready ``cfg`` for one call of its autograd function: the module's step workspace (if any), the parameters in the function's order,
    and the kernel-layout weight copies ``cfg.prep`` (for functions that have them) refreshed."""
    cfg.ws = getattr(module, "_ws", None)
    cfg.plist = plist
    if hasattr(cfg, "prep"):
        cfg.prep.prepare(force=module.training)
    return cfg


def get_normalization_layer(opts, num_features: int, norm_type: Optional[str] = None, *args, **kwargs) -> nn.Module:
    """cvnets/layers/normalization_layers.py: factory restricted to the norms on the hot path."""
    norm_type = norm_type or _opt(opts, "model.normalization.name", "batch_norm")
    momentum = _opt(opts, "model.normalization.momentum", 0.1)
    if norm_type in ("batch_norm", "batch_norm_2d"):
        return BatchNorm2d(num_features=num_features, momentum=momentum)
    if norm_type in ("layer_norm_2d", "layer_norm_nchw"):
        return LayerNorm2D_NCHW(num_features=num_features)
    if norm_type == "layer_norm":
        return LayerNorm(num_features)
    if norm_type == "layer_norm_fp32":
        return LayerNormFP32(num_features)
    raise NotImplementedError(f"normalization '{norm_type}' is not on the GPU hot path (batch_norm, layer_norm_2d, layer_norm, layer_norm_fp32 are)")


def build_activation_layer(opts, act_type: Optional[str] = None, *args, **kwargs) -> nn.Module:
    """cvnets/layers/activation/__init__.py: ``act_type`` overrides ``model.activation.name``."""
    name = (act_type or _opt(opts, "model.activation.name", "swish")).lower()
    table = {"swish": Swish, "silu": Swish, "gelu": GELU, "relu": ReLU, "hard_swish": Hardswish, "hard_sigmoid": Hardsigmoid, "sigmoid": Sigmoid}
    if name in table:
        return table[name]()
    raise NotImplementedError(f"activation '{name}' is not on the GPU hot path ({', '.join(sorted(table))} are)")


class Conv2d(nn.Conv2d):
    """cvnets/layers/conv_layer.py:18-66."""


class ConvLayer2d(BaseLayer):
    """cvnets/layers/conv_layer.py:69-267,275-277: ``self.block = Sequential(conv[, norm][, act])`` with keys
    ``block.conv``, ``block.norm``, ``block.act``; auto padding ``(k-1)//2 * dilation``; bias only on request."""

    def __init__(self, opts, in_channels: int, out_channels: int, kernel_size: Union[int, Tuple[int, ...]],
                 stride: Union[int, Tuple[int, ...]] = 1, dilation: Union[int, Tuple[int, ...]] = 1,
                 padding: Optional[Union[int, Tuple[int, ...]]] = None, groups: int = 1, bias: bool = False,
                 padding_mode: str = "zeros", use_norm: bool = True, use_act: bool = True,
                 norm_layer: Optional[nn.Module] = None, act_layer: Optional[nn.Module] = None, *args, **kwargs) -> None:
        super().__init__()
        if norm_layer is None and use_norm:
            norm_type = _opt(opts, "model.normalization.name", "batch_norm")
            norm_layer = get_normalization_layer(opts=opts, num_features=out_channels, norm_type=norm_type)
        if act_layer is None and use_act:
            act_layer = build_activation_layer(opts)
        if use_norm and isinstance(norm_layer, LayerNorm2D_NCHW):
            bias = True
        ks = (kernel_size,) * 2 if isinstance(kernel_size, int) else tuple(kernel_size)
        st = (stride,) * 2 if isinstance(stride, int) else tuple(stride)
        dl = (dilation,) * 2 if isinstance(dilation, int) else tuple(dilation)
        if padding is None:
            padding = tuple(int((ks[i] - 1) / 2) * dl[i] for i in range(2))
        assert in_channels % groups == 0 and out_channels % groups == 0
        block = nn.Sequential()
        block.add_module("conv", Conv2d(in_channels, out_channels, ks, st, padding, dl, groups, bias, padding_mode))
        self.norm_name = None
        if use_norm:
            block.add_module("norm", norm_layer)
            self.norm_name = norm_layer.__class__.__name__
        self.act_name = None
        if use_act:
            block.add_module("act", act_layer)
            self.act_name = act_layer.__class__.__name__
        self.block = block
        self.in_channels, self.out_channels = in_channels, out_channels
        self.stride, self.groups, self.kernel_size, self.bias, self.dilation = st, groups, ks, bias, dl
        self._stem = None

    def forward(self, x: Tensor, residual: Optional[Tensor] = None) -> Tensor:
        """Stand-alone use: the MobileViT stem pattern (3 -> C0, 3x3, stride 2, BN, Swish), any 1x1 conv (+bias) [+BatchNorm] [+Swish/GELU]
        and the depthwise 3x3 / 5x5 conv [+BatchNorm] [+Swish].  ``residual`` (1x1 only, extension) is added in the GEMM epilogue."""
        from types import SimpleNamespace
        from . import functional as Fn
        from . import ops
        from .ops import PreparedWeights as PW
        conv = self.block.conv
        _need_cuda(x, "ConvLayer2d")
        if (self.in_channels == 3 and self.kernel_size == (3, 3) and self.stride == (2, 2) and self.groups == 1
                and self.dilation == (1, 1) and conv.bias is None and self.norm_name == "BatchNorm2d" and self.act_name is not None
                and self.out_channels % 8 == 0):
            from .modules import _stem_forward
            return _stem_forward(self, x)
        kinds = {"Swish": ops.ACT_SILU, "GELU": ops.ACT_GELU, "ReLU": ops.ACT_RELU, "Hardswish": ops.ACT_HARDSWISH, "Hardsigmoid": ops.ACT_HARDSIGMOID,
                 "Sigmoid": ops.ACT_SIGMOID}
        if self.norm_name not in (None, "BatchNorm2d") or self.act_name not in (None, *kinds) or conv.padding_mode != "zeros":
            raise NotImplementedError(f"stand-alone ConvLayer2d with norm={self.norm_name}, act={self.act_name} has no kernel path")
        act = None if self.act_name is None else kinds[self.act_name]
        norm = self.block.norm if self.norm_name is not None else None
        pad = tuple(conv.padding) if not isinstance(conv.padding, str) else None
        # groups = 1: 1x1 convs are the GEMM itself; square k x k convs run as im2col + GEMM (ViT conv stem, MobileViT-v1 3x3 convs)
        pointwise = (self.groups == 1 and self.dilation == (1, 1) and self.kernel_size[0] == self.kernel_size[1] and self.stride[0] == self.stride[1]
                     and pad is not None and pad[0] == pad[1] and (self.in_channels % 8 == 0 or self.kernel_size[0] > 1))
        dil = self.dilation[0]
        # depthwise 3x3 (dilated: stride 1) and undilated 5x5 (EfficientNet)
        dw_pad = (self.kernel_size[0] - 1) // 2 * dil
        depthwise = (self.kernel_size in ((3, 3), (5, 5)) and self.groups == self.in_channels == self.out_channels
                     and self.dilation[0] == self.dilation[1] and self.stride in ((1, 1), (2, 2)) and (dil == 1 or self.stride == (1, 1))
                     and (dil == 1 or self.kernel_size == (3, 3)) and conv.bias is None and tuple(conv.padding) == (dw_pad, dw_pad))
        if depthwise:
            pointwise = False
        if not (pointwise or depthwise) or self.out_channels % 8 or (depthwise and self.in_channels % 8):
            raise NotImplementedError("stand-alone ConvLayer2d: undilated groups=1 convs with square kernels (out_channels % 8 == 0; in_channels % 8 == 0 "
                                      "for 1x1), depthwise 3x3 convs (dilated: stride 1) and undilated depthwise 5x5 convs have kernel paths")
        if self._stem is None:
            prep = PW()
            k = self.kernel_size[0]
            cfg = SimpleNamespace(prep=prep, cout=self.out_channels, act=act, has_bias=conv.bias is not None, stride=self.stride[0], k=k,
                                  pad=pad[0] if pad is not None else 0, dilation=dil)
            if pointwise and k == 1 and self.stride[0] == 1:
                cfg.i_w = prep.add(conv.weight, PW.KIND_ROWMAJOR)
                cfg.i_wt = prep.add(conv.weight, PW.KIND_TRANSPOSED)
            elif pointwise:
                cfg.i_w = prep.add(conv.weight, PW.KIND_PATCH, rot=k * k)
                cfg.i_wt = prep.add(conv.weight, PW.KIND_PATCH_T, rot=k * k)
            else:
                cfg.i_w = prep.add(conv.weight, PW.KIND_TAPMAJOR_F32)
            self._stem = cfg
        cfg = self._stem
        cfg.bn = Fn.bn_cfg(norm) if norm is not None else None
        g, b = (norm.weight, norm.bias) if norm is not None else (None, None)
        _bind(self, cfg, [conv.weight] + ([conv.bias] if conv.bias is not None else []) + ([g, b] if norm is not None else []))
        if not (pointwise and cfg.k > 1 and x.dtype == torch.float32 and self.in_channels % 8):
            x = Fn.to_bf16_cl(x)  # (fp32 images with few channels go through the gather kernel as they are)
        if pointwise:
            return Fn.PointwiseConvFn.apply(x, cfg, Fn.to_bf16_cl(residual) if residual is not None else None, conv.weight, conv.bias, g, b)
        if residual is not None:
            raise NotImplementedError("residual is supported for 1x1 convs only")
        if act not in (None, ops.ACT_SILU):
            raise NotImplementedError("depthwise conv followed by an activation other than Swish")
        return Fn.DepthwiseConvFn.apply(x, cfg, conv.weight, g, b)

    def __repr__(self):
        s = self.block[0].__repr__()[:-1]
        if self.norm_name is not None:
            s += ", normalization={}".format(self.norm_name)
        if self.act_name is not None:
            s += ", activation={}".format(self.act_name)
        return s + ")"


class LinearLayer(BaseLayer):
    """cvnets/layers/linear_layer.py:17-103."""

    def __init__(self, in_features: int, out_features: int, bias: Optional[bool] = True, channel_first: Optional[bool] = False,
                 *args, **kwargs) -> None:
        super().__init__()
        self.weight = nn.Parameter(torch.empty(out_features, in_features))
        self.bias = nn.Parameter(torch.empty(out_features)) if bias else None
        self.in_features, self.out_features, self.channel_first = in_features, out_features, channel_first
        self.reset_params()

    def reset_params(self):
        nn.init.xavier_uniform_(self.weight)
        if self.bias is not None:
            nn.init.constant_(self.bias, 0)

    def forward(self, x: Tensor) -> Tensor:
        """Stand-alone use (the classifier head fuses it with GlobalPool; TransformerEncoder fuses its four linears)."""
        from types import SimpleNamespace
        from . import functional as Fn
        from .ops import PreparedWeights as PW
        _need_cuda(x, "LinearLayer")
        if self.channel_first or x.shape[-1] != self.in_features or self.in_features % 8:
            raise NotImplementedError("LinearLayer: channel-last inputs with in_features % 8 == 0 are implemented")
        if getattr(self, "_cfg", None) is None:
            prep = PW()
            npad = (self.out_features + 7) // 8 * 8
            cfg = SimpleNamespace(prep=prep, cout=self.out_features, npad=npad, i_w=prep.add(self.weight, PW.KIND_ROWMAJOR, dst_rows=npad),
                                  i_wt=prep.add(self.weight, PW.KIND_TRANSPOSED, ldd=npad))
            if self.bias is not None:
                cfg.i_b = prep.add(self.bias, PW.KIND_VECTOR_F32, dst_rows=npad)
            self._cfg = cfg
        cfg = _bind(self, self._cfg, [self.weight] + ([self.bias] if self.bias is not None else []))
        return Fn.LinearFn.apply(x, cfg, self.weight, self.bias)

    def __repr__(self):
        return "{}(in_features={}, out_features={}, bias={}, channel_first={})".format(
            self.__class__.__name__, self.in_features, self.out_features, self.bias is not None, self.channel_first)


class GlobalPool(BaseLayer):
    """cvnets/layers/global_pool.py:16-83 (mean pooling only on the hot path)."""

    def __init__(self, pool_type: Optional[str] = "mean", keep_dim: Optional[bool] = False, *args, **kwargs) -> None:
        super().__init__()
        if pool_type != "mean":
            raise NotImplementedError("only mean pooling is on the GPU hot path")
        self.pool_type, self.keep_dim = pool_type, keep_dim

    def forward(self, x: Tensor) -> Tensor:
        from . import functional as Fn
        _need_cuda(x, "GlobalPool")
        if x.dim() != 4 or x.shape[1] % 8:
            raise NotImplementedError("GlobalPool: expects [B, C, H, W] with C % 8 == 0")
        return Fn.GlobalPoolFn.apply(Fn.to_bf16_cl(x), self.keep_dim)

    def __repr__(self):
        return "{}(type={})".format(self.__class__.__name__, self.pool_type)


class LinearSelfAttention(BaseLayer):
    """cvnets/layers/linear_attention.py:16-215.  Children ``qkv_proj`` (d -> 1+2d, bias) and ``out_proj`` (d -> d, bias);
    the forward runs inside MobileViTBlockv2Fn (qkv GEMM -> fused softmax/context/relu kernel -> out_proj GEMM)."""

    def __init__(self, opts, embed_dim: int, attn_dropout: Optional[float] = 0.0, bias: Optional[bool] = True, *args, **kwargs) -> None:
        super().__init__()
        self.qkv_proj = ConvLayer2d(opts=opts, in_channels=embed_dim, out_channels=1 + (2 * embed_dim), bias=bias, kernel_size=1,
                                    use_norm=False, use_act=False)
        self.attn_dropout = Dropout(p=attn_dropout)
        self.out_proj = ConvLayer2d(opts=opts, in_channels=embed_dim, out_channels=embed_dim, bias=bias, kernel_size=1,
                                    use_norm=False, use_act=False)
        self.embed_dim = embed_dim

    def forward(self, x: Tensor, x_prev: Optional[Tensor] = None, *args, residual: Optional[Tensor] = None, **kwargs) -> Tensor:
        """Stand-alone self-attention on x [B, d, P, N] / cross-attention against x_prev [B, d, P, M] (linear_attention.py:134-215).
        Inside MobileViTBlockv2 the same kernels run on the folded feature map.  ``residual`` (extension) is added in out_proj's epilogue."""
        from types import SimpleNamespace
        from . import functional as Fn
        from .ops import PreparedWeights as PW
        _need_cuda(x, "LinearSelfAttention")
        d = self.embed_dim
        if x.dim() != 4 or x.shape[1] != d or d % 8 or self.attn_dropout.p:
            raise NotImplementedError("LinearSelfAttention: expects [B, d, P, N] with d % 8 == 0 and attn_dropout == 0")
        if self.qkv_proj.block.conv.bias is None or self.out_proj.block.conv.bias is None:
            raise NotImplementedError("LinearSelfAttention with bias=False is not implemented")
        if getattr(self, "_cfg", None) is None:
            prep = PW()
            wq, bq, wo = self.qkv_proj.block.conv.weight, self.qkv_proj.block.conv.bias, self.out_proj.block.conv.weight
            # reference row order [q, K(d), V(d)] -> kernel order [K, V, q, pad(7)]  (rot = 1)
            self._cfg = SimpleNamespace(prep=prep, i_wqkv=prep.add(wq, PW.KIND_ROWMAJOR, rot=1, dst_rows=2 * d + 8),
                                        i_wqkvt=prep.add(wq, PW.KIND_TRANSPOSED, rot=1, ldd=2 * d + 8),
                                        i_bqkv=prep.add(bq, PW.KIND_VECTOR_F32, rot=1, dst_rows=2 * d + 8),
                                        i_wo=prep.add(wo, PW.KIND_ROWMAJOR), i_wot=prep.add(wo, PW.KIND_TRANSPOSED))
        cfg = _bind(self, self._cfg, [self.qkv_proj.block.conv.weight, self.qkv_proj.block.conv.bias, self.out_proj.block.conv.weight,
                                      self.out_proj.block.conv.bias])
        xp = Fn.to_bf16_cl(x_prev) if x_prev is not None else None
        res = Fn.to_bf16_cl(residual) if residual is not None else None
        return Fn.LinearSelfAttentionFn.apply(Fn.to_bf16_cl(x), cfg, xp, res, *cfg.plist)

    def __repr__(self):
        return "{}(embed_dim={}, attn_dropout={})".format(self.__class__.__name__, self.embed_dim, self.attn_dropout.p)


class MultiHeadAttention(BaseLayer):
    """cvnets/layers/multi_head_attention.py:18-309.  Same constructor (note: no ``opts``), children ``qkv_proj`` (C -> 3C) and
    ``out_proj`` (C -> output_dim) as ``LinearLayer``s, same ``forward(x_q, x_kv, key_padding_mask, attn_mask)`` signature.
    Self-attention only (the cross-attention branch, :159-185, raises); attention dropout must be 0."""

    def __init__(self, embed_dim: int, num_heads: int, attn_dropout: Optional[float] = 0.0, bias: Optional[bool] = True,
                 output_dim: Optional[int] = None, coreml_compatible: Optional[bool] = False, *args, **kwargs) -> None:
        if output_dim is None:
            output_dim = embed_dim
        super().__init__()
        if embed_dim % num_heads != 0:
            raise ValueError("Embedding dim must be divisible by number of heads in {}. Got: embed_dim={} and num_heads={}".format(
                self.__class__.__name__, embed_dim, num_heads))
        self.qkv_proj = LinearLayer(in_features=embed_dim, out_features=3 * embed_dim, bias=bias)
        self.attn_dropout = Dropout(p=attn_dropout)
        self.out_proj = LinearLayer(in_features=embed_dim, out_features=output_dim, bias=bias)
        self.head_dim = embed_dim // num_heads
        self.scaling = self.head_dim ** -0.5
        self.softmax = nn.Softmax(dim=-1)
        self.num_heads = num_heads
        self.embed_dim = embed_dim
        self.coreml_compatible = coreml_compatible
        self.use_separate_proj_weight = embed_dim != output_dim
        self._cfg = None

    def __repr__(self):
        return "{}(head_dim={}, num_heads={}, attn_dropout={})".format(self.__class__.__name__, self.head_dim, self.num_heads, self.attn_dropout.p)

    def check_supported(self):
        if self.attn_dropout.p and self.training:
            raise NotImplementedError("attention dropout > 0 in training mode is not implemented")
        if self.head_dim % 2 or not (2 <= self.head_dim <= 64):
            raise NotImplementedError(f"head_dim {self.head_dim} is not implemented (even values up to 64 are)")
        if self.qkv_proj.bias is None or self.out_proj.bias is None:
            raise NotImplementedError("bias=False is not implemented")

    def build_cfg(self, prep):
        """Register the kernel-layout weight copies in ``prep``; returns the index namespace used by the autograd functions."""
        from types import SimpleNamespace
        from .ops import PreparedWeights as PW
        self.check_supported()
        ix = SimpleNamespace(heads=self.num_heads, head_dim=self.head_dim, scale=self.scaling, out_dim=self.out_proj.out_features)
        ix.i_wqkv = prep.add(self.qkv_proj.weight, PW.KIND_ROWMAJOR)
        ix.i_wqkvt = prep.add(self.qkv_proj.weight, PW.KIND_TRANSPOSED)
        ix.i_wo = prep.add(self.out_proj.weight, PW.KIND_ROWMAJOR)
        ix.i_wot = prep.add(self.out_proj.weight, PW.KIND_TRANSPOSED)
        return ix

    def forward(self, x_q: Tensor, x_kv: Optional[Tensor] = None, key_padding_mask: Optional[Tensor] = None,
                attn_mask: Optional[Tensor] = None, *args, **kwargs) -> Tensor:
        from . import functional as Fn
        from .ops import PreparedWeights as PW
        if x_kv is not None:
            raise NotImplementedError("cross-attention (x_kv) is not implemented on the GPU path")
        if not x_q.is_cuda:
            raise RuntimeError("MultiHeadAttention: ml-cvnets_b200 has no CPU path")
        if x_q.dim() != 3:
            raise NotImplementedError("MultiHeadAttention expects [N, S, C]")
        if x_q.shape[1] > 256 and self.head_dim != 64:
            raise NotImplementedError(f"MultiHeadAttention: S = {x_q.shape[1]} > 256 needs head_dim 64 (the streaming attention kernels); "
                                      f"head_dim {self.head_dim} keeps a head in shared memory and supports S <= 256")
        if self._cfg is None:
            prep = PW()
            self._cfg = self.build_cfg(prep)
            self._cfg.prep = prep
        cfg = self._cfg
        cfg.masks = (attn_mask, key_padding_mask)
        cfg.prep.prepare(force=self.training)
        x = x_q.to(torch.bfloat16).contiguous()
        return Fn.MultiHeadAttentionFn.apply(x, cfg, self.qkv_proj.weight, self.qkv_proj.bias, self.out_proj.weight, self.out_proj.bias)

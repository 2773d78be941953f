"""ORACLE -- TEST INFRASTRUCTURE ONLY. Not part of the product path.

A CPU (fp32, plain PyTorch) restatement of the apple/ml-cvnets vision-backbone hot path that
``BASELINE.json:north_star`` names: ConvLayer2d(+BN+SiLU), InvertedResidual, LinearSelfAttention,
LinearAttnFFN, MobileViTBlockv2 and the MobileViTv2 classifier that assembles them.

Only ``tests/``, ``__graft_entry__.smoke()`` and ``bench.py``'s CPU-baseline legs may import this file.
The product (``ml-cvnets_b200``) never does: it fails loudly when its CUDA library is missing.

Parity status: PINNED.  ``tests/golden/make_golden.py`` imports the real reference from
``/root/reference`` (possible only in the build container), runs the reference ``nn.Module``s on seeded
inputs and commits their outputs/gradients under ``tests/golden/``; ``tests/test_oracle_golden.py``
checks every function below against those fixtures (fp32, atol/rtol 1e-5 class).

Every function is a *functional* restatement: parameters arrive in a flat ``dict`` keyed exactly like
the reference ``state_dict`` (SURVEY.md Appendix B), so nothing here depends on the product's module
classes.  All citations are relative to the reference checkout (``/root/reference``).
"""
from __future__ import annotations

import math
from typing import Dict, List, Optional, Tuple

import torch
import torch.nn.functional as F

Tensor = torch.Tensor
Params = Dict[str, Tensor]

BN_EPS = 1e-5  # cvnets/layers/normalization/batch_norm.py:31-47 (nn.BatchNorm2d default eps)
GN_EPS = 1e-5  # cvnets/layers/normalization/layer_norm.py:93-103 (nn.GroupNorm(1, C, eps=1e-5))


# --------------------------------------------------------------------------------------------
# configuration (cvnets/models/classification/config/mobilevit_v2.py:11-77, utils/math_utils.py:9-35)
# --------------------------------------------------------------------------------------------
def make_divisible(v, divisor: int = 8, min_value=None):
    """utils/math_utils.py:9-30."""
    if min_value is None:
        min_value = divisor
    new_v = max(min_value, int(v + divisor / 2) // divisor * divisor)
    if new_v < 0.9 * v:
        new_v += divisor
    return new_v


def mobilevit_v2_config(width_multiplier: float = 1.0) -> Dict:
    """cvnets/models/classification/config/mobilevit_v2.py:11-77."""
    wm = width_multiplier
    layer_0_dim = max(16, min(64, 32 * wm))
    layer_0_dim = int(make_divisible(layer_0_dim, divisor=8, min_value=16))
    return {
        "layer0": {"img_channels": 3, "out_channels": layer_0_dim},
        "layer1": {"out_channels": int(make_divisible(64 * wm, divisor=16)), "expand_ratio": 2,
                   "num_blocks": 1, "stride": 1, "block_type": "mv2"},
        "layer2": {"out_channels": int(make_divisible(128 * wm, divisor=8)), "expand_ratio": 2,
                   "num_blocks": 2, "stride": 2, "block_type": "mv2"},
        "layer3": {"out_channels": int(make_divisible(256 * wm, divisor=8)),
                   "attn_unit_dim": int(make_divisible(128 * wm, divisor=8)), "ffn_multiplier": 2,
                   "attn_blocks": 2, "patch_h": 2, "patch_w": 2, "stride": 2, "mv_expand_ratio": 2,
                   "block_type": "mobilevit"},
        "layer4": {"out_channels": int(make_divisible(384 * wm, divisor=8)),
                   "attn_unit_dim": int(make_divisible(192 * wm, divisor=8)), "ffn_multiplier": 2,
                   "attn_blocks": 4, "patch_h": 2, "patch_w": 2, "stride": 2, "mv_expand_ratio": 2,
                   "block_type": "mobilevit"},
        "layer5": {"out_channels": int(make_divisible(512 * wm, divisor=8)),
                   "attn_unit_dim": int(make_divisible(256 * wm, divisor=8)), "ffn_multiplier": 2,
                   "attn_blocks": 3, "patch_h": 2, "patch_w": 2, "stride": 2, "mv_expand_ratio": 2,
                   "block_type": "mobilevit"},
    }


# --------------------------------------------------------------------------------------------
# layers
# --------------------------------------------------------------------------------------------
def batch_norm(P: Params, pre: str, x: Tensor, training: bool, momentum: float = 0.1) -> Tensor:
    """cvnets/layers/normalization/batch_norm.py:14-49 == nn.BatchNorm2d(eps=1e-5, momentum=0.1).

    Training: batch mean / biased var normalise; running stats get the EMA with *unbiased* var and
    ``num_batches_tracked += 1`` (SURVEY App. A1).  ``P`` buffers are updated in place like the module.
    """
    rm, rv = P[pre + ".running_mean"], P[pre + ".running_var"]
    if training and (pre + ".num_batches_tracked") in P:
        P[pre + ".num_batches_tracked"] += 1
    return F.batch_norm(x, rm, rv, P[pre + ".weight"], P[pre + ".bias"], training, momentum, BN_EPS)


def conv_layer_2d(P: Params, pre: str, x: Tensor, *, stride: int = 1, groups: int = 1, use_norm: bool = True,
                  use_act: bool = True, training: bool = True, momentum: float = 0.1, act: str = "swish", dilation: int = 1) -> Tensor:
    """ConvLayer2d = Sequential(conv[, norm][, act]) (cvnets/layers/conv_layer.py:200-226,254-255).

    Auto padding ``(k-1)//2 * dilation`` (``:182-185``); norm = BatchNorm2d (``model.normalization.name=batch_norm``,
    ``:138-144``); act = Swish == nn.SiLU (cvnets/layers/activation/swish.py:13-20).
    """
    w = P[pre + ".block.conv.weight"]
    b = P.get(pre + ".block.conv.bias")
    k = w.shape[-1]
    x = F.conv2d(x, w, b, stride=stride, padding=(k - 1) // 2 * dilation, groups=groups, dilation=dilation)
    if use_norm:
        x = batch_norm(P, pre + ".block.norm", x, training, momentum)
    if use_act:
        x = F.silu(x) if act == "swish" else F.gelu(x)
    return x


def layer_norm_2d(P: Params, pre: str, x: Tensor) -> Tensor:
    """LayerNorm2D_NCHW == nn.GroupNorm(num_groups=1) (cvnets/layers/normalization/layer_norm.py:75-108):
    statistics over all of (C, P, N) per sample, per-channel affine."""
    return F.group_norm(x, 1, P[pre + ".weight"], P[pre + ".bias"], GN_EPS)


def linear_self_attention(P: Params, pre: str, x: Tensor, x_prev: Optional[Tensor] = None) -> Tensor:
    """LinearSelfAttention._forward_self_attn (cvnets/layers/linear_attention.py:134-161) and, with ``x_prev`` [B, d, P, M],
    _forward_cross_attn (:163-207): query + key are projected from x_prev with the first 1+d rows of the packed weight, the
    value from x with the last d rows; softmax / context over M.

    x: [B, d, P, N].  qkv 1x1 (d -> 1+2d, bias) -> split [1, d, d] -> softmax over N (dim=-1) ->
    ctx = sum_N(key * scores) -> relu(value) * ctx -> out_proj 1x1 (d -> d, bias).
    """
    d = x.shape[1]
    w, b = P[pre + ".qkv_proj.block.conv.weight"], P[pre + ".qkv_proj.block.conv.bias"]
    if x_prev is not None:
        assert x_prev.shape[2] == x.shape[2], "The number of pixels in a patch for query and key_value should be the same"
        qk = F.conv2d(x_prev, w[: d + 1], b[: d + 1])
        query, key = torch.split(qk, [1, d], dim=1)
        value = F.conv2d(x, w[d + 1:], b[d + 1:])
        context_scores = F.softmax(query, dim=-1)
        context_vector = (key * context_scores).sum(dim=-1, keepdim=True)
        out = F.relu(value) * context_vector.expand_as(value)
        return F.conv2d(out, P[pre + ".out_proj.block.conv.weight"], P[pre + ".out_proj.block.conv.bias"])
    qkv = F.conv2d(x, w, b)
    query, key, value = torch.split(qkv, [1, d, d], dim=1)
    context_scores = F.softmax(query, dim=-1)
    context_vector = (key * context_scores).sum(dim=-1, keepdim=True)
    out = F.relu(value) * context_vector.expand_as(value)
    return F.conv2d(out, P[pre + ".out_proj.block.conv.weight"], P[pre + ".out_proj.block.conv.bias"])


def linear_attn_ffn(P: Params, pre: str, x: Tensor, x_prev: Optional[Tensor] = None) -> Tensor:
    """LinearAttnFFN.forward (cvnets/modules/transformer.py:248-264), dropout p=0; with ``x_prev`` the cross-attention branch (:254-260:
    only x is normalised, x_prev enters the attention raw).

    x = x + LSA(GN1(x)[, x_prev]);  x = x + conv1x1(silu(conv1x1(GN1(x)))).  Child indices: pre_norm_attn.{0,1},
    pre_norm_ffn.{0,1,3} (``:192-228``).
    """
    a = layer_norm_2d(P, pre + ".pre_norm_attn.0", x)
    x = x + linear_self_attention(P, pre + ".pre_norm_attn.1", a, x_prev)
    f = layer_norm_2d(P, pre + ".pre_norm_ffn.0", x)
    f = F.silu(F.conv2d(f, P[pre + ".pre_norm_ffn.1.block.conv.weight"], P[pre + ".pre_norm_ffn.1.block.conv.bias"]))
    f = F.conv2d(f, P[pre + ".pre_norm_ffn.3.block.conv.weight"], P[pre + ".pre_norm_ffn.3.block.conv.bias"])
    return x + f


def layer_norm(P: Params, pre: str, x: Tensor, eps: float = 1e-5) -> Tensor:
    """LayerNorm, channel-last branch (cvnets/layers/normalization/layer_norm.py:14-72, ``super().forward``): nn.LayerNorm over
    the last dimension.  (The reference switches to a channel-first formula when ``x.shape[1] == C`` and ``x.ndim > 2``,
    ``:52-65`` -- i.e. for [N, S, C] inputs with S == C; the hot-path configs never have S == C and the product rejects it.)"""
    return F.layer_norm(x, (x.shape[-1],), P[pre + ".weight"], P[pre + ".bias"], eps)


def multi_head_attention(P: Params, pre: str, x: Tensor, num_heads: int, key_padding_mask: Optional[Tensor] = None,
                         attn_mask: Optional[Tensor] = None) -> Tensor:
    """MultiHeadAttention.forward_default, self-attention branch (cvnets/layers/multi_head_attention.py:135-239), dropout p=0.

    x: [N, S, C].  qkv = Linear(C -> 3C) reshaped [N,S,3,h,c] -> [N,h,3,S,c] (:148-153); q *= c^-0.5 (:187); attn = q k^T (:194);
    + attn_mask[N,1,S,T] (:197-208); masked_fill(key_padding_mask, -inf) (:210-224); softmax in fp32 then cast back (:226-228);
    attn v (:233); merge heads (:236); out_proj (:237).
    """
    b, s_len, c = x.shape
    hd = c // num_heads
    qkv = F.linear(x, P[pre + ".qkv_proj.weight"], P[pre + ".qkv_proj.bias"]).reshape(b, s_len, 3, num_heads, hd)
    qkv = qkv.transpose(1, 3).contiguous()
    q, k, v = qkv[:, :, 0], qkv[:, :, 1], qkv[:, :, 2]
    q = q * (hd ** -0.5)
    attn = torch.matmul(q, k.transpose(-1, -2))
    if attn_mask is not None:
        attn = attn + attn_mask.unsqueeze(1)
    if key_padding_mask is not None:
        attn = attn.masked_fill(key_padding_mask.unsqueeze(1).unsqueeze(2).to(torch.bool), float("-inf"))
    attn = F.softmax(attn.float(), dim=-1).to(attn.dtype)
    out = torch.matmul(attn, v).transpose(1, 2).reshape(b, s_len, -1)
    return F.linear(out, P[pre + ".out_proj.weight"], P[pre + ".out_proj.bias"])


def activation(x: Tensor, name: str) -> Tensor:
    """build_activation_layer(opts) for the two activations of the transformer recipes: swish (MobileViT) and gelu (ViT / CLIP)."""
    if name == "swish":
        return F.silu(x)
    if name == "gelu":
        return F.gelu(x)
    # MobileNetv3-style blocks (cvnets/layers/activation/{relu,hard_swish,hard_sigmoid,sigmoid}.py == nn.ReLU / Hardswish / Hardsigmoid / Sigmoid)
    if name == "relu":
        return F.relu(x)
    if name == "hard_swish":
        return F.hardswish(x)
    if name == "hard_sigmoid":
        return F.hardsigmoid(x)
    if name == "sigmoid":
        return torch.sigmoid(x)
    raise NotImplementedError(name)


def transformer_encoder(P: Params, pre: str, x: Tensor, num_heads: int, act: str = "swish", eps: float = 1e-5,
                        key_padding_mask: Optional[Tensor] = None, attn_mask: Optional[Tensor] = None,
                        drop_masks: Optional[Tuple[Optional[Tensor], Optional[Tensor], Optional[Tensor]]] = None) -> Tensor:
    """TransformerEncoder.forward (cvnets/modules/transformer.py:129-156), pre-norm:
    x = x + DropPath(Dropout(MHA(LN(x))));  x = x + DropPath(Dropout(Linear(Dropout_ffn(act(Linear(LN(x)))))))  (:77-100, 139-156).
    Child indices pre_norm_mha.{0,1}, pre_norm_ffn.{0,1,4}.  ``drop_masks`` = (attention-branch, ffn-hidden, ffn-branch) multiplicative masks
    (already scaled by 1/keep, stochastic-depth factor included) -- None = eval mode / p = 0: dropout and stochastic depth are the identity.
    The masks are an INPUT because no two generators produce the same Bernoulli draws; the parity tests take them from the kernel under test."""
    m_attn, m_hid, m_ffn = drop_masks if drop_masks is not None else (None, None, None)
    a = layer_norm(P, pre + ".pre_norm_mha.0", x, eps)
    a = multi_head_attention(P, pre + ".pre_norm_mha.1", a, num_heads, key_padding_mask, attn_mask)
    x = x + (a if m_attn is None else a * m_attn)
    f = layer_norm(P, pre + ".pre_norm_ffn.0", x, eps)
    f = activation(F.linear(f, P[pre + ".pre_norm_ffn.1.weight"], P[pre + ".pre_norm_ffn.1.bias"]), act)
    if m_hid is not None:
        f = f * m_hid
    f = F.linear(f, P[pre + ".pre_norm_ffn.4.weight"], P[pre + ".pre_norm_ffn.4.bias"])
    return x + (f if m_ffn is None else f * m_ffn)


# --------------------------------------------------------------------------------------------
# modules
# --------------------------------------------------------------------------------------------
def inverted_residual(P: Params, pre: str, x: Tensor, *, stride: int, training: bool = True,
                      momentum: float = 0.1, dilation: int = 1) -> Tensor:
    """InvertedResidual (cvnets/modules/mobilenetv2.py:141-246): exp_1x1 (if present) -> conv_3x3 depthwise
    (stride) -> red_1x1 (no act); residual iff stride==1 and Cin==Cout (``:227-235``)."""
    y = x
    if (pre + ".block.exp_1x1.block.conv.weight") in P:
        y = conv_layer_2d(P, pre + ".block.exp_1x1", y, training=training, momentum=momentum)
    hid = P[pre + ".block.conv_3x3.block.conv.weight"].shape[0]
    y = conv_layer_2d(P, pre + ".block.conv_3x3", y, stride=stride, groups=hid, training=training, momentum=momentum, dilation=dilation)
    y = conv_layer_2d(P, pre + ".block.red_1x1", y, use_act=False, training=training, momentum=momentum)
    cout = P[pre + ".block.red_1x1.block.conv.weight"].shape[0]
    if stride == 1 and x.shape[1] == cout:
        y = x + y
    return y


def squeeze_excitation(P: Params, pre: str, x: Tensor, *, act: str = "relu", scale_fn: str = "hard_sigmoid") -> Tensor:
    """SqueezeExcitation.forward (cvnets/modules/squeeze_excitation.py:45-83): x * scale_fn(fc2(act(fc1(AdaptiveAvgPool2d(1)(x))))); fc1 / fc2 are
    1x1 convs with bias and no norm; fc1's activation is the model-wide ``model.activation.name`` (ConvLayer2d use_act=True, :46-55)."""
    s = x.mean(dim=(2, 3), keepdim=True)
    s = activation(F.conv2d(s, P[pre + ".se_layer.fc1.block.conv.weight"], P[pre + ".se_layer.fc1.block.conv.bias"]), act)
    s = F.conv2d(s, P[pre + ".se_layer.fc2.block.conv.weight"], P[pre + ".se_layer.fc2.block.conv.bias"])
    return x * activation(s, scale_fn)


def inverted_residual_se(P: Params, pre: str, x: Tensor, *, stride: int = 1, act: str = "relu", se_scale: str = "hard_sigmoid", fc_act: str = "relu",
                         training: bool = True, momentum: float = 0.1, dilation: int = 1) -> Tensor:
    """InvertedResidualSE (cvnets/modules/mobilenetv2.py:16-138): exp_1x1 (1x1 + BN, if present) -> act -> conv_3x3 (depthwise k x k + BN) -> act ->
    se (if present) -> red_1x1 (1x1 + BN); residual iff stride == 1 and Cin == Cout (:124, :126-128)."""
    y = x
    if (pre + ".block.exp_1x1.block.conv.weight") in P:
        y = activation(conv_layer_2d(P, pre + ".block.exp_1x1", y, use_act=False, training=training, momentum=momentum), act)
    hid = P[pre + ".block.conv_3x3.block.conv.weight"].shape[0]
    y = conv_layer_2d(P, pre + ".block.conv_3x3", y, stride=stride, groups=hid, use_act=False, training=training, momentum=momentum, dilation=dilation)
    y = activation(y, act)
    if (pre + ".block.se.se_layer.fc1.block.conv.weight") in P:
        y = squeeze_excitation(P, pre + ".block.se", y, act=fc_act, scale_fn=se_scale)
    y = conv_layer_2d(P, pre + ".block.red_1x1", y, use_act=False, training=training, momentum=momentum)
    cout = P[pre + ".block.red_1x1.block.conv.weight"].shape[0]
    if stride == 1 and x.shape[1] == cout:
        y = x + y
    return y


def unfolding(fm: Tensor, ph: int = 2, pw: int = 2) -> Tuple[Tensor, Tuple[int, int]]:
    """MobileViTBlockv2.unfolding_pytorch (cvnets/modules/mobilevit_block.py:526-540)."""
    B, C, H, W = fm.shape
    patches = F.unfold(fm, kernel_size=(ph, pw), stride=(ph, pw))
    return patches.reshape(B, C, ph * pw, -1), (H, W)


def folding(patches: Tensor, output_size: Tuple[int, int], ph: int = 2, pw: int = 2) -> Tensor:
    """MobileViTBlockv2.folding_pytorch (cvnets/modules/mobilevit_block.py:542-555)."""
    B, C, Pp, N = patches.shape
    return F.fold(patches.reshape(B, C * Pp, N), output_size=output_size, kernel_size=(ph, pw), stride=(ph, pw))


def mobilevit_block_v2(P: Params, pre: str, x: Tensor, *, n_attn_blocks: int, patch_h: int = 2, patch_w: int = 2,
                       training: bool = True, momentum: float = 0.1, dilation: int = 1) -> Tensor:
    """MobileViTBlockv2.forward_spatial (cvnets/modules/mobilevit_block.py:605-626):
    local_rep (dw3x3+BN+SiLU, 1x1) -> unfold -> n x LinearAttnFFN -> layer_norm_2d -> fold -> conv_proj 1x1 + BN.
    Input H, W must be multiples of the patch (the bilinear ``resize_input_if_needed`` ``:595-603`` never fires
    at 256x256 and is out of scope)."""
    C = x.shape[1]
    assert x.shape[2] % patch_h == 0 and x.shape[3] % patch_w == 0
    fm = conv_layer_2d(P, pre + ".local_rep.0", x, groups=C, training=training, momentum=momentum, dilation=dilation)
    fm = conv_layer_2d(P, pre + ".local_rep.1", fm, use_norm=False, use_act=False)
    patches, out_size = unfolding(fm, patch_h, patch_w)
    for i in range(n_attn_blocks):
        patches = linear_attn_ffn(P, f"{pre}.global_rep.{i}", patches)
    patches = layer_norm_2d(P, f"{pre}.global_rep.{n_attn_blocks}", patches)
    fm = folding(patches, out_size, patch_h, patch_w)
    return conv_layer_2d(P, pre + ".conv_proj", fm, use_act=False, training=training, momentum=momentum)


# --------------------------------------------------------------------------------------------
# model
# --------------------------------------------------------------------------------------------
def mobilevit_v2_layout(width_multiplier: float = 1.0, output_stride: Optional[int] = None) -> List[Tuple[str, str, Dict]]:
    """Stage wiring of MobileViTv2.__init__/_make_layer (cvnets/models/classification/mobilevit_v2.py:25-226),
    as a flat list of (kind, state_dict prefix, kwargs).  ``output_stride`` 8 / 16 (segmentation backbones,
    base_image_encoder.py:38-47): layer_4 and/or layer_5 keep their resolution and dilate instead (mobilevit_v2.py:176-191)."""
    cfg = mobilevit_v2_config(width_multiplier)
    out: List[Tuple[str, str, Dict]] = [("stem", "conv_1", {})]
    dilation = 1
    dilate = {4: output_stride == 8, 5: output_stride in (8, 16)}
    for li in range(1, 6):
        c = cfg[f"layer{li}"]
        if c["block_type"] == "mv2":
            for i in range(c["num_blocks"]):
                out.append(("ir", f"layer_{li}.{i}", {"stride": c["stride"] if i == 0 else 1, "dilation": 1}))
        else:
            prev, stride = dilation, 2
            if dilate.get(li, False):
                dilation, stride = dilation * 2, 1
            out.append(("ir", f"layer_{li}.0", {"stride": stride, "dilation": prev}))
            out.append(("mvit", f"layer_{li}.1", {"n_attn_blocks": c["attn_blocks"], "dilation": dilation}))
    return out


def mobilevit_v2_forward(P: Params, x: Tensor, *, width_multiplier: float = 1.0, training: bool = True,
                         momentum: float = 0.1, return_stages: bool = False, output_stride: Optional[int] = None):
    """BaseImageEncoder.forward -> extract_features -> classifier
    (cvnets/models/classification/base_image_encoder.py:261-301; mobilevit_v2.py:37-45,91-94)."""
    stages = {}
    for kind, pre, kw in mobilevit_v2_layout(width_multiplier, output_stride):
        if kind == "stem":
            x = conv_layer_2d(P, pre, x, stride=2, training=training, momentum=momentum)
        elif kind == "ir":
            x = inverted_residual(P, pre, x, stride=kw["stride"], training=training, momentum=momentum, dilation=kw["dilation"])
        else:
            x = mobilevit_block_v2(P, pre, x, n_attn_blocks=kw["n_attn_blocks"], training=training, momentum=momentum, dilation=kw["dilation"])
        stages[pre] = x
    x = x.mean(dim=[-2, -1])  # GlobalPool(mean) cvnets/layers/global_pool.py:60-71
    logits = F.linear(x, P["classifier.1.weight"], P["classifier.1.bias"])  # cvnets/layers/linear_layer.py:90
    return (logits, stages) if return_stages else logits


# --------------------------------------------------------------------------------------------
# MobileViT v1 (cvnets/modules/mobilevit_block.py:19-326, cvnets/models/classification/mobilevit.py:19-300, config/mobilevit.py:14-200)
# --------------------------------------------------------------------------------------------
MIT_MODES = {  # mode: (mv2 expand, layer1 out, layer2 out, [(out, transformer dim, ffn dim, blocks)] x 3)
    "xx_small": (2, 16, 24, [(48, 64, 128, 2), (64, 80, 160, 4), (80, 96, 192, 3)]),
    "x_small": (4, 32, 48, [(64, 96, 192, 2), (80, 120, 240, 4), (96, 144, 288, 3)]),
    "small": (4, 32, 64, [(96, 144, 288, 2), (128, 192, 384, 4), (160, 240, 480, 3)]),
}


def mobilevit_block_v1_shapes(P: Dict, pre: str, c: int, d: int, ffn: int, n_blocks: int):
    _conv_bn(P, pre + ".local_rep.conv_3x3", c, c, 3)
    _conv_bn(P, pre + ".local_rep.conv_1x1", c, d, 1, norm=False)
    for i in range(n_blocks):
        transformer_encoder_shapes(P, f"{pre}.global_rep.{i}", d, ffn)
    _gn(P, f"{pre}.global_rep.{n_blocks}", d)
    _conv_bn(P, pre + ".conv_proj", d, c, 1)
    _conv_bn(P, pre + ".fusion", 2 * c, c, 3)


def mobilevit_v1_shapes(mode: str = "xx_small", n_classes: int = 1000) -> Dict[str, Tensor]:
    e, c1, c2, mits = MIT_MODES[mode]
    P: Dict[str, Tensor] = {}
    _conv_bn(P, "conv_1", 3, 16, 3)
    inverted_residual_shapes(P, "layer_1.0", 16, c1, e)
    c = c1
    for i in range(3):
        inverted_residual_shapes(P, f"layer_2.{i}", c, c2, e)
        c = c2
    for li, (co, d, f, n) in enumerate(mits):
        inverted_residual_shapes(P, f"layer_{3 + li}.0", c, co, e)
        c = co
        mobilevit_block_v1_shapes(P, f"layer_{3 + li}.1", c, d, f, n)
    _conv_bn(P, "conv_1x1_exp", c, min(4 * c, 960), 1)
    _linear(P, "classifier.fc", min(4 * c, 960), n_classes)
    return P


def mobilevit_block_v1(P: Params, pre: str, x: Tensor, *, n_blocks: int, num_heads: int = 4, patch: int = 2, training: bool = True) -> Tensor:
    """MobileViTBlock.forward_spatial (mobilevit_block.py:269-288), dropout p = 0: dense 3x3 + 1x1 -> unfolding [B*P, N, d] (:186-231) -> n x
    TransformerEncoder -> LayerNorm -> folding (:233-267) -> 1x1 + BN + act -> cat(res, fm) -> dense 3x3 fusion."""
    res = x
    fm = conv_layer_2d(P, pre + ".local_rep.conv_3x3", x, training=training)
    fm = conv_layer_2d(P, pre + ".local_rep.conv_1x1", fm, use_norm=False, use_act=False)
    B, d, H, W = fm.shape
    nh, nw = H // patch, W // patch
    t = fm.reshape(B * d * nh, patch, nw, patch).transpose(1, 2).reshape(B, d, nh * nw, patch * patch).transpose(1, 3)
    t = t.reshape(B * patch * patch, nh * nw, d)
    for i in range(n_blocks):
        t = transformer_encoder(P, f"{pre}.global_rep.{i}", t, num_heads, act="swish", eps=1e-5)
    t = layer_norm(P, f"{pre}.global_rep.{n_blocks}", t, eps=1e-5)
    t = t.contiguous().view(B, patch * patch, nh * nw, d).transpose(1, 3)
    fm = t.reshape(B * d * nh, nw, patch, patch).transpose(1, 2).reshape(B, d, H, W)
    fm = conv_layer_2d(P, pre + ".conv_proj", fm, training=training)
    return conv_layer_2d(P, pre + ".fusion", torch.cat((res, fm), dim=1), training=training)


def mobilevit_v1_layout(mode: str = "xx_small") -> List[Tuple[str, str, Dict]]:
    """Stage wiring of MobileViT.__init__/_make_layer (mobilevit.py:19-300) as a flat list of (kind, state_dict prefix, kwargs):
    the stem, the InvertedResiduals and MobileViTBlocks, and conv_1x1_exp (part of extract_features, before the classifier)."""
    _, _, _, mits = MIT_MODES[mode]
    out: List[Tuple[str, str, Dict]] = [("stem", "conv_1", {}), ("ir", "layer_1.0", {"stride": 1})]
    out += [("ir", f"layer_2.{i}", {"stride": 2 if i == 0 else 1}) for i in range(3)]
    for li, (_, _, _, n) in enumerate(mits):
        out += [("ir", f"layer_{3 + li}.0", {"stride": 2}), ("mvit", f"layer_{3 + li}.1", {"n_blocks": n})]
    out.append(("exp", "conv_1x1_exp", {}))
    return out


def mobilevit_v1_forward(P: Params, x: Tensor, *, mode: str = "xx_small", training: bool = True, return_stages: bool = False):
    """MobileViT.forward (mobilevit.py:19-300 + base_image_encoder.py:261-301), every dropout p = 0.  ``return_stages``: also the output of
    every entry of ``mobilevit_v1_layout``, keyed by its prefix."""
    stages = {}
    for kind, pre, kw in mobilevit_v1_layout(mode):
        if kind == "stem":
            x = conv_layer_2d(P, pre, x, stride=2, training=training)
        elif kind == "ir":
            x = inverted_residual(P, pre, x, stride=kw["stride"], training=training)
        elif kind == "mvit":
            x = mobilevit_block_v1(P, pre, x, n_blocks=kw["n_blocks"], training=training)
        else:
            x = conv_layer_2d(P, pre, x, training=training)
        stages[pre] = x
    logits = F.linear(x.mean(dim=[-2, -1]), P["classifier.fc.weight"], P["classifier.fc.bias"])
    return (logits, stages) if return_stages else logits


# --------------------------------------------------------------------------------------------
# VisionTransformer (cvnets/models/classification/vit.py:33-649, classification path; config/vit.py:12-116)
# --------------------------------------------------------------------------------------------
VIT_MODES = {"tiny": (192, 12, 3), "small": (384, 12, 6), "base": (768, 12, 12)}


def vit_shapes(mode: str = "base", n_classes: int = 1000) -> Dict[str, Tensor]:
    d, n, _ = VIT_MODES[mode]
    stem = max(32, d // 4)
    P: Dict[str, Tensor] = {"cls_token": torch.empty(1, 1, d)}
    _conv_bn(P, "patch_emb.0", 3, stem, 4)
    _conv_bn(P, "patch_emb.1", stem, stem, 2)
    _conv_bn(P, "patch_emb.2", stem, d, 2, norm=False, bias=True)
    _gn(P, "post_transformer_norm", d)
    for i in range(n):
        transformer_encoder_shapes(P, f"transformer.{i}", d, 4 * d)
    _linear(P, "classifier", d, n_classes)
    P["pos_embed.pos_embed.pos_embed"] = torch.empty(1, 1, 196, d)
    return P


def vit_forward(P: Params, x: Tensor, *, mode: str = "base", training: bool = True, act: str = "gelu") -> Tensor:
    """VisionTransformer.forward for 224x224 inputs: conv stem (4x4 s4 p1 + BN + act, 2x2 s2 + BN + act, 2x2 s2 + bias; vit.py:90-121),
    tokens = cat(cls, patch + pos) (:476-507: no positional term on the cls token), N pre-norm encoders with LayerNorm eps 1e-6
    (:204-208), post_transformer_norm, classifier on the cls token (:545-560, :563-573)."""
    d, n, heads = VIT_MODES[mode]
    h = conv_layer_2d(P, "patch_emb.0", x, stride=4, training=training, act=act)
    h = conv_layer_2d(P, "patch_emb.1", h, stride=2, training=training, act=act)
    h = conv_layer_2d(P, "patch_emb.2", h, stride=2, use_norm=False, use_act=False)
    tok = h.flatten(2).transpose(1, 2)
    assert tok.shape[1] == P["pos_embed.pos_embed.pos_embed"].shape[2], "interpolated positional embeddings are out of scope"
    tok = tok + P["pos_embed.pos_embed.pos_embed"].reshape(1, tok.shape[1], d)
    tok = torch.cat((P["cls_token"].expand(x.shape[0], -1, -1), tok), dim=1)
    for i in range(n):
        tok = transformer_encoder(P, f"transformer.{i}", tok, heads, act=act, eps=1e-6)
    tok = layer_norm(P, "post_transformer_norm", tok, eps=1e-6)
    return F.linear(tok[:, 0], P["classifier.weight"], P["classifier.bias"])


# --------------------------------------------------------------------------------------------
# CLIP (cvnets/models/multi_modal_img_text/clip.py, cvnets/text_encoders/transformer.py:23-440,
# image_projection_layers/simple_projection_head.py, loss_fn/multi_modal_img_text/contrastive_loss_clip.py:56-97)
# --------------------------------------------------------------------------------------------
def clip_shapes(vit_mode: str = "base", proj: int = 512, text_dim: int = 512, text_layers: int = 12, vocab: int = 49408, ctx: int = 77) -> Dict[str, Tensor]:
    P: Dict[str, Tensor] = {"logit_scale": torch.empty(())}
    for k, v in vit_shapes(vit_mode).items():
        if not k.startswith("classifier."):
            P["image_encoder." + k] = v
    P["image_encoder.classifier.proj"] = torch.empty(VIT_MODES[vit_mode][0], proj)
    P["text_encoder.projection_layer"] = torch.empty(text_dim, proj)
    P["text_encoder.embedding_layer.weight"] = torch.empty(vocab, text_dim)
    P["text_encoder.positional_embedding.pos_embed.pos_embed"] = torch.empty(1, 1, ctx, text_dim)
    for i in range(text_layers):
        transformer_encoder_shapes(P, f"text_encoder.transformer.{i}", text_dim, int(math.ceil(text_dim * 4.0 / 16.0) * 16.0))
    _gn(P, "text_encoder.final_layer_norm", text_dim)
    return P


def clip_forward(P: Params, images: Tensor, tokens: Tensor, *, vit_mode: str = "base", text_layers: int = 12, text_heads: int = 8,
                 training: bool = True) -> Tuple[Tensor, Tensor]:
    """CLIP.forward (clip.py:144-215): L2-normalised image features (ViT cls embedding @ proj) and text features (embedding + positional
    embedding -> causal pre-norm encoders with LayerNorm eps 1e-5 and the model-wide activation -> final LayerNorm -> end-of-text token
    @ projection_layer); transformer.py:328-425."""
    Pi = {k[len("image_encoder."):]: v for k, v in P.items() if k.startswith("image_encoder.")}
    d, n, heads = VIT_MODES[vit_mode]
    h = conv_layer_2d(Pi, "patch_emb.0", images, stride=4, training=training, act="gelu")
    h = conv_layer_2d(Pi, "patch_emb.1", h, stride=2, training=training, act="gelu")
    h = conv_layer_2d(Pi, "patch_emb.2", h, stride=2, use_norm=False, use_act=False)
    tok = h.flatten(2).transpose(1, 2) + Pi["pos_embed.pos_embed.pos_embed"].reshape(1, -1, d)
    tok = torch.cat((Pi["cls_token"].expand(images.shape[0], -1, -1), tok), dim=1)
    for i in range(n):
        tok = transformer_encoder(Pi, f"transformer.{i}", tok, heads, act="gelu", eps=1e-6)
    cls = layer_norm(Pi, "post_transformer_norm", tok, eps=1e-6)[:, 0]
    img = F.normalize(cls @ Pi["classifier.proj"], dim=-1)
    S = tokens.shape[1]
    t = F.embedding(tokens, P["text_encoder.embedding_layer.weight"]) + P["text_encoder.positional_embedding.pos_embed.pos_embed"].reshape(1, S, -1)
    mask = torch.full((S, S), float("-inf"), device=t.device).triu_(1).unsqueeze(0).expand(tokens.shape[0], -1, -1)
    for i in range(text_layers):
        t = transformer_encoder(P, f"text_encoder.transformer.{i}", t, text_heads, act="gelu", eps=1e-5, attn_mask=mask)
    t = layer_norm(P, "text_encoder.final_layer_norm", t, eps=1e-5)
    t = t[torch.arange(tokens.shape[0]), tokens.argmax(dim=-1)] @ P["text_encoder.projection_layer"]
    return img, F.normalize(t, dim=-1)


def clip_loss(img: Tensor, txt: Tensor, logit_scale: Tensor) -> Tensor:
    """ContrastiveLossClip._forward_clip on one rank (contrastive_loss_clip.py:56-97)."""
    s = torch.clamp(logit_scale.exp(), 0, 100.0)
    labels = torch.arange(img.shape[0], device=img.device)
    return 0.5 * (F.cross_entropy(s * img @ txt.t(), labels) + F.cross_entropy(s * txt @ img.t(), labels))


# --------------------------------------------------------------------------------------------
# parameter construction (shape contract: SURVEY.md App. B) + deterministic seeding used by the golden files
# --------------------------------------------------------------------------------------------
def _conv_bn(P: Dict, pre: str, cin: int, cout: int, k: int, groups: int = 1, norm: bool = True, bias: bool = False):
    P[pre + ".block.conv.weight"] = torch.empty(cout, cin // groups, k, k)
    if bias:
        P[pre + ".block.conv.bias"] = torch.empty(cout)
    if norm:
        P[pre + ".block.norm.weight"] = torch.empty(cout)
        P[pre + ".block.norm.bias"] = torch.empty(cout)
        P[pre + ".block.norm.running_mean"] = torch.empty(cout)
        P[pre + ".block.norm.running_var"] = torch.empty(cout)
        P[pre + ".block.norm.num_batches_tracked"] = torch.zeros((), dtype=torch.long)


def inverted_residual_shapes(P: Dict, pre: str, cin: int, cout: int, expand_ratio: float = 2):
    hid = make_divisible(int(round(cin * expand_ratio)), 8)  # mobilenetv2.py:176
    if expand_ratio != 1:
        _conv_bn(P, pre + ".block.exp_1x1", cin, hid, 1)
    _conv_bn(P, pre + ".block.conv_3x3", hid, hid, 3, groups=hid)
    _conv_bn(P, pre + ".block.red_1x1", hid, cout, 1)


def inverted_residual_se_shapes(P: Dict, pre: str, cin: int, cout: int, expand_ratio: float, use_se: bool = True, kernel_size: int = 3,
                                squeeze_factor: int = 4):
    hid = make_divisible(int(round(cin * expand_ratio)), 8)  # mobilenetv2.py:56
    if expand_ratio != 1:
        _conv_bn(P, pre + ".block.exp_1x1", cin, hid, 1)
    _conv_bn(P, pre + ".block.conv_3x3", hid, hid, kernel_size, groups=hid)
    if use_se:
        sq = max(make_divisible(hid // squeeze_factor, 8), 32)  # squeeze_excitation.py:43-44
        _conv_bn(P, pre + ".block.se.se_layer.fc1", hid, sq, 1, norm=False, bias=True)
        _conv_bn(P, pre + ".block.se.se_layer.fc2", sq, hid, 1, norm=False, bias=True)
    _conv_bn(P, pre + ".block.red_1x1", hid, cout, 1)


def _gn(P: Dict, pre: str, c: int):
    P[pre + ".weight"] = torch.empty(c)
    P[pre + ".bias"] = torch.empty(c)


def _linear(P: Dict, pre: str, cin: int, cout: int):
    P[pre + ".weight"] = torch.empty(cout, cin)
    P[pre + ".bias"] = torch.empty(cout)


def multi_head_attention_shapes(P: Dict, pre: str, c: int):
    _linear(P, pre + ".qkv_proj", c, 3 * c)
    _linear(P, pre + ".out_proj", c, c)


def transformer_encoder_shapes(P: Dict, pre: str, c: int, ffn: int):
    _gn(P, pre + ".pre_norm_mha.0", c)
    multi_head_attention_shapes(P, pre + ".pre_norm_mha.1", c)
    _gn(P, pre + ".pre_norm_ffn.0", c)
    _linear(P, pre + ".pre_norm_ffn.1", c, ffn)
    _linear(P, pre + ".pre_norm_ffn.4", ffn, c)


def linear_attn_ffn_shapes(P: Dict, pre: str, d: int, ffn: int):
    _gn(P, pre + ".pre_norm_attn.0", d)
    _conv_bn(P, pre + ".pre_norm_attn.1.qkv_proj", d, 1 + 2 * d, 1, norm=False, bias=True)
    _conv_bn(P, pre + ".pre_norm_attn.1.out_proj", d, d, 1, norm=False, bias=True)
    _gn(P, pre + ".pre_norm_ffn.0", d)
    _conv_bn(P, pre + ".pre_norm_ffn.1", d, ffn, 1, norm=False, bias=True)
    _conv_bn(P, pre + ".pre_norm_ffn.3", ffn, d, 1, norm=False, bias=True)


def mobilevit_block_v2_shapes(P: Dict, pre: str, c: int, d: int, n_attn_blocks: int, ffn_multiplier: float = 2.0):
    _conv_bn(P, pre + ".local_rep.0", c, c, 3, groups=c)
    _conv_bn(P, pre + ".local_rep.1", c, d, 1, norm=False)
    ffn = int((ffn_multiplier * d) // 16 * 16)  # mobilevit_block.py:475
    for i in range(n_attn_blocks):
        linear_attn_ffn_shapes(P, f"{pre}.global_rep.{i}", d, ffn)
    _gn(P, f"{pre}.global_rep.{n_attn_blocks}", d)
    _conv_bn(P, pre + ".conv_proj", d, c, 1)


def mobilevit_v2_shapes(width_multiplier: float = 1.0, n_classes: int = 1000) -> Dict[str, Tensor]:
    cfg = mobilevit_v2_config(width_multiplier)
    P: Dict[str, Tensor] = {}
    c = cfg["layer0"]["out_channels"]
    _conv_bn(P, "conv_1", 3, c, 3)
    for li in range(1, 6):
        lc = cfg[f"layer{li}"]
        co = lc["out_channels"]
        if lc["block_type"] == "mv2":
            for i in range(lc["num_blocks"]):
                inverted_residual_shapes(P, f"layer_{li}.{i}", c, co, lc["expand_ratio"])
                c = co
        else:
            inverted_residual_shapes(P, f"layer_{li}.0", c, co, lc["mv_expand_ratio"])
            c = co
            mobilevit_block_v2_shapes(P, f"layer_{li}.1", c, lc["attn_unit_dim"], lc["attn_blocks"], lc["ffn_multiplier"])
    P["classifier.1.weight"] = torch.empty(n_classes, c)
    P["classifier.1.bias"] = torch.empty(n_classes)
    return P


def seeded_fill_(P: Dict[str, Tensor], seed: int) -> Dict[str, Tensor]:
    """Deterministic, reference-independent parameter values (CPU generator, sorted key order) so the golden
    fixtures only need to store outputs.  Non-trivial BN/GN affine and running stats on purpose."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    for k in sorted(P.keys()):
        t = P[k]
        if k.endswith("num_batches_tracked"):
            t.zero_()
        elif k.endswith("running_mean"):
            t.copy_(0.1 * torch.randn(t.shape, generator=g))
        elif k.endswith("running_var"):
            t.copy_(1.0 + 0.2 * torch.rand(t.shape, generator=g))
        elif k == "logit_scale":
            t.fill_(math.log(1.0 / 0.07))
        elif k.endswith("cls_token") or k.endswith("pos_embed.pos_embed") or k.endswith("embedding_layer.weight"):
            t.copy_(0.05 * torch.randn(t.shape, generator=g))
        elif t.dim() == 1 and k.endswith(".weight"):  # BN / GN gamma
            t.copy_(1.0 + 0.2 * torch.randn(t.shape, generator=g))
        elif t.dim() == 1:  # biases, beta
            t.copy_(0.1 * torch.randn(t.shape, generator=g))
        else:
            fan_in = t[0].numel()
            t.copy_(torch.randn(t.shape, generator=g) * (1.0 / math.sqrt(fan_in)))
    return P


def seeded_input(shape, seed: int) -> Tensor:
    g = torch.Generator(device="cpu").manual_seed(seed)
    return torch.randn(shape, generator=g)


def clone_params(P: Params, requires_grad: bool = True, device=None, dtype=None) -> Params:
    out = {}
    for k, v in P.items():
        v = v.detach().clone()
        if device is not None:
            v = v.to(device)
        if v.is_floating_point():
            if dtype is not None:
                v = v.to(dtype)
            is_buffer = k.endswith("running_mean") or k.endswith("running_var")
            v.requires_grad_(requires_grad and not is_buffer)
        out[k] = v
    return out


# --------------------------------------------------------------------------------------------
# the training step the metric is quoted on (SURVEY.md 8d): fwd + CE(label_smoothing=0.1) + bwd + AdamW
# --------------------------------------------------------------------------------------------
def training_step(P: Params, opt: Optional[torch.optim.Optimizer], x: Tensor, y: Tensor, width_multiplier: float = 1.0):
    """One reference-style step: engine/training_engine.py:257-307 restated without AMP (CPU refuses AMP,
    engine/utils.py:31-32).  Returns the loss value."""
    logits = mobilevit_v2_forward(P, x, width_multiplier=width_multiplier, training=True)
    loss = F.cross_entropy(logits, y, label_smoothing=0.1)  # loss_fn/classification/cross_entropy.py:19-95
    if opt is not None:
        opt.zero_grad(set_to_none=True)
    loss.backward()
    if opt is not None:
        opt.step()
    return float(loss.detach())

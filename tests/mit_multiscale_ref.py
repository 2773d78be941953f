"""MobileViT-v1 at the variable-batch sampler's crops: the fp32 oracle with the reference's bilinear resize in unfolding / folding, and the
recipe's (crop, batch) table.

``oracle.cvnets_oracle.mobilevit_block_v1`` unfolds maps whose sides are multiples of the patch.  At the recipe crops 160 and 288 the stride-32
map is 5x5 and 9x9: the reference (cvnets/modules/mobilevit_block.py:186-267) then resizes it up to the next multiple with
``F.interpolate(mode="bilinear", align_corners=False)`` before unfolding, and the folded map back down afterwards.  ``mobilevit_v1_forward``
here is the oracle's forward with that resize; at multiples of the patch it computes exactly what the oracle does."""
import math

import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O

PATCH, HEADS = 2, 4
# variable_batch_pairs(256, 256, 128, 5, 32, 160, 320, 160, 320): the sampler of every MobileViT-v1 recipe (crop 256, batch 128, 5 scales
# from 160 to 320, check_scale 32); tests/test_mobilevit_v1_multiscale_cpu.py checks it against the library's own sampler
RECIPE_PAIRS = [(160, 327), (192, 227), (256, 128), (288, 101), (320, 81)]
# MobileViT-S at 192 has 144 tokens of width 144 in layer 3: the reference's LayerNorm takes its channel-first branch there, which the
# library refuses (TransformerEncoder.prepare), so S trains on the other four pairs
S_PAIRS = [p for p in RECIPE_PAIRS if p[0] != 192]
# the fixtures tests/golden/make_golden_mit_multiscale.py writes: (mode, crop)
FIXTURES = [("xx_small", 160), ("xx_small", 288), ("xx_small", 320), ("x_small", 320), ("small", 160), ("small", 320)]


def fixture_name(mode, crop):
    return f"mobilevit_v1_{mode}_{crop}_fp32.pt"


def unfold(fm, patch=PATCH):
    """MobileViTBlock.unfolding: [B, d, H, W] -> [B*P, N, d] tokens of the map resized up to multiples of the patch, and the info to fold"""
    B, d, H, W = fm.shape
    Hn, Wn = math.ceil(H / patch) * patch, math.ceil(W / patch) * patch
    if (Hn, Wn) != (H, W):
        fm = F.interpolate(fm, size=(Hn, Wn), mode="bilinear", align_corners=False)
    nh, nw = Hn // patch, Wn // patch
    t = fm.reshape(B * d * nh, patch, nw, patch).transpose(1, 2).reshape(B, d, nh * nw, patch * patch).transpose(1, 3)
    return t.reshape(B * patch * patch, nh * nw, d), (B, d, H, W, Hn, Wn)


def fold(t, info, patch=PATCH):
    """MobileViTBlock.folding: the inverse reshapes, then the resize back to the original map size"""
    B, d, H, W, Hn, Wn = info
    nh, nw = Hn // patch, Wn // patch
    t = t.contiguous().view(B, patch * patch, nh * nw, d).transpose(1, 3)
    fm = t.reshape(B * d * nh, nw, patch, patch).transpose(1, 2).reshape(B, d, Hn, Wn)
    if (Hn, Wn) != (H, W):
        fm = F.interpolate(fm, size=(H, W), mode="bilinear", align_corners=False)
    return fm


def mobilevit_block_v1(P, pre, x, *, n_blocks, num_heads=HEADS, training=True):
    """oracle.cvnets_oracle.mobilevit_block_v1 with the resize of unfolding / folding"""
    res = x
    fm = O.conv_layer_2d(P, pre + ".local_rep.conv_3x3", x, training=training)
    fm = O.conv_layer_2d(P, pre + ".local_rep.conv_1x1", fm, use_norm=False, use_act=False)
    t, info = unfold(fm)
    for i in range(n_blocks):
        t = O.transformer_encoder(P, f"{pre}.global_rep.{i}", t, num_heads, act="swish", eps=1e-5)
    t = O.layer_norm(P, f"{pre}.global_rep.{n_blocks}", t, eps=1e-5)
    fm = fold(t, info)
    fm = O.conv_layer_2d(P, pre + ".conv_proj", fm, training=training)
    return O.conv_layer_2d(P, pre + ".fusion", torch.cat((res, fm), dim=1), training=training)


def mobilevit_v1_forward(P, x, *, mode="xx_small", training=True):
    """oracle.cvnets_oracle.mobilevit_v1_forward at any crop"""
    for kind, pre, kw in O.mobilevit_v1_layout(mode):
        if kind == "stem":
            x = O.conv_layer_2d(P, pre, x, stride=2, training=training)
        elif kind == "ir":
            x = O.inverted_residual(P, pre, x, stride=kw["stride"], training=training)
        elif kind == "mvit":
            x = mobilevit_block_v1(P, pre, x, n_blocks=kw["n_blocks"], training=training)
        else:
            x = O.conv_layer_2d(P, pre, x, training=training)
    return F.linear(x.mean(dim=[-2, -1]), P["classifier.fc.weight"], P["classifier.fc.bias"])


def blocks(mode, crop):
    """(layer, map side H, tokens N, transformer dim d, head dim) of each MobileViTBlock at ``crop``"""
    shapes = O.mobilevit_v1_shapes(mode)
    out = []
    for kind, pre, _ in O.mobilevit_v1_layout(mode):
        if kind != "mvit":
            continue
        li = int(pre.split("_")[1].split(".")[0])
        d = shapes[pre + ".local_rep.conv_1x1.block.conv.weight"].shape[0]
        H = crop
        for _ in range(li):  # the stem and each stride-2 stage: ceil halving (3x3, pad 1)
            H = (H - 1) // 2 + 1
        N = (math.ceil(H / PATCH)) ** 2
        out.append((li, H, N, d, d // HEADS))
    return out

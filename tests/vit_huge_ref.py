"""fp32 restatement of the ViT-H/16 classifier (cvnets/models/classification/config/vit.py "huge": 1280 wide, 32 layers, 20 heads of 64),
built from the oracle's pieces (oracle/cvnets_oracle.py).  The oracle's ``vit_shapes`` / ``vit_forward`` cover the tiny / small / base
geometries; this is the same parameter tree and forward at the huge one, with the positional table resized as the reference resizes it
(tests/vit_multiscale_ref.py), so any input whose sides are multiples of 16 works."""
from typing import Dict

import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O
from vit_multiscale_ref import vit_pos_embed

D, LAYERS, HEADS = 1280, 32, 20


def vit_huge_shapes(n_classes: int = 1000) -> Dict[str, torch.Tensor]:
    """The reference's state_dict keys and shapes of VisionTransformer(mode="huge")."""
    stem = max(32, D // 4)
    P: Dict[str, torch.Tensor] = {"cls_token": torch.empty(1, 1, D)}
    O._conv_bn(P, "patch_emb.0", 3, stem, 4)
    O._conv_bn(P, "patch_emb.1", stem, stem, 2)
    O._conv_bn(P, "patch_emb.2", stem, D, 2, norm=False, bias=True)
    O._gn(P, "post_transformer_norm", D)
    for i in range(LAYERS):
        O.transformer_encoder_shapes(P, f"transformer.{i}", D, 4 * D)
    O._linear(P, "classifier", D, n_classes)
    P["pos_embed.pos_embed.pos_embed"] = torch.empty(1, 1, 196, D)
    return P


def vit_huge_forward(P, x: torch.Tensor, *, training: bool = True, act: str = "gelu") -> torch.Tensor:
    """vit.py:476-573 at the huge geometry (checkpointing changes what is stored, not what is computed)."""
    h = O.conv_layer_2d(P, "patch_emb.0", x, stride=4, training=training, act=act)
    h = O.conv_layer_2d(P, "patch_emb.1", h, stride=2, training=training, act=act)
    h = O.conv_layer_2d(P, "patch_emb.2", h, stride=2, use_norm=False, use_act=False)
    tok = h.flatten(2).transpose(1, 2)
    tok = tok + vit_pos_embed(P["pos_embed.pos_embed.pos_embed"], tok.shape[1])
    tok = torch.cat((P["cls_token"].expand(x.shape[0], -1, -1), tok), dim=1)
    for i in range(LAYERS):
        tok = O.transformer_encoder(P, f"transformer.{i}", tok, HEADS, act=act, eps=1e-6)
    tok = O.layer_norm(P, "post_transformer_norm", tok, eps=1e-6)
    return F.linear(tok[:, 0], P["classifier.weight"], P["classifier.bias"])

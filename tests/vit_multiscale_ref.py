"""fp32 restatement of VisionTransformer.forward at ANY input size, built from the oracle's pieces (oracle/cvnets_oracle.py).

``oracle.vit_forward`` covers 224 x 224 only.  At other sizes the reference resizes its 196-entry positional table with
F.interpolate(size=(N, C), mode="bilinear", align_corners=False) (cvnets/layers/positional_embedding.py:90-95): a 1-D linear resample of
the flattened patch index.  ``vit_forward_any_size`` does exactly that and is otherwise the oracle's ViT forward."""
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O


def vit_pos_embed(pe: torch.Tensor, n: int) -> torch.Tensor:
    """LearnablePositionalEmbedding.forward (positional_embedding.py:84-103): the [1, 1, n_pos, C] table as [1, n, C], resized when n != n_pos."""
    if n != pe.shape[2]:
        pe = F.interpolate(pe, size=(n, pe.shape[3]), mode="bilinear")
    return pe.reshape(1, n, pe.shape[3])


def vit_forward_any_size(P, x: torch.Tensor, *, mode: str = "base", training: bool = True, act: str = "gelu") -> torch.Tensor:
    """vit.py:476-573 for inputs whose sides are multiples of 16 (square or not); identical to oracle.vit_forward at 224 x 224."""
    d, n, heads = O.VIT_MODES[mode]
    h = O.conv_layer_2d(P, "patch_emb.0", x, stride=4, training=training, act=act)
    h = O.conv_layer_2d(P, "patch_emb.1", h, stride=2, training=training, act=act)
    h = O.conv_layer_2d(P, "patch_emb.2", h, stride=2, use_norm=False, use_act=False)
    tok = h.flatten(2).transpose(1, 2)
    tok = tok + vit_pos_embed(P["pos_embed.pos_embed.pos_embed"], tok.shape[1])
    tok = torch.cat((P["cls_token"].expand(x.shape[0], -1, -1), tok), dim=1)
    for i in range(n):
        tok = O.transformer_encoder(P, f"transformer.{i}", tok, heads, act=act, eps=1e-6)
    tok = O.layer_norm(P, "post_transformer_norm", tok, eps=1e-6)
    return F.linear(tok[:, 0], P["classifier.weight"], P["classifier.bias"])

"""fp32 restatement of CLIP zero-shot evaluation from the oracle's pieces (cvnets/text_encoders/transformer.py:354-504,
cvnets/models/multi_modal_img_text/clip.py:184-202), for any causal prefix of the text rows.  Pinned to the real reference by
tests/test_clip_zeroshot_cpu.py against tests/golden/clip_zeroshot_fp32.pt."""
from typing import Optional

import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O


def image_features(P, images, *, vit_mode="small", training=False):
    """L2-normalised image features: the image half of oracle.clip_forward (eval-mode BatchNorm by default)."""
    Pi = {k[len("image_encoder."):]: v for k, v in P.items() if k.startswith("image_encoder.")}
    d, n, heads = O.VIT_MODES[vit_mode]
    h = O.conv_layer_2d(Pi, "patch_emb.0", images, stride=4, training=training, act="gelu")
    h = O.conv_layer_2d(Pi, "patch_emb.1", h, stride=2, training=training, act="gelu")
    h = O.conv_layer_2d(Pi, "patch_emb.2", h, stride=2, use_norm=False, use_act=False)
    tok = h.flatten(2).transpose(1, 2) + Pi["pos_embed.pos_embed.pos_embed"].reshape(1, -1, d)
    tok = torch.cat((Pi["cls_token"].expand(images.shape[0], -1, -1), tok), dim=1)
    for i in range(n):
        tok = O.transformer_encoder(Pi, f"transformer.{i}", tok, heads, act="gelu", eps=1e-6)
    cls = O.layer_norm(Pi, "post_transformer_norm", tok, eps=1e-6)[:, 0]
    return F.normalize(cls @ Pi["classifier.proj"], dim=-1)


def text_projected(P, tokens, *, text_layers=4, text_heads=4, length: Optional[int] = None):
    """end-of-text features @ projection_layer of [R, L] tokens, NOT normalised.  ``length``: run only the first ``length`` tokens of every
    row (each row's end-of-text token must lie inside), with the first ``length`` rows of the positional table and a causal mask."""
    S = tokens.shape[1] if length is None else length
    tokens = tokens[:, :S]
    pe = P["text_encoder.positional_embedding.pos_embed.pos_embed"]
    t = F.embedding(tokens, P["text_encoder.embedding_layer.weight"]) + pe[:, :, :S].reshape(1, S, -1)
    mask = torch.full((S, S), float("-inf"), device=t.device).triu_(1).unsqueeze(0).expand(tokens.shape[0], -1, -1)
    for i in range(text_layers):
        t = O.transformer_encoder(P, f"text_encoder.transformer.{i}", t, text_heads, act="gelu", eps=1e-5, attn_mask=mask)
    t = O.layer_norm(P, "text_encoder.final_layer_norm", t, eps=1e-5)
    return t[torch.arange(tokens.shape[0]), tokens.argmax(dim=-1)] @ P["text_encoder.projection_layer"]


def text_features(P, tokens, **kw):
    """[B, L] -> [B, d]; [B, N, L] -> [B, N, d] (transformer.py:506-549)."""
    if tokens.dim() == 3:
        b, n, L = tokens.shape
        return text_features(P, tokens.reshape(b * n, L), **kw).view(b, n, -1)
    return F.normalize(text_projected(P, tokens, **kw), dim=-1)


def zero_shot_table(P, tokens, **kw):
    """[B, Cl, M, L] prompts -> fp32 [d, Cl]: the first batch element's captions, normalised, averaged per class, normalised again."""
    _, Cl, M, L = tokens.shape
    f = text_features(P, tokens[0].reshape(Cl * M, L), **kw).view(Cl, M, -1)
    return F.normalize(f.mean(dim=1), dim=-1).t().contiguous()

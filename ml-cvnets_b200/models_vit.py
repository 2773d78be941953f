"""VisionTransformer assembler (mirror of cvnets/models/classification/vit.py:33-649 for the classification path): conv-stem patch embedding
-> [cls] + positional embedding -> N x TransformerEncoder -> LayerNorm -> classifier on the cls token (or the token mean).

Host code like the MobileViTv2 assembler: same attribute names / ``state_dict`` keys as the reference (``patch_emb.{0,1,2}.block.*``,
``cls_token``, ``pos_embed.pos_embed.pos_embed``, ``transformer.{i}.*``, ``post_transformer_norm.*``, ``classifier.*``), every forward /
backward kernel is the library's.  BASELINE.json configs[2]: ViT-B/16, bf16, 224x224 (examples/vit/classification/vit_base.yaml).
Any input resolution whose sides are multiples of 16 works, square or not (the multi-scale recipes feed 128-320 px crops): when the patch
grid does not hold the table's 196 entries, the positional table is linearly resampled in the token-assembly kernel exactly as the
reference's F.interpolate does (cvnets/layers/positional_embedding.py:90-95), and sequences over 256 tokens run on the streaming attention
kernels (every ViT mode has head_dim 64).  With ``model.classification.gradient_checkpointing`` (the ViT-H recipes), training splits the
encoder stack as torch's checkpoint_sequential does for the reference (vit.py:526-533) into ``model.classification.vit.checkpoint_segments``
segments; the first segments - 1 runs keep only their input and are recomputed in the backward (modules.checkpointed_encoders), the
remaining layers run normally.  The option does nothing in eval mode.  Not implemented (raises): SimpleFPN (detection), sinusoidal
positional embeddings, output_stride, attention-probability dropout > 0 in training.
"""
from __future__ import annotations

import argparse
from types import SimpleNamespace
from typing import Dict, Tuple

import numpy as np
import torch
from torch import Tensor, nn

from . import functional as Fn
from . import ops
from .layers import ConvLayer2d, Dropout, LinearLayer, _bind, get_normalization_layer
from .models_base import ImageEncoder, init_weights
from .modules import TransformerEncoder, checkpointed_encoders


def default_vit_opts(mode: str = "base", n_classes: int = 1000, **extra) -> argparse.Namespace:
    """The recipe's model options (examples/vit/classification/vit_base.yaml:80-97; the ViT-H recipes set gradient_checkpointing)."""
    kv = {
        "model.classification.name": "vit", "model.classification.n_classes": n_classes, "model.classification.vit.mode": mode,
        "model.classification.vit.norm_layer": "layer_norm_fp32", "model.classification.vit.dropout": 0.0,
        "model.classification.vit.stochastic_dropout": 0.0, "model.classification.vit.no_cls_token": False,
        "model.classification.vit.sinusoidal_pos_emb": False, "model.classification.vit.use_simple_fpn": False,
        "model.classification.gradient_checkpointing": False, "model.classification.vit.checkpoint_segments": 4,
        "model.activation.name": "gelu", "model.normalization.name": "batch_norm", "model.normalization.momentum": 0.1,
        "model.layer.conv_init": "kaiming_normal", "model.layer.linear_init": "trunc_normal", "model.layer.linear_init_std_dev": 0.02,
    }
    return argparse.Namespace(**{**kv, **extra})


def get_vit_configuration(opts) -> Dict:
    """cvnets/models/classification/config/vit.py:12-116."""
    mode = getattr(opts, "model.classification.vit.mode", "base").lower()
    dropout = getattr(opts, "model.classification.vit.dropout", 0.0)
    norm_layer = getattr(opts, "model.classification.vit.norm_layer", "layer_norm")
    dims = {"tiny": (192, 12, 3), "small": (384, 12, 6), "base": (768, 12, 12), "large": (1024, 24, 16), "huge": (1280, 32, 20)}
    if mode not in dims:
        raise NotImplementedError(f"ViT mode {mode}")
    d, n, h = dims[mode]
    return {"embed_dim": d, "n_transformer_layers": n, "n_attn_heads": h, "ffn_dim": d * 4, "norm_layer": norm_layer, "pos_emb_drop_p": 0.1 if mode == "tiny" else 0.0,
            "attn_dropout": 0.0, "ffn_dropout": 0.0, "dropout": dropout}


class LearnablePositionalEmbedding(nn.Module):
    """cvnets/layers/positional_embedding.py:53-110: parameter ``pos_embed`` [1, 1, num_embeddings, C], trunc-normal(0.02) initialised."""

    def __init__(self, num_embeddings: int, embedding_dim: int):
        super().__init__()
        self.pos_embed = nn.Parameter(torch.empty(1, 1, num_embeddings, embedding_dim))
        self.num_embeddings, self.embedding_dim = num_embeddings, embedding_dim
        nn.init.trunc_normal_(self.pos_embed, mean=0, std=embedding_dim ** -0.5)


class PositionalEmbedding(nn.Module):
    """cvnets/layers/positional_embedding.py:17-50 (learnable variant only)."""

    def __init__(self, opts, num_embeddings: int, embedding_dim: int, is_learnable: bool = True, *args, **kwargs):
        super().__init__()
        if not is_learnable:
            raise NotImplementedError("sinusoidal positional embeddings are not implemented")
        self.pos_embed = LearnablePositionalEmbedding(num_embeddings, embedding_dim)


class VisionTransformer(ImageEncoder):
    def __init__(self, opts, *args, **kwargs) -> None:
        super().__init__(opts)
        num_classes = getattr(opts, "model.classification.n_classes", 1000)
        if getattr(opts, "model.classification.vit.use_simple_fpn", False):
            raise NotImplementedError("SimpleFPN (detection) is out of scope")
        cfg = get_vit_configuration(opts)
        d, ffn, n_layers, heads, norm_layer = cfg["embed_dim"], cfg["ffn_dim"], cfg["n_transformer_layers"], cfg["n_attn_heads"], cfg["norm_layer"]
        stem_dim = max(32, d // 4)
        self.patch_emb = nn.Sequential(
            ConvLayer2d(opts=opts, in_channels=3, out_channels=stem_dim, kernel_size=4, stride=4, bias=False, use_norm=True, use_act=True),
            ConvLayer2d(opts=opts, in_channels=stem_dim, out_channels=stem_dim, kernel_size=2, stride=2, bias=False, use_norm=True, use_act=True),
            ConvLayer2d(opts=opts, in_channels=stem_dim, out_channels=d, kernel_size=2, stride=2, bias=True, use_norm=False, use_act=False))
        sd = getattr(opts, "model.classification.vit.stochastic_dropout", 0.0)
        per_layer_sd = [round(float(v), 3) for v in np.linspace(0, sd, n_layers)]  # vit.py:129-132
        self.post_transformer_norm = get_normalization_layer(opts=opts, num_features=d, norm_type=norm_layer)
        self.transformer = nn.Sequential(*[
            TransformerEncoder(opts=opts, embed_dim=d, ffn_latent_dim=ffn, num_heads=heads, attn_dropout=cfg["attn_dropout"], dropout=cfg["dropout"],
                               ffn_dropout=cfg["ffn_dropout"], transformer_norm_layer=norm_layer, stochastic_dropout=per_layer_sd[i]) for i in range(n_layers)])
        self.classifier = LinearLayer(d, num_classes)
        self.reset_parameters(opts)
        if not getattr(opts, "model.classification.vit.no_cls_token", False):
            self.cls_token = nn.Parameter(torch.zeros(size=(1, 1, d)))
            nn.init.trunc_normal_(self.cls_token, std=0.02)
        else:
            self.cls_token = None
        self.pos_embed = PositionalEmbedding(opts=opts, num_embeddings=(224 // 16) ** 2, embedding_dim=d,
                                             is_learnable=not getattr(opts, "model.classification.vit.sinusoidal_pos_emb", False))
        self.emb_dropout = Dropout(p=cfg["pos_emb_drop_p"])
        self.embed_dim = d
        self.model_conf_dict = {"conv1": {"in": 3, "out": d}, "cls": {"in": d, "out": num_classes}}
        for m in self.modules():  # update_layer_norm_eps (vit.py:204-208)
            if isinstance(m, nn.LayerNorm):
                m.eps = 1e-6
        self._tok = SimpleNamespace()
        self.gradient_checkpointing = bool(getattr(opts, "model.classification.gradient_checkpointing", False))
        self.checkpoint_segments = int(getattr(opts, "model.classification.vit.checkpoint_segments", 4))
        if self.gradient_checkpointing and not 1 <= self.checkpoint_segments <= n_layers:
            raise ValueError(f"checkpoint_segments must be in 1..{n_layers}, got {self.checkpoint_segments}")

    def reset_parameters(self, opts) -> None:
        """cvnets/misc/init_utils.py:110-150."""
        init_weights(self.modules(), "kaiming_normal", "trunc_normal", getattr(opts, "model.layer.linear_init_std_dev", 0.02))

    # ---- forward (vit.py:476-560)
    def extract_patch_embeddings(self, x: Tensor) -> Tuple[Tensor, Tuple[int, int]]:
        patch = self.patch_emb(x)  # [B, d, nh, nw], channels-last == token-major [B*N, d]
        n_h, n_w = patch.shape[-2:]
        pe = self.pos_embed.pos_embed.pos_embed  # resampled to n_h * n_w rows inside the token kernel when the counts differ
        tok = _bind(self, self._tok, [pe] + ([self.cls_token] if self.cls_token is not None else []))
        # emb_dropout (vit.py: positional-embedding dropout, 0.1 in the 'tiny' config): hashed-mask kernel in training, identity otherwise
        return self.emb_dropout(Fn.VitTokensFn.apply(patch, tok, pe, self.cls_token)), (n_h, n_w)

    def extract_features(self, x: Tensor, *args, **kwargs) -> Tensor:
        x, _ = self.extract_patch_embeddings(x)
        if self.training and self.gradient_checkpointing and torch.is_grad_enabled():
            layers = list(self.transformer)
            size = len(layers) // self.checkpoint_segments  # torch.utils.checkpoint.checkpoint_sequential's split
            end = size * (self.checkpoint_segments - 1)
            for start in range(0, end, size):
                x = checkpointed_encoders(layers[start:start + size], x)
            for layer in layers[end:]:
                x = layer(x)
        else:
            x = self.transformer(x)
        # LayerNorm is per token, so normalising only the token the classifier reads equals the reference's norm-then-select
        x = x[:, 0] if self.cls_token is not None else None
        if x is None:
            raise NotImplementedError("no_cls_token (mean over tokens) is not implemented")
        return self.post_transformer_norm(x)

    def forward_classifier(self, x: Tensor, *args, **kwargs) -> Tensor:
        return self.classifier(self.extract_features(x))

"""CLIP (mirror of cvnets/models/multi_modal_img_text/clip.py, cvnets/text_encoders/transformer.py:23-440, image_projection_layers/
simple_projection_head.py and loss_fn/multi_modal_img_text/contrastive_loss_clip.py) -- BASELINE.json configs[4].

    model = CLIP(default_clip_opts())                    # ViT-B/16 image tower + 12-layer text transformer, projection 512
    img, txt, logit_scale = model(images, text_tokens)   # L2-normalised features
    loss = clip_contrastive_loss(img, txt, logit_scale)  # all-gather over the process group when distributed

    model.eval()                                         # zero-shot classification (transformer.py:428-504, clip.py:171-202)
    table = model.zero_shot_table(prompts)               # prompts [1, classes, captions, L] -> fp32 [d, classes]
    logits = model.zero_shot_logits(images, table)       # 100 * img @ table, fp32 [B, classes]
    acc = ZeroShotAccuracy(model, prompts)               # engine.py: top-1 / top-5 over an evaluation set, counted on the device

Same attribute names / ``state_dict`` keys as the reference (image_encoder.*, text_encoder.{embedding_layer, positional_embedding,
transformer.{i}, final_layer_norm, projection_layer}, logit_scale).  Host code only; every kernel is the library's.  3-D and 4-D text
batches are encoded at each caption's causal prefix (TextTransformer._encode_rows).  Not implemented: key_padding_mask with causal masking
off (beyond full-length encoding), sinusoidal embeddings, dropout > 0 in training.
"""
from __future__ import annotations

import argparse
import math
from types import SimpleNamespace
from typing import Optional, Tuple

import torch
from torch import Tensor, nn

from . import functional as Fn
from . import ops
from .layers import Dropout, get_normalization_layer
from .models_vit import PositionalEmbedding, VisionTransformer, default_vit_opts
from .modules import TransformerEncoder, _require_cuda
from .ops import PreparedWeights as PW


def default_clip_opts(vit_mode: str = "base", projection_dim: int = 512, text_dim: int = 512, text_layers: int = 12, text_heads: int = 8,
                      vocab_size: int = 49408, context_length: int = 77, **extra) -> argparse.Namespace:
    """config/multi_modal_img_text/clip_vit.yaml model section."""
    opts = default_vit_opts(vit_mode)
    kv = {
        "model.multi_modal_image_text.name": "clip", "model.multi_modal_image_text.clip.projection_dim": projection_dim,
        "model.text.name": "transformer", "model.text.transformer.model_dim": text_dim, "model.text.transformer.n_transformer_layers": text_layers,
        "model.text.transformer.n_heads_per_layer": text_heads, "model.text.transformer.ffn_multiplier_per_layer": 4.0,
        "model.text.transformer.causal_masking": True, "model.text.transformer.norm_layer": "layer_norm_fp32",
        "model.text.transformer.dropout": 0.0, "model.text.transformer.attn_dropout": 0.0, "model.text.transformer.ffn_dropout": 0.0,
        "model.text.transformer.no_pos_embedding": False, "dataset.text_vocab_size": vocab_size, "dataset.text_context_length": context_length,
        "dataset.padding_index": None,
    }
    kv.update(extra)
    for k, v in kv.items():
        setattr(opts, k, v)
    return opts


class Embedding(nn.Embedding):
    """cvnets/layers/embedding.py."""

    def __init__(self, opts, num_embeddings: int, embedding_dim: int, padding_idx: Optional[int] = None, *args, **kwargs):
        super().__init__(num_embeddings=num_embeddings, embedding_dim=embedding_dim, padding_idx=padding_idx)


class _Projection(nn.Module):
    """Holder of the kernel-layout caches of an [in, out] projection parameter (the parameter itself stays on its owner)."""

    def __init__(self):
        super().__init__()
        self._cfg = None

    def apply_to(self, x: Tensor, P: nn.Parameter, owner: nn.Module) -> Tensor:
        if self._cfg is None:
            prep = PW()
            self._cfg = SimpleNamespace(prep=prep, i_p=prep.add(P, PW.KIND_ROWMAJOR), i_pt=prep.add(P, PW.KIND_TRANSPOSED))
        cfg = self._cfg
        cfg.ws, cfg.plist = getattr(owner, "_ws", None), [P]
        cfg.prep.prepare(force=owner.training)
        return Fn.ProjectionFn.apply(x, cfg, P)


class TextTransformer(nn.Module):
    def __init__(self, opts, projection_dim: int, *args, **kwargs) -> None:
        super().__init__()
        d = getattr(opts, "model.text.transformer.model_dim", 512)
        n_layers = getattr(opts, "model.text.transformer.n_transformer_layers", 6)
        heads = getattr(opts, "model.text.transformer.n_heads_per_layer", 8)
        mult = getattr(opts, "model.text.transformer.ffn_multiplier_per_layer", 4.0)
        norm_layer = getattr(opts, "model.text.transformer.norm_layer", "layer_norm")
        self.vocab_size = getattr(opts, "dataset.text_vocab_size")
        ctx_len = getattr(opts, "dataset.text_context_length")
        if getattr(opts, "dataset.padding_index", None) is not None:
            raise NotImplementedError("padding_idx is not implemented")
        self.projection_dim = projection_dim
        self.embedding_layer = Embedding(opts=opts, embedding_dim=d, padding_idx=None, num_embeddings=self.vocab_size)
        self.embed_scale = d ** -0.5
        no_pos = getattr(opts, "model.text.transformer.no_pos_embedding", False)
        self.positional_embedding = None if no_pos else PositionalEmbedding(opts=opts, num_embeddings=ctx_len, embedding_dim=d, is_learnable=True)
        self.embedding_dropout = Dropout(p=getattr(opts, "model.text.transformer.embed_dropout", 0.0))
        ffn_dims = [int(math.ceil(d * mult / 16.0) * 16.0)] * n_layers
        self.transformer = nn.ModuleList([
            TransformerEncoder(opts=opts, embed_dim=d, num_heads=heads, ffn_latent_dim=ffn_dims[i],
                               attn_dropout=getattr(opts, "model.text.transformer.attn_dropout", 0.0),
                               ffn_dropout=getattr(opts, "model.text.transformer.ffn_dropout", 0.0),
                               dropout=getattr(opts, "model.text.transformer.dropout", 0.0), transformer_norm_layer=norm_layer)
            for i in range(n_layers)])
        self.final_layer_norm = get_normalization_layer(opts, num_features=d, norm_type=norm_layer)
        self.projection_layer = nn.Parameter(torch.empty(d, projection_dim))
        self.model_dim = d
        self.causal_masking = getattr(opts, "model.text.transformer.causal_masking", False)
        self.classes_per_split_zero_shot = max(1, int(getattr(opts, "model.text.transformer.classes_per_split_zero_shot", 1)))
        self.zero_shot_token_budget = 1 << 18  # tokens per tower call when encoding 3-D / 4-D batches: bounds their activation memory
        self.reset_parameters_clip_style()
        self._emb = SimpleNamespace()
        self._proj = _Projection()
        self._mask = None

    def reset_parameters_clip_style(self):
        """transformer.py:181-211."""
        nn.init.normal_(self.embedding_layer.weight, mean=0.0, std=0.02)
        attn_std = self.model_dim ** -0.5
        proj_std = attn_std * ((2 * len(self.transformer)) ** -0.5)
        fc_std = (2 * self.model_dim) ** -0.5
        for block in self.transformer:
            nn.init.normal_(block.pre_norm_mha[1].qkv_proj.weight, mean=0.0, std=attn_std)
            nn.init.normal_(block.pre_norm_mha[1].out_proj.weight, mean=0.0, std=proj_std)
            nn.init.normal_(block.pre_norm_ffn[1].weight, mean=0.0, std=fc_std)
            nn.init.normal_(block.pre_norm_ffn[4].weight, mean=0.0, std=proj_std)
        nn.init.normal_(self.projection_layer, mean=0.0, std=attn_std)

    def build_attention_mask(self, context_length: int, batch_size: int, device) -> Tensor:
        """transformer.py:343-353: additive causal mask, -inf above the diagonal, expanded over the batch."""
        if self._mask is None or self._mask.shape[0] != batch_size or self._mask.shape[1] != context_length or self._mask.device != device:
            m = torch.full((context_length, context_length), float("-inf"), device=device).triu_(1)
            self._mask = m.unsqueeze(0).expand(batch_size, -1, -1).contiguous()
        return self._mask

    def forward(self, text_tokens: Tensor, key_padding_mask: Optional[Tensor] = None, *args, **kwargs) -> Tensor:
        """transformer.py:506-551: [B, L] -> [B, d] features; [B, N, L] (several captions per image) -> [B, N, d]; [B, Cl, M, L] (zero-shot
        prompts: M captions per class, eval mode only) -> the fp32 [d, Cl] class table of ``forward_zero_shot``."""
        _require_cuda(text_tokens, "TextTransformer")
        if text_tokens.dim() == 4:
            return self.forward_zero_shot(text_tokens, key_padding_mask)
        if text_tokens.dim() == 3:
            b, n, L = text_tokens.shape
            kpm = key_padding_mask.reshape(b * n, L) if key_padding_mask is not None else None
            if torch.is_grad_enabled():  # training on multi-caption batches: full length, the 2-D path's autograd
                return self.forward(text_tokens.reshape(b * n, L), kpm).view(b, n, -1)
            feats, where = self._encode_rows(text_tokens.reshape(b * n, L), kpm)
            return Fn.L2NormFn.apply(feats)[where].view(b, n, -1)
        if text_tokens.dim() != 2:
            raise NotImplementedError(f"text tokens of rank {text_tokens.dim()}: expected [B, L], [B, N, L] or [B, classes, captions, L]")
        pe = self._checked_pos_embed(text_tokens.shape[-1])
        return Fn.L2NormFn.apply(self._tower(text_tokens.contiguous(), pe, key_padding_mask))

    def _checked_pos_embed(self, L: int) -> Optional[Tensor]:
        if self.training and self.embedding_dropout.p > 0:
            raise NotImplementedError("embedding dropout > 0 in training mode is not implemented")
        pe = self.positional_embedding.pos_embed.pos_embed if self.positional_embedding is not None else None
        if pe is not None and pe.shape[2] != L:
            raise NotImplementedError("interpolated positional embeddings are not implemented (sequence length must equal the context length)")
        return pe

    def _tower(self, tokens: Tensor, pe: Optional[Tensor], key_padding_mask: Optional[Tensor]) -> Tensor:
        """transformer.py:354-423 up to the projection: bf16 [b, projection_dim] features of the end-of-text tokens, not yet normalised.
        ``pe`` holds the first tokens.shape[1] rows of the positional table."""
        emb = self._emb
        emb.ws, emb.plist = getattr(self, "_ws", None), [self.embedding_layer.weight] + ([pe] if pe is not None else [])
        x = Fn.EmbeddingFn.apply(tokens, emb, self.embedding_layer.weight, pe)
        attn_mask = None
        if self.causal_masking:
            attn_mask = self.build_attention_mask(tokens.shape[1], tokens.shape[0], tokens.device)
            key_padding_mask = None
        for layer in self.transformer:
            x = layer(x, key_padding_mask=key_padding_mask, attn_mask=attn_mask)
        x = Fn.EotGatherFn.apply(x, tokens)       # LayerNorm is per token: normalising only the gathered token equals norm-then-gather
        x = self.final_layer_norm(x)
        return self._proj.apply_to(x, self.projection_layer, self)

    @torch.no_grad()
    def _encode_rows(self, tokens: Tensor, key_padding_mask: Optional[Tensor]) -> Tuple[Tensor, Tensor]:
        """Encodes the rows of a [R, L] token matrix without autograd, in length-bucketed chunks of at most ``zero_shot_token_budget`` tokens.

        With causal masking the end-of-text feature depends only on tokens 0..eot: LayerNorm, the GEMMs and the FFN act per token and
        attention only looks back.  So each row runs at its own prefix length L' = eot + 1, rounded up to a multiple of 8 (fewer distinct
        lengths, hence fewer and larger tower calls), on the first L' rows of the positional table and an [L', L'] causal mask.  A chunk
        holds rows of one L' only, so a row's result does not depend on which other rows share its chunk, nor on the budget.  Without
        causal masking every row runs at full length (and the key-padding mask, if any, applies).

        Returns (features bf16 [R, projection_dim] before normalisation, in length-sorted order; where: int64 [R], the feature row of token
        row r)."""
        R, L = tokens.shape
        pe = self._checked_pos_embed(L)
        tokens = tokens.contiguous()
        if self.causal_masking:
            lengths = ((tokens.argmax(dim=-1) + 8) // 8 * 8).clamp_(max=L)
            order = torch.argsort(lengths, stable=True)
            counts = torch.bincount(lengths, minlength=L + 1).tolist()  # one host sync per table
            key_padding_mask = None
        else:
            order = torch.arange(R, device=tokens.device)
            counts = [0] * L + [R]
        where = torch.empty_like(order)
        where[order] = torch.arange(R, device=tokens.device)
        feats = torch.empty((R, self.projection_dim), device=tokens.device, dtype=torch.bfloat16)
        start = 0
        for Lp, n in enumerate(counts):
            rows = max(1, self.zero_shot_token_budget // max(Lp, 1))
            for i in range(start, start + n, rows):
                idx = order[i:min(i + rows, start + n)]
                kpm = key_padding_mask[idx].contiguous() if key_padding_mask is not None else None
                feats[i:i + idx.numel()] = self._tower(tokens[idx, :Lp].contiguous(), pe[:, :, :Lp] if pe is not None else None, kpm)
            start += n
        return feats, where

    def forward_zero_shot(self, text_tokens: Tensor, key_padding_mask: Optional[Tensor] = None) -> Tensor:
        """transformer.py:428-504: the class table of zero-shot classification, fp32 [d, Cl] = transpose(normalize(mean over the M captions
        of normalize(caption feature))), from the prompts of the first batch element of [B, Cl, M, L] (every element holds the same
        prompts).  Eval mode only.  The captions are encoded by ``_encode_rows``; ``classes_per_split_zero_shot`` is accepted and, as in
        the reference, does not change the result (``zero_shot_token_budget`` bounds the memory instead).  The per-caption normalisation,
        the mean and the final normalisation are one kernel (cvb_zs_class_embed) in fp32."""
        if self.training:
            raise NotImplementedError("Zero-shot evaluation is only supported with eval mode")
        _, Cl, M, L = text_tokens.shape
        kpm = key_padding_mask[0].reshape(Cl * M, L) if key_padding_mask is not None else None
        feats, where = self._encode_rows(text_tokens[0].reshape(Cl * M, L), kpm)
        return ops.zs_class_embed(feats, where.to(torch.int32), Cl, M)


class SimpleImageProjectionHead(nn.Module):
    """image_projection_layers/simple_projection_head.py:20-80 (``simple_projection_nc2nc``): x @ proj, then F.normalize."""

    def __init__(self, opts, in_dim: int, out_dim: int, *args, **kwargs) -> None:
        super().__init__()
        self.proj = nn.Parameter((in_dim ** -0.5) * torch.randn(size=(in_dim, out_dim)))
        self.in_dim, self.out_dim, self.feature_normalization = in_dim, out_dim, True
        self._proj = _Projection()

    def forward(self, x: Tensor, *args, **kwargs) -> Tensor:
        return Fn.L2NormFn.apply(self._proj.apply_to(x, self.proj, self))


class CLIP(nn.Module):
    def __init__(self, opts, *args, **kwargs) -> None:
        super().__init__()
        proj = getattr(opts, "model.multi_modal_image_text.clip.projection_dim", 256)
        self.image_encoder = VisionTransformer(opts)
        self.image_encoder.classifier = SimpleImageProjectionHead(opts, self.image_encoder.embed_dim, proj)
        self.text_encoder = TextTransformer(opts, projection_dim=proj)
        self.logit_scale = nn.Parameter(torch.ones([]) * math.log(1.0 / 0.07))
        self.cache_text_features_zero_shot = bool(getattr(opts, "model.multi_modal_image_text.clip.cache_text_features_zero_shot", False))
        self.cached_text_features = None

    def forward(self, images: Tensor, text_tokens: Tensor) -> Tuple[Tensor, Tensor, Tensor]:
        """(image features [B, d], text output, raw logit_scale).  The text output is what ``TextTransformer`` returns for the rank of
        ``text_tokens``: [B, d], [B, N, d], or in eval mode the [d, Cl] zero-shot class table of 4-D prompts."""
        img = self.image_encoder(images)
        txt = self.zero_shot_table(text_tokens) if text_tokens.dim() == 4 else self.text_encoder(text_tokens)
        return img, txt, self.logit_scale

    def zero_shot_table(self, class_tokens: Tensor) -> Tensor:
        """fp32 [d, Cl] class table of zero-shot prompts [B, Cl, M, L] (eval mode).  With
        ``model.multi_modal_image_text.clip.cache_text_features_zero_shot`` it is computed once and reused (clip.py:171-178).  Unlike the
        reference, which never drops that cache, ``train()`` and ``clear_zero_shot_cache()`` drop it: a table kept across further training
        would score the new weights against the old text tower.  The cache holds zero-shot tables only."""
        if self.cache_text_features_zero_shot and not self.training:
            if self.cached_text_features is None:
                self.cached_text_features = self.text_encoder(class_tokens)
            return self.cached_text_features
        return self.text_encoder(class_tokens)

    def clear_zero_shot_cache(self) -> None:
        self.cached_text_features = None

    def train(self, mode: bool = True):
        if mode:
            self.cached_text_features = None
        return super().train(mode)

    def zero_shot_logits(self, images: Tensor, class_table_or_tokens: Tensor, targets: Optional[Tensor] = None,
                         hits: Optional[Tensor] = None) -> Tensor:
        """clip.py:184-202 in eval mode: fp32 zero_shot_image_logits [B, Cl] = 100 * image features @ table (the fixed factor 100, not the
        logit scale), without autograd.  ``class_table_or_tokens``: an fp32 [d, Cl] table or 4-D prompts (see ``zero_shot_table``).  With
        ``targets`` (int64 [B]) and ``hits`` (int64 [2] on the device), the batch's top-1 / top-5 hits (metrics/topk_accuracy.py) are added
        into ``hits`` without a host sync."""
        if self.training:
            raise NotImplementedError("Zero-shot evaluation is only supported with eval mode")
        with torch.no_grad():
            table = class_table_or_tokens if class_table_or_tokens.dim() == 2 else self.zero_shot_table(class_table_or_tokens)
            img = self.image_encoder(images)
            return ops.zs_logits_topk(img, table, 100.0, targets, hits)


def clip_contrastive_loss(image_features: Tensor, text_features: Tensor, logit_scale: Tensor, process_group=None, _cfg=None) -> Tensor:
    """ContrastiveLossClip (loss_fn/multi_modal_img_text/contrastive_loss_clip.py:56-97): features of all ranks are gathered when a process
    group is initialised (gather_all_features), the labels are the global diagonal."""
    import torch.distributed as dist
    cfg = _cfg if _cfg is not None else SimpleNamespace(scale=None, ws=None)
    if not hasattr(cfg, "world"):
        on = dist.is_available() and dist.is_initialized()
        cfg.world, cfg.rank, cfg.group = (dist.get_world_size(process_group), dist.get_rank(process_group), process_group) if on else (1, 0, None)
    return Fn.ClipLossFn.apply(image_features, text_features, logit_scale, cfg)

"""The transformer workloads' training geometries, CPU only: ViT-B/16 at the bench resolution and at the variable-batch sampler's 320² and 128²
crops, ViT-S/16, the CLIP ViT-H/16 image tower, the ViT-H/16 finetune crop and both CLIP text towers.

The table is derived, not written down: widths, heads and FFN dims come from the oracle's parameter trees (``oracle.vit_shapes`` /
``clip_shapes``, tests/vit_huge_ref.py) and the model's configuration tables (``get_vit_configuration``, ``default_clip_opts``), batches from
the recipes' batch rules.  ``tests/test_transformer_shapes_gpu.py`` runs every kernel of the encoder at these geometries; this file pins the
table and, through restatements of the host-side launch formulas (csrc/gemm_tc.cu ``launch_tc``, csrc/wgrad_tc.cu ``launch_wgrad_tc``), that
the geometries do reach the paths the small kernel tests never do: a weight panel streamed through the A ring across many tiles per CTA, single-split
multi-wave weight gradients, ragged last M tiles, and the streaming attention kernels."""
import math
import os
import sys

import pytest

from oracle import cvnets_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from vit_huge_ref import vit_huge_shapes  # noqa: E402

H100_SMS = 132           # H100 SXM5; the GPU tests use the device's own count
BENCH_RES, PATCH = 224, 16
VIT_BATCH = 256          # examples/vit/classification/vit_base.yaml: 256 images of 224² per GPU
CLIP_BATCH = 256         # config/multi_modal_img_text/clip_vit.yaml and the ViT-H/16 CLIP recipe: 256 pairs per GPU
FINETUNE_BATCH = 64      # the ViT-H/16 ImageNet finetune recipe: 64 images of 224² per GPU
CLIP_H_TEXT = {"text_dim": 768, "text_heads": 12}  # examples/range_augment/clip/clip_vit_huge.yaml's text tower


def sampler_batch(base, crop):
    """the variable-batch sampler's batch at a crop: the 224² batch scaled by pixel count (tools/bench_vit_multiscale.py)"""
    return base * BENCH_RES * BENCH_RES // (crop * crop)


def _image_tower(gid, recipe, mode, B, crop):
    import ml_cvnets_b200 as m
    cfg = m.get_vit_configuration(m.default_vit_opts(mode))
    P = vit_huge_shapes() if mode == "huge" else O.vit_shapes(mode)
    C, ffn = P["cls_token"].shape[-1], P["transformer.0.pre_norm_ffn.1.weight"].shape[0]
    assert (C, ffn) == (cfg["embed_dim"], cfg["ffn_dim"]), mode
    stem = P["patch_emb.2.block.conv.weight"]
    n_patch = (crop // PATCH) ** 2
    return dict(id=gid, recipe=recipe, B=B, S=n_patch + 1, C=C, heads=cfg["n_attn_heads"], ffn=ffn, causal=False, eps=1e-6, act="gelu",
                n_patch=n_patch, n_pos=P["pos_embed.pos_embed.pos_embed"].shape[2], stem_k=stem.shape[1] * stem.shape[2] * stem.shape[3])


def _text_tower(gid, recipe, vit_mode, **text):
    import ml_cvnets_b200 as m
    opts = m.default_clip_opts(vit_mode, **text)
    P = O.clip_shapes("base", **({"text_dim": text["text_dim"]} if "text_dim" in text else {}))
    w1 = P["text_encoder.transformer.0.pre_norm_ffn.1.weight"]
    C = getattr(opts, "model.text.transformer.model_dim")
    assert w1.shape[1] == C
    return dict(id=gid, recipe=recipe, B=CLIP_BATCH, S=P["text_encoder.positional_embedding.pos_embed.pos_embed"].shape[2], C=C,
                heads=getattr(opts, "model.text.transformer.n_heads_per_layer"), ffn=w1.shape[0],
                causal=bool(getattr(opts, "model.text.transformer.causal_masking")), eps=1e-5, act="gelu", n_patch=None)


def geometries():
    """every transformer geometry the recipes train, with the recipe's batch"""
    return [
        _image_tower("vitb224", "ViT-B/16 224² (bench)", "base", VIT_BATCH, 224),
        _image_tower("vitb320", "ViT-B/16 sampler crop 320²", "base", sampler_batch(VIT_BATCH, 320), 320),
        _image_tower("vitb128", "ViT-B/16 sampler crop 128²", "base", sampler_batch(VIT_BATCH, 128), 128),
        _image_tower("vits224", "ViT-S/16 224² (bench vit_small)", "small", VIT_BATCH, 224),
        _image_tower("vith224", "CLIP ViT-H/16 image tower", "huge", CLIP_BATCH, 224),
        _image_tower("vith320", "ViT-H/16 finetune 320²", "huge", round(FINETUNE_BATCH * BENCH_RES ** 2 / 320 ** 2), 320),
        _text_tower("text512", "CLIP B/16 text tower", "base"),
        _text_tower("text768", "CLIP ViT-H text tower", "huge", **CLIP_H_TEXT),
    ]


# ------------------------------------------------------------------------------------------- restatements of the host-side launch formulas
def keep_normalised(g):
    """functional._encoder_forward: the LayerNorm prologue runs once as a pre-pass and its output is kept for the weight gradients"""
    from ml_cvnets_b200 import ops
    C, ffn = g["C"], g["ffn"]
    return C >= ops.WIDE_K and 3 * C >= ops.WIDE_N_WGRAD and ffn >= ops.WIDE_N_WGRAD


def gemm_launch(M, N, K, sms, nvec=0):
    """csrc/gemm_tc.cu launch_tc / launch_tc_impl for a one-operand load mode (nvec: per-channel fp32 vectors of the prologue)"""
    KT = (K + 31) // 32
    stagebuf = 128 * 136 * 2 + nvec * KT * 32 * 4 + 1024
    panel = KT * 8192
    resident = panel + stagebuf + 6 * 8192 <= 216 * 1024
    fixed, stage = (panel + stagebuf, 8192) if resident else (stagebuf, 8192 + 8192)
    nst = min(12, (216 * 1024 - fixed) // stage)
    n_tiles, m_tiles = (N + 127) // 128, (M + 127) // 128
    gy = max(1, min(sms // n_tiles, m_tiles))
    return dict(streams_weights=not resident, KT=KT, nst=nst, ctas=n_tiles * gy, tiles_per_cta=(m_tiles + gy - 1) // gy)


def wgrad_launch(M, N, K, sms):
    """csrc/wgrad_tc.cu launch_wgrad_tc (K % 64 == 0, K >= 128)"""
    nb, kb = (N + 127) // 128, (K + 127) // 128
    splits = max(1, sms // (nb * kb))
    splits = min(splits, (M + 255) // 256)
    m_per_cta = ((M + splits - 1) // splits + 63) // 64 * 64
    splits = (M + m_per_cta - 1) // m_per_cta
    return dict(splits=splits, ctas=nb * kb * splits, stages_per_cta=(m_per_cta + 63) // 64, nst=6)


def encoder_gemms(g):
    """(name, N, K) of the encoder's GEMMs (forward, then input gradients) and weight gradients, functional.py _encoder_forward / _backward"""
    C, ffn = g["C"], g["ffn"]
    fwd = [("qkv", 3 * C, C), ("out_proj", C, C), ("ffn1", ffn, C), ("ffn2", C, ffn),
           ("ffn2 dgrad", ffn, C), ("ffn1 dgrad", C, ffn), ("out_proj dgrad", C, C), ("qkv dgrad", C, 3 * C)]
    wgrad = [("ffn2 wgrad", C, ffn), ("ffn1 wgrad", ffn, C), ("out_proj wgrad", C, C), ("qkv wgrad", 3 * C, C)]
    return fwd, wgrad


def attention_route(g):
    """cvb_mha_fwd / bwd with head_dim 64: register-resident wgmma kernels up to 256 tokens, streaming kernels beyond"""
    return "register" if g["S"] <= 256 else "streaming"


# ------------------------------------------------------------------------------------------- tests
EXPECTED = {  # id: (B, S, C, heads, ffn, causal)
    "vitb224": (256, 197, 768, 12, 3072, False), "vitb320": (125, 401, 768, 12, 3072, False), "vitb128": (784, 65, 768, 12, 3072, False),
    "vits224": (256, 197, 384, 6, 1536, False), "vith224": (256, 197, 1280, 20, 5120, False), "vith320": (31, 401, 1280, 20, 5120, False),
    "text512": (256, 77, 512, 8, 2048, True), "text768": (256, 77, 768, 12, 3072, True),
}


def test_geometry_table():
    got = {g["id"]: (g["B"], g["S"], g["C"], g["heads"], g["ffn"], g["causal"]) for g in geometries()}
    assert got == EXPECTED
    for g in geometries():
        assert g["C"] // g["heads"] == 64, g["id"]  # every recipe has head_dim 64
        assert g["eps"] == (1e-5 if g["causal"] else 1e-6)
        if g["n_patch"] is not None:
            assert g["n_pos"] == (BENCH_RES // PATCH) ** 2 and g["stem_k"] == 4 * max(32, g["C"] // 4)


def test_ragged_rows_and_attention_routes():
    gs = {g["id"]: g for g in geometries()}
    ragged = {k for k, g in gs.items() if (g["B"] * g["S"]) % 128}
    assert ragged == {"vitb320", "vitb128", "vith320"}, ragged
    assert {k for k, g in gs.items() if attention_route(g) == "streaming"} == {"vitb320", "vith320"}
    # register-resident grids of B * H CTAs at the full recipe batch
    assert gs["vitb224"]["B"] * gs["vitb224"]["heads"] == 3072 and gs["vith224"]["B"] * gs["vith224"]["heads"] == 5120


def test_layernorm_routes():
    """vits224 is the one geometry whose LayerNorm prologue stays inside the GEMM / weight-gradient kernels at the encoder level"""
    assert {g["id"] for g in geometries() if not keep_normalised(g)} == {"vits224"}


def test_streamed_weight_panels_cross_tiles():
    """At K >= 768 the weight panel rides the A ring; at the FFN-down K the ring's stage index wraps across tile boundaries (KT % nst != 0) and
    every CTA walks many tiles"""
    for g in geometries():
        M = g["B"] * g["S"]
        fwd, _ = encoder_gemms(g)
        for name, N, K in fwd:
            L = gemm_launch(M, N, K, H100_SMS)
            assert L["streams_weights"] == (K >= 768), (g["id"], name, L)
            assert L["ctas"] <= H100_SMS
        L = gemm_launch(M, g["C"], g["ffn"], H100_SMS)  # ffn2: K = 4C
        assert L["streams_weights"] and L["KT"] % L["nst"] != 0, (g["id"], L)
        if g["C"] >= 768 and g["n_patch"] == 196:
            assert L["tiles_per_cta"] >= 18, (g["id"], L)
    vb = next(g for g in geometries() if g["id"] == "vitb224")
    assert gemm_launch(vb["B"] * vb["S"], 768, 3072, H100_SMS)["KT"] == 96
    vh = next(g for g in geometries() if g["id"] == "vith224")
    assert gemm_launch(vh["B"] * vh["S"], 1280, 5120, H100_SMS)["KT"] == 160


def test_large_weight_gradients_run_one_split_over_several_waves():
    for g in geometries():
        if g["C"] < 768:
            continue
        M = g["B"] * g["S"]
        _, wg = encoder_gemms(g)
        for name, N, K in wg:
            L = wgrad_launch(M, N, K, H100_SMS)
            if name in ("ffn1 wgrad", "ffn2 wgrad", "qkv wgrad"):
                assert L["splits"] == 1 and L["stages_per_cta"] == math.ceil(M / 64), (g["id"], name, L)
            if name in ("ffn1 wgrad", "ffn2 wgrad"):
                assert L["ctas"] > H100_SMS, (g["id"], name, L)
    vb = next(g for g in geometries() if g["id"] == "vitb224")
    assert wgrad_launch(50432, 3072, 768, H100_SMS) == dict(splits=1, ctas=144, stages_per_cta=788, nst=6)
    assert vb["B"] * vb["S"] == 50432
    assert wgrad_launch(50432, 5120, 1280, H100_SMS) == dict(splits=1, ctas=400, stages_per_cta=788, nst=6)


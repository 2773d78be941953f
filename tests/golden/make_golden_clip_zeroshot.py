"""Golden fixture FROM THE REAL REFERENCE for CLIP zero-shot evaluation (see make_golden.py for the method).

The reduced CLIP of clip_small_fp32.pt (make_golden_r2.py: seed-71 weights, ViT-small image tower, 4-layer / 256-wide causal text tower,
context 16, vocabulary 1000, projection 128) in eval mode; BatchNorm running statistics are the seeded ones, as in the eval fixtures of
make_golden_r2.py.
  * prompts [2, 12, 5, 16]: 12 classes x 5 captions, the end-of-text id 999 at positions spread over 3..15.  The second batch element
    holds other prompts: the reference encodes the first only (transformer.py:453-461).
  * the [128, 12] class table (transformer.py:428-504) at classes_per_split_zero_shot 1 and 5 (asserted equal to fp32 rounding: the split only bounds
    memory), zero_shot_image_logits of 8 images at 224^2 (clip.py:184-202), and top-1 / top-5 of labels in [0, 12)
    (metrics/topk_accuracy.py);
  * a 3-D batch [3, 2, 16] (several captions per image) and its [3, 2, 128] text features (transformer.py:534-549).

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_clip_zeroshot.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import O, get_model, load_seeded, make_opts, torch  # noqa: E402

from metrics.topk_accuracy import top_k_accuracy  # noqa: E402

EOT = 999


def prompts(shape, gen):
    """random ids in [1, EOT) with one end-of-text token per row, at positions cycling over 3..15."""
    t = torch.randint(1, EOT, shape, generator=gen)
    rows = t.view(-1, shape[-1])
    pos = (torch.arange(rows.shape[0]) * 7) % 13 + 3
    rows[torch.arange(rows.shape[0]), pos] = EOT
    return t


def main():
    torch.manual_seed(0)
    opts = make_opts(1.0)
    for k, v in {"dataset.category": "multi_modal_image_text", "model.multi_modal_image_text.name": "clip", "model.multi_modal_image_text.clip.projection_dim": 128,
                 "model.classification.name": "vit", "model.classification.vit.mode": "small", "model.classification.vit.norm_layer": "layer_norm_fp32",
                 "model.activation.name": "gelu", "model.classification.activation.name": "gelu", "model.image_projection_head.name": "simple_projection_nc2nc",
                 "model.text.name": "transformer", "model.text.transformer.model_dim": 256, "model.text.transformer.n_transformer_layers": 4,
                 "model.text.transformer.n_heads_per_layer": 4, "model.text.transformer.ffn_multiplier_per_layer": 4.0,
                 "model.text.transformer.causal_masking": True, "model.text.transformer.norm_layer": "layer_norm_fp32", "dataset.text_vocab_size": 1000,
                 "dataset.text_context_length": 16, "dataset.padding_index": None, "ddp.use_distributed": False, "ddp.rank": 0,
                 "model.multi_modal_image_text.clip.cache_text_features_zero_shot": False}.items():
        setattr(opts, k, v)
    model = get_model(opts)
    P = O.clip_shapes("small", proj=128, text_dim=256, text_layers=4, vocab=1000, ctx=16)
    seed = 71
    load_seeded(model, P, seed)
    model.eval()
    gen = torch.Generator().manual_seed(381)
    tokens = prompts((2, 12, 5, 16), gen)
    tokens_3d = prompts((3, 2, 16), gen)
    x_seed = 382
    images = O.seeded_input((8, 3, 224, 224), x_seed)
    labels = torch.randint(0, 12, (8,), generator=gen)
    with torch.no_grad():
        tables = {}
        for split in (1, 5):
            model.text_encoder.classes_per_split_zero_shot = split
            tables[split] = model.text_encoder(tokens).clone()
        gap = float((tables[1] - tables[5]).abs().max())
        assert gap <= 1e-6, gap
        out = model({"image": images, "text": tokens})
        logits = out["zero_shot_image_logits"].clone()
        top1, top5 = (float(a) for a in top_k_accuracy(logits, labels, top_k=(1, 5)))
        text_3d = model.text_encoder(tokens_3d).clone()
    assert tuple(tables[1].shape) == (128, 12) and tuple(logits.shape) == (8, 12) and tuple(text_3d.shape) == (3, 2, 128)
    fx = dict(seed=seed, x_seed=x_seed, tokens=tokens, labels=labels, table=tables[1], table_split5=tables[5], split_gap=gap,
              zero_shot_image_logits=logits, top1=top1, top5=top5, tokens_3d=tokens_3d, text_3d=text_3d)
    out_path = os.path.join(HERE, "clip_zeroshot_fp32.pt")
    torch.save(fx, out_path)
    print(out_path, os.path.getsize(out_path), "bytes; split gap", gap, "top1", top1, "top5", top5)


if __name__ == "__main__":
    main()

"""CLIP ViT-B/16 zero-shot evaluation on the library's kernels (config/multi_modal_img_text/clip_vit.yaml: zero_shot_eval, ImageNet's
1000 classes x 78 prompt templates at context 77).

    python tools/bench_clip_zeroshot.py OUTDIR [--reps 3] [--seed 0]

Writes OUTDIR/clip_zeroshot.json and prints it:
  * the card (name, power limit, SM clocks) read by nvidia-smi in the same run;
  * the class-table build (78 000 captions through the 12-layer text tower + cvb_zs_class_embed), CUDA events, with each caption run at its
    causal prefix (the library's path) and at the full context length (the reference's batching, on the same kernels), the speed-up, and
    how far apart the two tables are;
  * one zero-shot batch: B = 256 images at 224 px through the image tower in eval mode, then logits and top-1 / top-5 counts
    (cvb_zs_logits_topk); and the logits / top-k kernel alone.
The prompts are synthetic: CLIP's BPE vocabulary is a download, so real prompt lengths are not available here.  Each caption's end-of-text
position is 1 + t + c, with a template length t uniform in [4, 14] and a class-name length c uniform in [1, 6] (positions 6..21); token
ids are uniform below the end-of-text id.  The truncation speed-up depends on that distribution.
"""
import argparse
import json
import os
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)
sys.path.insert(0, os.path.join(REPO, "tools"))
from bench_vit_multiscale import card, timed  # noqa: E402

CLASSES, TEMPLATES, CONTEXT = 1000, 78, 77


def synthetic_prompts(vocab, seed):
    g = torch.Generator().manual_seed(seed)
    n = CLASSES * TEMPLATES
    tokens = torch.randint(1, vocab - 1, (n, CONTEXT), generator=g)
    eot = 1 + torch.randint(4, 15, (n,), generator=g) + torch.randint(1, 7, (n,), generator=g)
    tokens[torch.arange(n), eot] = vocab - 1  # the end-of-text token is the highest id
    tokens[torch.arange(CONTEXT).view(1, -1) > eot.view(-1, 1)] = 0  # padding after it, as a tokenizer writes
    return tokens.view(1, CLASSES, TEMPLATES, CONTEXT), eot


def full_length_table(enc, tokens, ops):
    """The reference's batching on the library's kernels: every caption at the full context length, in prompt order."""
    rows = tokens[0].reshape(-1, CONTEXT)
    pe = enc.positional_embedding.pos_embed.pos_embed
    step = max(1, enc.zero_shot_token_budget // CONTEXT)
    with torch.no_grad():
        feats = torch.cat([enc._tower(rows[i:i + step].contiguous(), pe, None) for i in range(0, rows.shape[0], step)])
        return ops.zs_class_embed(feats, torch.arange(rows.shape[0], device=rows.device, dtype=torch.int32), CLASSES, TEMPLATES)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--seed", type=int, default=0)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_clip_zeroshot needs a CUDA device")
    import ml_cvnets_b200 as m
    from ml_cvnets_b200 import ops
    os.makedirs(args.outdir, exist_ok=True)
    torch.manual_seed(args.seed)
    model = m.CLIP(m.default_clip_opts()).cuda().eval()
    enc = model.text_encoder
    tokens, eot = synthetic_prompts(enc.vocab_size, args.seed)
    tokens = tokens.cuda()
    res = {"card": card(), "model": "CLIP ViT-B/16 (default options), eval mode, random weights",
           "prompts": {"classes": CLASSES, "templates": TEMPLATES, "context": CONTEXT, "synthetic": True,
                       "eot_position": "1 + U[4, 14] + U[1, 6] (CLIP's BPE files are a download: real prompt lengths are not available offline)",
                       "mean_eot_position": float(eot.float().mean()), "token_budget": enc.zero_shot_token_budget}}
    truncated = model.zero_shot_table(tokens)
    full = full_length_table(enc, tokens, ops)
    res["table"] = {
        "truncated_ms": timed(lambda: model.zero_shot_table(tokens), args.reps),
        "full_length_ms": timed(lambda: full_length_table(enc, tokens, ops), args.reps),
        "rel_l2_truncated_vs_full": float((truncated - full).norm() / full.norm()),
        "bitwise_equal": bool(torch.equal(truncated, full)),
        "tokens_truncated": int(((eot + 8) // 8 * 8).clamp(max=CONTEXT).sum()), "tokens_full": CLASSES * TEMPLATES * CONTEXT}
    res["table"]["speedup"] = res["table"]["full_length_ms"] / res["table"]["truncated_ms"]
    print(json.dumps(res["table"]), flush=True)
    B = 256
    g = torch.Generator(device="cuda").manual_seed(args.seed + 1)
    images = torch.randn(B, 3, 224, 224, device="cuda", generator=g)
    targets = torch.randint(0, CLASSES, (B,), device="cuda", generator=g)
    hits = torch.zeros(2, device="cuda", dtype=torch.int64)
    with torch.no_grad():
        img, _ = model.encode_images(images)
    for _ in range(3):
        model.zero_shot_logits(images, truncated, targets=targets, hits=hits)
        ops.zs_logits_topk(img, truncated, 100.0, targets, hits)
    iters = 10 * args.reps
    res["batch"] = {"batch": B, "resolution": 224,
                    "image_tower_and_topk_ms": timed(lambda: model.zero_shot_logits(images, truncated, targets=targets, hits=hits), iters),
                    "logits_topk_kernel_ms": timed(lambda: ops.zs_logits_topk(img, truncated, 100.0, targets, hits), iters)}
    res["batch"]["img_per_s"] = B / (res["batch"]["image_tower_and_topk_ms"] * 1e-3)
    print(json.dumps(res["batch"]), flush=True)
    res["card_after"] = card()
    with open(os.path.join(args.outdir, "clip_zeroshot.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""The ViT-H/16 recipes' training steps, with recomputing gradient checkpointing of the encoder stacks:
  * clip (examples/range_augment/clip/clip_vit_huge.yaml): CLIP with a ViT-H/16 image tower (4 checkpointed segments) and a 768-wide, 12-layer
    text tower (every layer checkpointed), B = 256 synthetic image-text pairs at 224^2, RangeAugment with the NA loss, AdamW (0.9, 0.98, eps
    1e-6, weight decay 0.2), EMA 0.0005, the whole step captured as one CUDA graph;
  * finetune (examples/range_augment/clip_finetune_imagenet/clip_vit_huge.yaml): the ViT-H/16 classifier, B = 64 at 224^2 and the variable-batch
    sampler's 320^2 crop at its batch (round(64 * 224^2 / 320^2) = 31), AdamW (weight decay 0.2), label smoothing 0.1, eager steps with
    checkpointing on and off alternated on the same model.

    python tools/bench_vit_huge.py OUTDIR [--steps 5] [--rounds 3] [--skip-clip] [--skip-finetune]

Writes OUTDIR/vit_huge.json and prints it: the card (name, power limit, SM clocks) read by nvidia-smi in the same run, step times from CUDA
events, images/s, launches per step, the peak allocated / reserved memory, and the step's model FLOPs (GEMMs and attention, counted from the
shapes: 2 per multiply-add, backward = 2x forward, the recompute counted on its own) against NVIDIA's 989 TFLOP/s dense-BF16 data-sheet figure
for the H100 SXM.  Attention is counted over the full S x S score matrix, also under the text tower's causal mask.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

PEAK_BF16 = 989e12
AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True, "model.learn_augmentation.lr_multiplier": 1.0}
CKPT = {"model.classification.gradient_checkpointing": True, "model.classification.vit.checkpoint_segments": 4}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return {"query": q, "nvidia_smi": out.splitlines()[0] if out else None, "torch_name": torch.cuda.get_device_name()}


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def encoder_fwd_flops(N, S, C, ffn):
    """One pre-norm encoder layer's forward: qkv / out_proj / FFN GEMMs and the two attention products."""
    return 2 * N * S * (3 * C * C + C * C + 2 * C * ffn) + 4 * N * S * S * C


def vit_fwd_flops(B, res, C, layers):
    g = res // 16
    stem = max(32, C // 4)
    conv = 2 * B * ((res // 4) ** 2 * stem * 48 + (res // 8) ** 2 * stem * stem * 4 + g * g * C * stem * 4)
    return conv + layers * encoder_fwd_flops(B, g * g + 1, C, 4 * C)


def flop_report(fwd, recompute, ms):
    total = 3 * fwd + recompute
    return {"model_flops_fwd_bwd": 3 * fwd, "recompute_flops": recompute, "tflops_per_s_with_recompute": total / ms / 1e9,
            "share_of_989_tflops_model": 3 * fwd / ms / 1e-3 / PEAK_BF16, "share_of_989_tflops_with_recompute": total / ms / 1e-3 / PEAK_BF16}


def bench_clip(m, B, steps, rounds):
    torch.manual_seed(0)
    opts = m.default_clip_opts("huge", projection_dim=512, text_dim=768, text_layers=12, text_heads=12, **AUG, **CKPT,
                               **{"model.text.transformer.gradient_checkpoint": True})
    model = m.CLIP(opts).cuda().train()
    na = m.NeuralAugmentationLoss(target_value=(40, 20), curriculum_method="cosine", period=12)

    def clip_loss(mod, im, tok, cfg):
        img, txt, scale, x_aug = mod(im, tok)
        return m.clip_contrastive_loss(img, txt, scale, _cfg=cfg), x_aug

    step = m.TrainStep(model, lr=5e-4, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.2, max_norm=None, ema_momentum=0.0005, aug_loss=na,
                       forward_loss=clip_loss)
    x = torch.rand(B, 3, 224, 224, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(1234)
    tok = torch.randint(1, 49406, (B, 77), device="cuda", generator=gen)
    tok[torch.arange(B, device="cuda"), torch.randint(1, 77, (B,), device="cuda", generator=gen)] = 49407
    torch.cuda.reset_peak_memory_stats()
    step.capture(x, tok)
    step(x, tok)
    times = [timed(lambda: step(x, tok), steps) for _ in range(rounds)]
    ms = min(times)
    img_fwd = vit_fwd_flops(B, 224, 1280, 32)
    txt_fwd = 12 * encoder_fwd_flops(B, 77, 768, 3072)
    recompute = 24 * encoder_fwd_flops(B, 197, 1280, 5120) + txt_fwd  # image layers 0-23 (3 of 4 segments) and every text layer
    out = {"batch": B, "res": 224, "step_ms": {"rounds": times, "min": ms}, "images_per_s": B / ms * 1e3, "launches_per_step": step.launches_per_step,
           "max_memory_allocated_GiB": torch.cuda.max_memory_allocated() / 2**30, "max_memory_reserved_GiB": torch.cuda.max_memory_reserved() / 2**30,
           "loss_parts": step.loss_parts.tolist(), "n_params": sum(p.numel() for p in model.parameters())}
    out.update(flop_report(img_fwd + txt_fwd, recompute, ms))
    return out


def bench_finetune(m, steps, rounds):
    torch.manual_seed(0)
    model = m.VisionTransformer(m.default_vit_opts("huge", n_classes=1000, **CKPT)).cuda().train()
    step = m.TrainStep(model, lr=1e-5, betas=(0.9, 0.999), weight_decay=0.2, max_norm=1.0, label_smoothing=0.1)
    res = {}
    for crop, B in ((224, 64), (320, 31)):
        x = torch.rand(B, 3, crop, crop, device="cuda")
        y = torch.randint(0, 1000, (B,), device="cuda")
        times, mem = {"on": [], "off": []}, {}
        for mode in ("off", "on"):  # warm-up of both configurations (the recompute's scratch is planned on its first steps)
            model.gradient_checkpointing = mode == "on"
            for _ in range(3):
                step(x, y)
        for _ in range(rounds):
            for mode in ("off", "on"):
                model.gradient_checkpointing = mode == "on"
                step(x, y)
                torch.cuda.synchronize()
                base = torch.cuda.memory_allocated()
                torch.cuda.reset_peak_memory_stats()
                times[mode].append(timed(lambda: step(x, y), steps))
                mem[mode] = (torch.cuda.max_memory_allocated() - base) / 2**30
        fwd = vit_fwd_flops(B, crop, 1280, 32)
        g = crop // 16
        recompute = 24 * encoder_fwd_flops(B, g * g + 1, 1280, 5120)
        on, off = min(times["on"]), min(times["off"])
        res[f"{crop}x{crop}"] = {
            "batch": B, "step_ms": {k: {"rounds": v, "min": min(v)} for k, v in times.items()}, "images_per_s": {"on": B / on * 1e3, "off": B / off * 1e3},
            "recompute_cost_ms": on - off, "recompute_cost_fraction": (on - off) / off, "step_memory_growth_GiB": mem,
            "memory_saved_GiB": mem["off"] - mem["on"], "on": flop_report(fwd, recompute, on), "off": flop_report(fwd, 0, off)}
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256, help="CLIP step batch (the recipe's per-GPU 256)")
    ap.add_argument("--skip-clip", action="store_true")
    ap.add_argument("--skip-finetune", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vit_huge.py needs a CUDA device")
    import ml_cvnets_b200 as m
    os.makedirs(a.outdir, exist_ok=True)
    res = {"card": card(), "device_total_GiB": torch.cuda.get_device_properties(0).total_memory / 2**30}
    if not a.skip_clip:
        res["clip_vit_h16_step"] = bench_clip(m, a.batch, a.steps, a.rounds)
        torch.cuda.empty_cache()
    if not a.skip_finetune:
        res["finetune_vit_h16_step"] = bench_finetune(m, a.steps, a.rounds)
    res["card_after"] = card()
    with open(os.path.join(a.outdir, "vit_huge.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Captured against eager training steps at a variable-batch recipe's (crop, batch) table, with ONE model and ONE TrainStep for all shapes.

    python tools/bench_multiscale.py OUTDIR --model efficientnet_b0 | vit_b16 | clip_b16 [--steps 20] [--eager-steps 5] [--seq 60]

Writes OUTDIR/multiscale_<model>.json and prints it:
  * the card (name, power limit, SM clocks) read by nvidia-smi in the same run;
  * per (crop, batch): the eager step (before capture, on the same TrainStep) and the captured step in ms (CUDA events over --eager-steps /
    --steps steps after warm-up), images/s and launches per step;
  * images/s over a sampler-like random sequence of --seq shapes (each batch copied into its graph's static buffers, as a training loop does);
  * the graphs' memory pool and torch's reserved memory after capturing every shape, next to the same after capturing only the most demanding
    shape (the largest input) in a fresh process.

Tables: examples/range_augment/classification/efficientnet_b0.yaml and examples/vit/classification/vit_base.yaml (128..320 px, 10 and 25
scales), examples/range_augment/clip/clip_vit_base.yaml (160..320 px, 5 scales); train_batch_size0 256.  Optimizers as the recipes: SGD-Nesterov
for EfficientNet, AdamW for ViT and CLIP.
"""
import argparse
import json
import os
import random
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

TABLES = {"efficientnet_b0": dict(crop_w=224, crop_h=224, batch=256, max_scales=10, check_scale=32, min_w=128, max_w=320, min_h=128, max_h=320),
          "vit_b16": dict(crop_w=224, crop_h=224, batch=256, max_scales=25, check_scale=32, min_w=128, max_w=320, min_h=128, max_h=320),
          "clip_b16": dict(crop_w=224, crop_h=224, batch=256, max_scales=5, check_scale=32, min_w=160, max_w=320, min_h=160, max_h=320)}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return {"query": q, "nvidia_smi": out.splitlines()[0] if out else None, "torch_name": torch.cuda.get_device_name()}


def build(m, model_name):
    torch.manual_seed(0)
    if model_name == "efficientnet_b0":
        model = m.EfficientNet(m.default_effnet_opts("b0", n_classes=1000)).cuda().train()
        ts = m.TrainStep(model, optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None, label_smoothing=0.1,
                         ema_momentum=0.0005)
    elif model_name == "vit_b16":
        model = m.VisionTransformer(m.default_vit_opts("base")).cuda().train()
        ts = m.TrainStep(model, lr=2e-3, weight_decay=0.05, max_norm=10.0, label_smoothing=0.1)
    else:
        model = m.CLIP(m.default_clip_opts("base")).cuda().train()

        def forward_loss(mdl, im, tok, cfg):
            img, txt, scale = mdl(im, tok)
            return m.clip_contrastive_loss(img, txt, scale, _cfg=cfg)
        ts = m.TrainStep(model, lr=5e-4, weight_decay=0.2, max_norm=1.0, forward_loss=forward_loss)
    return model, ts


def inputs(model_name, h, w, b, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(b, 3, h, w, device="cuda", generator=g)
    if model_name == "clip_b16":
        tok = torch.randint(1, 49406, (b, 77), device="cuda", generator=g)
        tok[:, -1] = 49407
        return x, tok
    return x, torch.randint(0, 1000, (b,), device="cuda", generator=g)


def timed(fn, n):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / n


def memory(ts):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    return {"graph_pool_bytes": ts.graph_pool_bytes(), "reserved_bytes": torch.cuda.memory_reserved(), "allocated_bytes": torch.cuda.memory_allocated()}


def single_arm(model_name, h, w, b):
    """Capture only (h, w, b) on a fresh model: the memory one graph reserves."""
    import ml_cvnets_b200 as m
    _, ts = build(m, model_name)
    ts.capture(*inputs(model_name, h, w, b, 1))
    return memory(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--model", choices=sorted(TABLES), default="efficientnet_b0")
    ap.add_argument("--steps", type=int, default=20, help="captured replays timed per shape (after 3 untimed)")
    ap.add_argument("--eager-steps", type=int, default=5, help="eager steps timed per shape (after 2 untimed)")
    ap.add_argument("--seq", type=int, default=60, help="length of the random shape sequence")
    ap.add_argument("--single-arm", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_multiscale needs a CUDA device")
    if args.single_arm:
        print(json.dumps(single_arm(args.model, *(int(v) for v in args.single_arm.split(",")))))
        return
    import ml_cvnets_b200 as m
    pairs = m.variable_batch_pairs(**TABLES[args.model])
    os.makedirs(args.outdir, exist_ok=True)
    res = {"card": card(), "model": args.model, "table": pairs, "steps": args.steps, "eager_steps": args.eager_steps, "shapes": []}
    _, ts = build(m, args.model)
    data = {(h, w, b): inputs(args.model, h, w, b, h * 1000 + b) for h, w, b in pairs}
    rows = {}
    for key, ex in data.items():  # eager, before capture, on the TrainStep that is captured below: real training steps
        for _ in range(2):
            ts.step(*ex)
        from ml_cvnets_b200 import ops
        n0 = ops.launch_count
        ms = timed(lambda: ts.step(*ex), args.eager_steps)
        rows[key] = {"crop_h": key[0], "crop_w": key[1], "batch": key[2], "eager_ms": ms,
                     "eager_launches_per_step": (ops.launch_count - n0) // args.eager_steps}
        print(json.dumps(rows[key]), flush=True)
    n_eager = ts.eager_steps
    ts.capture_shapes(list(data.values()))
    res["memory_all_shapes"] = memory(ts)
    res["warmup_steps_in_capture"] = ts.eager_steps - n_eager
    for key, ex in data.items():
        feed = inputs(args.model, *key, 7)  # a different batch: the replay copies it into the static buffers, as a loop does
        for _ in range(3):
            ts.step(*feed)
        ms = timed(lambda: ts.step(*feed), args.steps)
        r = rows[key]
        r.update(captured_ms=ms, captured_img_per_s=key[2] / (ms * 1e-3), eager_img_per_s=key[2] / (r["eager_ms"] * 1e-3),
                 speedup=r["eager_ms"] / ms, launches_per_step=ts.launches_per_shape[tuple(tuple(t.shape) for t in ex)])
        res["shapes"].append(r)
        print(json.dumps(r), flush=True)
    rnd = random.Random(0)
    seq = [rnd.choice(pairs) for _ in range(args.seq)]
    feeds = {key: inputs(args.model, *key, 11) for key in data}
    for key in seq[:3]:
        ts.step(*feeds[key])
    it = iter(seq)
    ms = timed(lambda: ts.step(*feeds[next(it)]), len(seq))
    res["sequence"] = {"steps": len(seq), "ms_per_step": ms, "img_per_s": sum(b for _, _, b in seq) / (ms * len(seq) * 1e-3)}
    print(json.dumps(res["sequence"]), flush=True)
    big = max(pairs, key=lambda p: p[0] * p[1] * p[2] * 3 if args.model != "clip_b16" else p[0] * p[1] * p[2] * 3 + p[2] * 77 * 8)
    out = subprocess.run([sys.executable, os.path.abspath(__file__), args.outdir, "--model", args.model, "--single-arm", ",".join(map(str, big))],
                         capture_output=True, text=True)
    if out.returncode != 0:
        raise SystemExit(f"single-shape arm failed: {out.stderr[-2000:]}")
    res["memory_most_demanding_shape_only"] = dict(json.loads(out.stdout.strip().splitlines()[-1]), shape=big)
    res["graph_pool_ratio"] = res["memory_all_shapes"]["graph_pool_bytes"] / max(1, res["memory_most_demanding_shape_only"]["graph_pool_bytes"])
    res["card_after"] = card()
    with open(os.path.join(args.outdir, f"multiscale_{args.model}.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}))


if __name__ == "__main__":
    main()

"""Captured against eager training steps at a variable-batch recipe's (crop, batch) table, with ONE model and ONE TrainStep for all shapes.

    python tools/bench_multiscale.py OUTDIR --model efficientnet_b0 | efficientnet_b3 | vit_b16 | clip_b16 | mobilevit_xxs | mobilevit_s
                                             [--steps 20] [--eager-steps 5] [--seq 60]
    python tools/bench_multiscale.py OUTDIR --model efficientnet_b3 --accum-freq 2 [--steps 20] [--seq 60]

Writes OUTDIR/multiscale_<model>.json and prints it:
  * the card (name, power limit, SM clocks) read by nvidia-smi in the same run;
  * per (crop, batch): the eager step (before capture, on the same TrainStep) and the captured step in ms (CUDA events over --eager-steps /
    --steps steps after warm-up), images/s and launches per step;
  * images/s over a sampler-like random sequence of --seq shapes (each batch copied into its graph's static buffers, as a training loop does);
  * the graphs' memory pool and torch's reserved memory after capturing every shape, next to the same after capturing only the most demanding
    shape (the largest input) in a fresh process.

With ``--accum-freq K`` (K > 1; writes OUTDIR/multiscale_<model>_accum<K>.json) the run compares gradient accumulation with the plain step
instead, two captured TrainSteps on one model definition: accum_freq 1 and K.  Reported: per (crop, batch) the captured ms per micro-batch of
each, timed in alternating rounds; images/s of each over one random sequence of --seq shapes; each one's graph pool; and cvb_grad_accumulate
alone at the EfficientNet-B3 and CLIP ViT-H/16 parameter counts (CUDA events; 12 bytes per element -- read acc and g, write acc -- over the
time, against the H100 SXM data sheet's 3.35 TB/s).

Tables: examples/range_augment/classification/efficientnet_b0.yaml and examples/vit/classification/vit_base.yaml (128..320 px, 10 and 25
scales), examples/range_augment/clip/clip_vit_base.yaml (160..320 px, 5 scales); train_batch_size0 256.  efficientnet_b3.yaml of the same
directory: 300 px x 128 images, 160..448 px, 10 scales, accum_freq 2, RangeAugment (target PSNR 40 -> 5, cosine over 400 epochs), EMA
0.0005.  config/classification/imagenet/mobilevit.yaml (every MobileViT-v1 recipe): 256 px x 128 images, 160..320 px, 5 scales, AdamW (weight
decay 0.01), EMA 0.0005.  MobileViT-S drops the 192 px pair: its layer 3 has 144 tokens of width 144 there, where the reference's LayerNorm
normalises over the token axis, which the library refuses (TransformerEncoder.prepare).  Optimizers as the recipes: SGD-Nesterov for
EfficientNet, AdamW for ViT, CLIP and MobileViT.
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
          "clip_b16": dict(crop_w=224, crop_h=224, batch=256, max_scales=5, check_scale=32, min_w=160, max_w=320, min_h=160, max_h=320),
          "efficientnet_b3": dict(crop_w=300, crop_h=300, batch=128, max_scales=10, check_scale=32, min_w=160, max_w=448, min_h=160, max_h=448),
          "mobilevit_xxs": dict(crop_w=256, crop_h=256, batch=128, max_scales=5, check_scale=32, min_w=160, max_w=320, min_h=160, max_h=320),
          "mobilevit_s": dict(crop_w=256, crop_h=256, batch=128, max_scales=5, check_scale=32, min_w=160, max_w=320, min_h=160, max_h=320)}
# (h, w) pairs a model cannot train at, and why
SKIP = {"mobilevit_s": {(192, 192): "layer 3 has 144 tokens of width 144: the reference's LayerNorm takes its token-axis branch, which the library "
                                    "refuses"}}


def recipe_pairs(m, model_name):
    return [p for p in m.variable_batch_pairs(**TABLES[model_name]) if p[:2] not in SKIP.get(model_name, {})]
AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return {"query": q, "nvidia_smi": out.splitlines()[0] if out else None, "torch_name": torch.cuda.get_device_name()}


def build(m, model_name, accum_freq=1):
    torch.manual_seed(0)
    if model_name == "efficientnet_b3":
        model = m.EfficientNet(m.default_effnet_opts("b3", n_classes=1000, **AUG)).cuda().train()
        na = m.NeuralAugmentationLoss(target_value=(40, 5), curriculum_method="cosine", period=400)
        ts = m.TrainStep(model, optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None, label_smoothing=0.1,
                         ema_momentum=0.0005, ema_buffers=True, aug_loss=na, accum_freq=accum_freq)
    elif model_name == "efficientnet_b0":
        model = m.EfficientNet(m.default_effnet_opts("b0", n_classes=1000)).cuda().train()
        ts = m.TrainStep(model, optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None, label_smoothing=0.1,
                         ema_momentum=0.0005)
    elif model_name.startswith("mobilevit"):
        model = m.MobileViT(m.default_mit_opts({"mobilevit_xxs": "xx_small", "mobilevit_s": "small"}[model_name])).cuda().train()
        ts = m.TrainStep(model, lr=2e-3, weight_decay=0.01, max_norm=None, label_smoothing=0.1, ema_momentum=0.0005)
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


def accumulate_alone(m, n, reps=50):
    """cvb_grad_accumulate over n fp32 elements: ms per launch (CUDA events over ``reps`` launches after 5 untimed) and 12 n bytes / time."""
    from ml_cvnets_b200 import ops
    acc, g = torch.zeros(n, device="cuda"), torch.randn(n, device="cuda")
    for _ in range(5):
        ops.grad_accumulate(acc, g)
    ms = timed(lambda: ops.grad_accumulate(acc, g), reps)
    tbs = 12.0 * n / (ms * 1e-3) / 1e12
    return {"n": n, "ms": ms, "bytes": 12 * n, "tb_per_s": tbs, "fraction_of_3.35_tb_per_s": tbs / 3.35}


def compare_accum(m, args):
    """accum_freq 1 against args.accum_freq on the recipe's table: both TrainSteps captured, timed per micro-batch in alternating rounds."""
    pairs = recipe_pairs(m, args.model)
    res = {"card": card(), "model": args.model, "table": pairs, "accum_freq": args.accum_freq, "steps": args.steps, "shapes": []}
    data = {(h, w, b): inputs(args.model, h, w, b, h * 1000 + b) for h, w, b in pairs}
    arms = {}
    for k in (1, args.accum_freq):
        model, ts = build(m, args.model, accum_freq=k)
        ts.set_mix("mixup", 0.7)
        ts.capture_shapes(list(data.values()))
        arms[k] = (model, ts)
        res[f"memory_accum{k}"] = memory(ts)
        res[f"launches_accum{k}"] = {"per_micro_step": max(ts.launches_per_shape.values()), "update": ts.launches_per_update}
        print(json.dumps({f"accum_freq {k}": res[f"memory_accum{k}"], "launches": res[f"launches_accum{k}"]}), flush=True)
    res["graph_pool_ratio"] = res[f"memory_accum{args.accum_freq}"]["graph_pool_bytes"] / max(1, res["memory_accum1"]["graph_pool_bytes"])
    rounds = 3
    for key in data:
        feed = inputs(args.model, *key, 7)
        row = {"crop_h": key[0], "crop_w": key[1], "batch": key[2]}
        ms = {k: 0.0 for k in arms}
        for k, (_, ts) in arms.items():
            for _ in range(2 * args.accum_freq):
                ts.step(*feed)
        for _ in range(rounds):
            for k, (_, ts) in arms.items():
                # whole windows per round, so both arms time the same mix of micro-steps and updates
                n = max(args.accum_freq, args.steps // rounds // args.accum_freq * args.accum_freq)
                ms[k] += timed(lambda: ts.step(*feed), n) / rounds
        row.update({f"captured_ms_accum{k}": v for k, v in ms.items()})
        row["ratio"] = ms[args.accum_freq] / ms[1]
        res["shapes"].append(row)
        print(json.dumps(row), flush=True)
    rnd = random.Random(0)
    seq = [rnd.choice(pairs) for _ in range(args.seq // args.accum_freq * args.accum_freq)]
    feeds = {key: inputs(args.model, *key, 11) for key in data}
    res["sequence"] = {"steps": len(seq)}
    for k, (_, ts) in arms.items():
        it = iter(seq)
        ms = timed(lambda: ts.step(*feeds[next(it)]), len(seq))
        res["sequence"][f"img_per_s_accum{k}"] = sum(b for _, _, b in seq) / (ms * len(seq) * 1e-3)
    print(json.dumps(res["sequence"]), flush=True)
    n_b3 = arms[1][1].ws.n
    del arms
    torch.cuda.empty_cache()
    res["accumulate_alone"] = {"efficientnet_b3": accumulate_alone(m, n_b3)}
    with torch.device("meta"):  # the parameter count only
        n_clip_h = sum(p.numel() for p in m.CLIP(m.default_clip_opts("huge")).parameters())
    res["accumulate_alone"]["clip_vit_h16"] = accumulate_alone(m, n_clip_h)
    print(json.dumps(res["accumulate_alone"]), flush=True)
    res["card_after"] = card()
    with open(os.path.join(args.outdir, f"multiscale_{args.model}_accum{args.accum_freq}.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "shapes"}))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--model", choices=sorted(TABLES), default="efficientnet_b0")
    ap.add_argument("--steps", type=int, default=20, help="captured replays timed per shape (after 3 untimed)")
    ap.add_argument("--eager-steps", type=int, default=5, help="eager steps timed per shape (after 2 untimed)")
    ap.add_argument("--seq", type=int, default=60, help="length of the random shape sequence")
    ap.add_argument("--accum-freq", type=int, default=1, help="> 1: compare TrainStep(accum_freq=K) with the plain step instead")
    ap.add_argument("--single-arm", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.accum_freq < 1:
        raise SystemExit("--accum-freq must be >= 1")
    if not torch.cuda.is_available():
        raise SystemExit("bench_multiscale needs a CUDA device")
    if args.single_arm:
        print(json.dumps(single_arm(args.model, *(int(v) for v in args.single_arm.split(",")))))
        return
    import ml_cvnets_b200 as m
    os.makedirs(args.outdir, exist_ok=True)
    if args.accum_freq > 1:
        compare_accum(m, args)
        return
    pairs = recipe_pairs(m, args.model)
    res = {"card": card(), "model": args.model, "table": pairs, "skipped": {f"{h}x{w}": why for (h, w), why in SKIP.get(args.model, {}).items()},
           "steps": args.steps, "eager_steps": args.eager_steps, "shapes": []}
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

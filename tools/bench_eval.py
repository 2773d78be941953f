"""Validation throughput of the classification recipes: eager against captured EvalStep passes, live model and EMA twin, and the cost of the
buffer EMA in the captured training step.

    python tools/bench_eval.py OUTDIR [--batches 20] [--steps 20]

Writes OUTDIR/bench_eval.json and prints it:
  * the card (name, power limit, SM clocks) read by nvidia-smi in the same run;
  * per model -- MobileViTv2-1.0 at 256^2, EfficientNet-b0 at 224^2, ViT-B/16 at 224^2, 1000 classes, validation batch 100 -- the eager and
    the captured eval pass of the live model and of the EMA twin (TrainStep.ema_model()): ms per batch (CUDA events over --batches batches
    after warm-up, metrics included) and images/s; the eval graph pool's memory;
  * per model, the captured training step (the recipe's optimizer and EMA momentum 0.0005, training batch 64) with ema_buffers off and on,
    alternated three times, and the difference in ms.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

VAL_BATCH = 100
TRAIN_BATCH = 64
MODELS = {"mobilevit_v2_1.0": 256, "efficientnet_b0": 224, "vit_b16": 224}


def card():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        out = f"nvidia-smi unavailable: {e}"
    return {"query": q, "nvidia_smi": out.splitlines()[0] if out else None, "torch_name": torch.cuda.get_device_name()}


def build(m, name, ema_buffers):
    torch.manual_seed(0)
    if name == "efficientnet_b0":
        model = m.EfficientNet(m.default_effnet_opts("b0", n_classes=1000)).cuda().train()
        return model, m.TrainStep(model, optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None,
                                  label_smoothing=0.1, ema_momentum=0.0005, ema_buffers=ema_buffers)
    if name == "vit_b16":
        model = m.VisionTransformer(m.default_vit_opts("base")).cuda().train()
    else:
        model = m.MobileViTv2(m.default_opts(1.0)).cuda().train()
    return model, m.TrainStep(model, lr=2e-3, weight_decay=0.05, max_norm=10.0, label_smoothing=0.1, ema_momentum=0.0005, ema_buffers=ema_buffers)


def timed(fn, n):
    """ms per call: CUDA events around n calls after the caller's warm-up."""
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    start.record()
    for i in range(n):
        fn(i)
    end.record()
    end.synchronize()
    return start.elapsed_time(end) / n


def eval_numbers(m, model, res, n_batches):
    from ml_cvnets_b200.engine import EvalStep
    g = torch.Generator(device="cuda").manual_seed(1)
    xs = [torch.randn(VAL_BATCH, 3, res, res, device="cuda", generator=g) for _ in range(4)]
    ys = [torch.randint(0, 1000, (VAL_BATCH,), device="cuda", generator=g) for _ in range(4)]
    out = {}
    eager = EvalStep(model)
    for i in range(3):
        eager.update(xs[i % 4], ys[i % 4])
    out["eager_ms"] = timed(lambda i: eager.update(xs[i % 4], ys[i % 4]), n_batches)
    cap = EvalStep(model).capture(batch=VAL_BATCH, crop=(res, res))
    for i in range(3):
        cap.update(xs[i % 4], ys[i % 4])
    out["captured_ms"] = timed(lambda i: cap.update(xs[i % 4], ys[i % 4]), n_batches)
    out["eager_img_s"] = 1000.0 * VAL_BATCH / out["eager_ms"]
    out["captured_img_s"] = 1000.0 * VAL_BATCH / out["captured_ms"]
    out["speedup"] = out["eager_ms"] / out["captured_ms"]
    out["graph_pool_mib"] = cap.graph_pool_bytes() / 2 ** 20
    out["launches_per_batch"] = cap.launches_per_crop[(3, res, res)]
    return out


def captured_train_step(m, name, res, on):
    model, step = build(m, name, on)
    g = torch.Generator(device="cuda").manual_seed(2)
    x = torch.randn(TRAIN_BATCH, 3, res, res, device="cuda", generator=g)
    y = torch.randint(0, 1000, (TRAIN_BATCH,), device="cuda", generator=g)
    step.capture(x, y)
    for _ in range(3):
        step(x, y)
    return model, step, x, y


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--batches", type=int, default=20)
    ap.add_argument("--steps", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_eval.py measures on a CUDA device; none is visible")
    import ml_cvnets_b200 as m
    os.makedirs(a.outdir, exist_ok=True)
    res_all = {"card": card(), "val_batch": VAL_BATCH, "train_batch": TRAIN_BATCH, "models": {}}
    for name, res in MODELS.items():
        r = {"crop": res}
        steps = {on: captured_train_step(m, name, res, on) for on in (False, True)}
        ms = {False: [], True: []}
        for _ in range(3):  # alternate the two steps so that drift of the shared host hits both alike
            for on in (False, True):
                _, st, x, y = steps[on]
                ms[on].append(timed(lambda i: st(x, y), a.steps))
        r["train_step_ms"] = {"ema_buffers_off": ms[False], "ema_buffers_on": ms[True],
                              "extra_ms": min(ms[True]) - min(ms[False]), "launches_off": steps[False][1].launches_per_step,
                              "launches_on": steps[True][1].launches_per_step}
        model, st = steps[True][0], steps[True][1]
        del steps
        r["live"] = eval_numbers(m, model, res, a.batches)
        r["ema"] = eval_numbers(m, st.ema_model(), res, a.batches)
        res_all["models"][name] = r
        del model, st, r
        torch.cuda.synchronize()
        torch.cuda.empty_cache()
    path = os.path.join(a.outdir, "bench_eval.json")
    with open(path, "w") as f:
        json.dump(res_all, f, indent=1)
    print(json.dumps(res_all))


if __name__ == "__main__":
    main()

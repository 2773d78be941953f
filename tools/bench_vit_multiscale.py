"""ViT-B/16 training at the variable-batch sampler's crops (examples/vit/classification/vit_base.yaml: 128-320 px, batch 256 * 224^2 / crop^2).

    python tools/bench_vit_multiscale.py OUTDIR [--steps 10] [--warmup 3]

Writes OUTDIR/vit_multiscale.json and prints it:
  * the card (name, power limit, SM clocks) read by nvidia-smi in the same run;
  * per crop: the captured TrainStep time (fresh model and TrainStep per crop, CUDA events over --steps replays) and img/s;
  * per crop: mha_fwd / mha_bwd alone (CUDA events) with achieved TFLOP/s against the algorithmic 4 B H S^2 64 (forward) and 2.5x that
    (backward), next to torch.nn.functional.scaled_dot_product_attention on the same shapes as a yardstick.
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

CROPS = (128, 160, 192, 224, 256, 288, 320)


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


def step_time(m, crop, B, steps, warmup):
    torch.manual_seed(0)
    model = m.VisionTransformer(m.default_vit_opts("base")).cuda().train()
    ts = m.TrainStep(model, lr=2e-3, weight_decay=0.05, max_norm=10.0, label_smoothing=0.1)
    g = torch.Generator(device="cuda").manual_seed(crop)
    x = torch.randn(B, 3, crop, crop, device="cuda", generator=g)
    y = torch.randint(0, 1000, (B,), device="cuda", generator=g)
    ts.eager_steps = 0
    ts.capture(x, y, warmup=warmup)
    for _ in range(warmup):
        ts.step(x, y)
    ms = timed(lambda: ts.step(x, y), steps)
    loss = float(ts.step(x, y))
    del ts, model
    torch.cuda.empty_cache()
    return ms, loss


def attention_times(ops, B, S, H=12, iters=20):
    c = 64
    g = torch.Generator(device="cuda").manual_seed(S)
    qkv = torch.randn(B * S, 3 * H * c, device="cuda", generator=g).to(torch.bfloat16)
    dO = torch.randn(B * S, H * c, device="cuda", generator=g).to(torch.bfloat16)
    scale = c ** -0.5
    O, LSE = ops.mha_fwd(qkv, B, S, H, c, scale)
    ops.mha_bwd(qkv, O, dO, LSE, B, S, H, c, scale)
    fwd = timed(lambda: ops.mha_fwd(qkv, B, S, H, c, scale), iters)
    bwd = timed(lambda: ops.mha_bwd(qkv, O, dO, LSE, B, S, H, c, scale), iters)
    q, k, v = (t.detach().clone().requires_grad_(True) for t in qkv.view(B, S, 3, H, c).permute(2, 0, 3, 1, 4))
    do = dO.view(B, S, H, c).transpose(1, 2)
    out = F.scaled_dot_product_attention(q, k, v)
    out.backward(do)
    sdpa_fwd = timed(lambda: F.scaled_dot_product_attention(q, k, v), iters)
    out = F.scaled_dot_product_attention(q, k, v)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    total = 0.0
    for _ in range(iters):  # backward alone: a fresh forward per iteration outside the timed window
        out = F.scaled_dot_product_attention(q, k, v)
        e0.record()
        torch.autograd.grad(out, (q, k, v), do)
        e1.record()
        torch.cuda.synchronize()
        total += e0.elapsed_time(e1)
    sdpa_bwd = total / iters
    flop_f = 4.0 * B * H * S * S * c
    flop_b = 2.5 * flop_f
    tf = lambda flop, ms: flop / (ms * 1e-3) / 1e12  # noqa: E731
    return {"kernels": "streaming (mha_long)" if S > 256 else "register-resident (mha_tc)",
            "fwd_ms": fwd, "bwd_ms": bwd, "fwd_tflops": tf(flop_f, fwd), "bwd_tflops": tf(flop_b, bwd),
            "sdpa_fwd_ms": sdpa_fwd, "sdpa_bwd_ms": sdpa_bwd, "sdpa_fwd_tflops": tf(flop_f, sdpa_fwd), "sdpa_bwd_tflops": tf(flop_b, sdpa_bwd)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--crops", default=",".join(str(c) for c in CROPS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_vit_multiscale needs a CUDA device")
    import ml_cvnets_b200 as m
    from ml_cvnets_b200 import ops
    os.makedirs(args.outdir, exist_ok=True)
    res = {"card": card(), "model": "ViT-B/16 bf16 training step (fwd + CE + bwd + clip + AdamW), captured TrainStep", "steps": args.steps, "crops": []}
    for crop in (int(c) for c in args.crops.split(",")):
        B = 256 * 224 * 224 // (crop * crop)
        S = (crop // 16) ** 2 + 1
        ms, loss = step_time(m, crop, B, args.steps, args.warmup)
        row = {"crop": crop, "batch": B, "tokens": S, "step_ms": ms, "img_per_s": B / (ms * 1e-3), "loss": loss,
               "attention": attention_times(ops, B, S)}
        res["crops"].append(row)
        print(json.dumps(row), flush=True)
    res["card_after"] = card()
    with open(os.path.join(args.outdir, "vit_multiscale.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res["card"]), json.dumps(res["card_after"]))


if __name__ == "__main__":
    main()

"""RangeAugment cost on the EfficientNet-B0 recipe (examples/range_augment/classification/efficientnet_b0.yaml): 224^2, B = 256, SGD (momentum 0.9,
Nesterov, weight decay 4e-5), EMA 0.0005, label smoothing 0.1, mixup every step.

    python tools/bench_range_augment.py OUTDIR [--steps 10] [--rounds 3] [--batch 256]

Writes OUTDIR/range_augment.json and prints it:
  * the card (name, power limit, SM clocks) read by nvidia-smi in the same run;
  * the captured TrainStep with and without RangeAugment (+ the NA loss), the two timed in alternating rounds (CUDA events over --steps
    replays each);
  * the new kernels alone at the step's shapes (CUDA events), achieved bytes/s against 3.35 TB/s, bytes = the tensors each must read and
    write once (the image is read once per pass, twice under mixup);
  * eager PyTorch on the same GPU: the tests/efficientnet_ref.py network under bf16 autocast with and without the restated reference augmentor
    and its PSNR loss (tests/range_augment_ref.py, torch's own random draws), forward + backward, alternated; and the augmentor + loss alone.
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
sys.path.insert(0, os.path.join(REPO, "tests"))

HBM = 3.35e12
AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True, "model.learn_augmentation.lr_multiplier": 1.0}


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


def make_step(m, B, res, augment):
    from ml_cvnets_b200.models_effnet import default_effnet_opts
    torch.manual_seed(0)
    model = m.EfficientNet(default_effnet_opts("b0", n_classes=1000, **(AUG if augment else {}))).cuda().train()
    na = m.NeuralAugmentationLoss(target_value=(40, 10), curriculum_method="cosine", period=400) if augment else None
    step = m.TrainStep(model, optimizer="sgd", lr=0.1, weight_decay=4e-5, momentum=0.9, nesterov=True, label_smoothing=0.1, ema_momentum=0.0005,
                       max_norm=None, aug_loss=na)
    step.set_mix("mixup", 0.7)
    x = torch.rand(B, 3, res, res, device="cuda")
    y = torch.randint(0, 1000, (B,), device="cuda")
    step.capture(x, y)
    return step, x, y


def kernels(m, B, H, W):
    ops = m.ops
    x = torch.rand(B, 3, H, W, device="cuda")
    mix = torch.tensor([1.0, 0.7, 0, 0, 0, 0], device="cuda")
    key = torch.tensor([12345], device="cuda", dtype=torch.int64)
    raw = [torch.tensor(v, device="cuda") for v in (0.5, 1.5, 0.5, 1.5, 0.0, 0.1)]
    tab = torch.empty(4 + 3 * B, device="cuda")
    mu = torch.zeros(2, 3 * B, device="cuda", dtype=torch.float64)
    coef = torch.empty(3 * B, 3, device="cuda")
    sq = torch.empty(B, 3, device="cuda", dtype=torch.float64)
    red = torch.empty(3 * B, 3, device="cuda", dtype=torch.float64)
    ops.na_plan(key, B, 7, tab)
    ops.na_stats(x, mix, key, True, mu)
    ops.na_compose(tab, mu, raw, B, coef)
    y = ops.na_apply(x, mix, key, coef, True, sq)
    img = x.numel() * 4
    C0, Ho, Wo = 32, H // 2, W // 2
    dz = torch.randn(B * Ho * Wo, C0, device="cuda").to(torch.bfloat16)
    yb = torch.randn(B * Ho * Wo, C0, device="cuda").to(torch.bfloat16)
    cf = torch.randn(3, C0, device="cuda")
    Ws = torch.randn(C0, 32, device="cuda").to(torch.bfloat16)
    runs = {
        "na_stats": (lambda: ops.na_stats(x, mix, key, True, mu), 2 * img),
        "na_apply": (lambda: ops.na_apply(x, mix, key, coef, True, sq), 3 * img),
        "na_bwd_reduce": (lambda: ops.na_bwd_reduce(y, None, x, mix, key, coef, True, red), 3 * img),
        "stem_dgrad": (lambda: ops.stem_dgrad(dz, yb, cf, Ws, B, Ho, Wo), 2 * dz.numel() * 2 + img),
        "na_plan": (lambda: ops.na_plan(key, B, 7, tab), tab.numel() * 4),
    }
    out = {}
    for name, (fn, nbytes) in runs.items():
        for _ in range(3):
            fn()
        ms = timed(fn, 20)
        out[name] = {"ms": ms, "bytes": nbytes, "TB_per_s": nbytes / ms / 1e9, "share_of_hbm_peak": nbytes / ms / 1e-3 / HBM}
    total_ms = sum(v["ms"] for v in out.values())
    total_bytes = sum(v["bytes"] for v in out.values())
    out["all_new_kernels"] = {"ms": total_ms, "bytes": total_bytes, "share_of_hbm_peak": total_bytes / total_ms / 1e-3 / HBM}
    return out


def _torch_draws(B, H, W):
    """The reference's draws (neural_aug.py:214-236) made with torch's generator on the GPU."""
    import range_augment_ref as R
    nsel = max(1, B // 2)
    order = list(R.NAMES)
    random.shuffle(order)
    draws = {"order": order}
    for name in order:
        d = {"idx": torch.randperm(B, device="cuda")[:nsel], "u": torch.rand(nsel, device="cuda")}
        if name == "noise":
            d["eps"] = torch.randn(nsel, 3, H, W, device="cuda")
        draws[name] = d
    return draws


def eager_reference(B, H, W, n, rounds):
    """The tests/efficientnet_ref.py network in eager PyTorch (bf16 autocast, the reference's AMP path) with and without the restated reference
    augmentor and its PSNR loss: forward + backward per step (no optimizer), the two alternated."""
    import efficientnet_ref as E
    import range_augment_ref as R
    from oracle import cvnets_oracle as O
    P = O.seeded_fill_(E.efficientnet_shapes("b0"), 1)
    P.update(R.seeded_aug_params(2))
    P = O.clone_params(P, device="cuda")
    raw = R.raw_from(P)
    x = torch.rand(B, 3, H, W, device="cuda")
    y = torch.randint(0, 1000, (B,), device="cuda")
    t = R.psnr_to_mse(30.0)

    def once(aug):
        with torch.autocast("cuda", dtype=torch.bfloat16):
            xin = R.augment(x, raw, _torch_draws(B, H, W)) if aug else x
            logits = E.efficientnet_forward(P, xin, mode="b0")
        loss = torch.nn.functional.cross_entropy(logits.float(), y, label_smoothing=0.1)
        if aug:
            loss = loss + R.na_loss(xin, x, t)
        loss.backward()
        for v in P.values():
            v.grad = None

    times = {"without": [], "with": []}
    for aug in (False, True):
        for _ in range(2):
            once(aug)
    for _ in range(rounds):
        for name, aug in (("without", False), ("with", True)):
            times[name].append(timed(lambda: once(aug), n))
    aug_only = {"ms_fwd_bwd": timed(lambda: R.na_loss(R.augment(x, {k: (a.detach().requires_grad_(True), b.detach().requires_grad_(True))
                                                                          for k, (a, b) in raw.items()}, _torch_draws(B, H, W)), x, t).backward(), n)}
    return {"what": "tests/efficientnet_ref.py b0 + tests/range_augment_ref.py augmentor and PSNR loss, eager bf16 autocast, forward + backward, "
                    "no optimizer step", "ms": {k: {"rounds": v, "min": min(v)} for k, v in times.items()},
            "added_by_range_augment_min": min(times["with"]) - min(times["without"]), "augmentor_and_loss_alone": aug_only}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--res", type=int, default=224)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_range_augment.py needs a CUDA device")
    import ml_cvnets_b200 as m
    os.makedirs(a.outdir, exist_ok=True)
    res = {"card": card(), "batch": a.batch, "res": a.res}
    plain = make_step(m, a.batch, a.res, False)
    aug = make_step(m, a.batch, a.res, True)
    times = {"without": [], "with": []}
    for _ in range(a.rounds):
        for name, (step, x, y) in (("without", plain), ("with", aug)):
            step(x, y)
            times[name].append(timed(lambda: step(x, y), a.steps))
    res["step_ms"] = {k: {"rounds": v, "min": min(v)} for k, v in times.items()}
    res["step_ms"]["added_by_range_augment_min"] = min(times["with"]) - min(times["without"])
    res["launches_per_step"] = {"without": plain[0].launches_per_step, "with": aug[0].launches_per_step}
    del plain, aug
    torch.cuda.empty_cache()
    res["kernels"] = kernels(m, a.batch, a.res, a.res)
    res["eager_pytorch_reference"] = eager_reference(a.batch, a.res, a.res, a.steps, a.rounds)
    res["card_after"] = card()
    with open(os.path.join(a.outdir, "range_augment.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""EfficientNet-B0 training step at the recipe's 224^2, B = 256 per GPU (examples/range_augment/classification/efficientnet_b0.yaml): forward,
cross entropy with label smoothing 0.1, backward, SGD (momentum 0.9, Nesterov, weight decay 4e-5 without BN / bias decay) and EMA 0.0005.

    python tools/bench_efficientnet.py OUTDIR [--steps 10] [--warmup 3] [--batch 256]

Writes OUTDIR/efficientnet.json and prints it:
  * the card (name, power limit, SM clocks) read by nvidia-smi in the same run;
  * the captured TrainStep (CUDA events over --steps replays) and img/s;
  * the same model in eager PyTorch on the same GPU: a torch restatement with torch's own layers (bf16 autocast, channels_last,
    torch.optim.SGD, EMA as torch ops) -- the yardstick;
  * the depthwise 5x5 kernels alone at every b0 shape (forward with BN statistics, fused backward with BNB gradient and dW), CUDA events,
    achieved bytes/s against 3.35 TB/s (bytes = the tensors each kernel must read and write once).
"""
import argparse
import json
import os
import subprocess
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, REPO)

HBM = 3.35e12


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


class _TorchBlock(nn.Module):
    """EfficientNetBlock restated with torch layers (same arithmetic as cvnets/modules/efficientnet.py, stochastic depth 0)."""

    def __init__(self, e, k, s, ci, co):
        super().__init__()
        from ml_cvnets_b200.modules import make_divisible
        hid = make_divisible(int(round(ci * e)), 8)
        sq = max(make_divisible(hid // (4 * e), 8), 32)
        layers = [] if e == 1 else [nn.Conv2d(ci, hid, 1, bias=False), nn.BatchNorm2d(hid), nn.SiLU()]
        layers += [nn.Conv2d(hid, hid, k, s, (k - 1) // 2, groups=hid, bias=False), nn.BatchNorm2d(hid), nn.SiLU()]
        self.pre = nn.Sequential(*layers)
        self.fc1, self.fc2 = nn.Conv2d(hid, sq, 1), nn.Conv2d(sq, hid, 1)
        self.red = nn.Sequential(nn.Conv2d(hid, co, 1, bias=False), nn.BatchNorm2d(co))
        self.res = s == 1 and ci == co

    def forward(self, x):
        h = self.pre(x)
        h = h * torch.sigmoid(self.fc2(F.silu(self.fc1(h.mean((2, 3), keepdim=True)))))
        h = self.red(h)
        return x + h if self.res else h


def torch_b0(n_classes=1000):
    from ml_cvnets_b200.models_effnet import default_effnet_opts, get_effnet_configuration, LAYERS
    cfg = get_effnet_configuration(default_effnet_opts("b0"))
    blocks = []
    for name in LAYERS:
        for e, k, s, ci, co, n in cfg[name]:
            for i in range(n):
                blocks.append(_TorchBlock(e, k, s if i == 0 else 1, ci if i == 0 else co, co))
    return nn.Sequential(nn.Conv2d(3, 32, 3, 2, 1, bias=False), nn.BatchNorm2d(32), nn.SiLU(), *blocks,
                         nn.Conv2d(cfg["layer_5"][-1][4], cfg["last_channels"], 1, bias=False), nn.BatchNorm2d(cfg["last_channels"]), nn.SiLU(),
                         nn.AdaptiveAvgPool2d(1), nn.Flatten(), nn.Linear(cfg["last_channels"], n_classes))


def bench_ours(B, steps, warmup):
    import ml_cvnets_b200 as m
    torch.manual_seed(0)
    model = m.EfficientNet(m.default_effnet_opts("b0")).cuda()
    ts = m.TrainStep(model, optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None, label_smoothing=0.1,
                     ema_momentum=0.0005)
    x = torch.randn(B, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (B,), device="cuda")
    ts.capture(x, y, warmup=warmup)
    for _ in range(warmup):
        ts(x, y)
    ms = timed(lambda: ts(x, y), steps)
    loss = float(ts(x, y))
    del ts, model
    torch.cuda.empty_cache()
    return {"ms": ms, "img_s": B / ms * 1e3, "loss": loss}


def bench_eager(B, steps, warmup):
    torch.manual_seed(0)
    model = torch_b0().cuda().to(memory_format=torch.channels_last)
    decay = [p for p in model.parameters() if p.dim() > 1]
    no_decay = [p for p in model.parameters() if p.dim() == 1]
    opt = torch.optim.SGD([{"params": decay, "weight_decay": 4e-5}, {"params": no_decay, "weight_decay": 0.0}], lr=0.1, momentum=0.9, nesterov=True)
    scaler = torch.amp.GradScaler("cuda")
    ema = [p.detach().clone() for p in model.parameters()]
    x = torch.randn(B, 3, 224, 224, device="cuda").contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, 1000, (B,), device="cuda")

    def step():
        opt.zero_grad(set_to_none=True)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(model(x), y, label_smoothing=0.1)
        scaler.scale(loss).backward()
        scaler.step(opt)
        scaler.update()
        with torch.no_grad():
            torch._foreach_lerp_(ema, [p.detach() for p in model.parameters()], 0.0005)

    for _ in range(warmup):
        step()
    ms = timed(step, steps)
    del model, opt
    torch.cuda.empty_cache()
    return {"ms": ms, "img_s": B / ms * 1e3}


def bench_dw5(B, reps):
    """Every b0 5x5 depthwise shape: (C, H_in, stride)."""
    from ml_cvnets_b200 import ops
    shapes = [(144, 56, 2), (240, 28, 1), (240, 28, 2), (672, 14, 1), (672, 14, 2), (1152, 7, 1)]
    out = []
    for C, H, s in shapes:
        Ho = (H - 1) // s + 1
        x = torch.randn(B * H * H, C, device="cuda").bfloat16()
        Wt = torch.randn(25, C, device="cuda").bfloat16().float()
        p = (torch.rand(C, device="cuda") + 0.5, 0.1 * torch.randn(C, device="cuda"), 0.1 * torch.randn(C, device="cuda"))
        st = torch.zeros(2, C, device="cuda", dtype=torch.float64)
        y = ops.dw_fwd(x, B, H, H, C, s, Wt, col_stats=st, ksize=5)
        dz = torch.randn_like(y)
        dW = torch.zeros(25, C, device="cuda")
        fwd = lambda: ops.dw_fwd(x, B, H, H, C, s, Wt, col_stats=st, ksize=5)  # noqa: E731
        bwd = lambda: ops.dw_bwd(dz, x, B, H, H, C, s, Wt, g_mode=ops.A_BNB, Y2=y, g_p=p, dWt=dW, ksize=5)  # noqa: E731
        fwd(), bwd()
        t_f, t_b = timed(fwd, reps), timed(bwd, reps)
        nx, ny = B * H * H * C * 2, B * Ho * Ho * C * 2
        out.append({"C": C, "H": H, "stride": s, "B": B, "fwd_us": t_f * 1e3, "fwd_TBps": (nx + ny) / t_f / 1e9, "fwd_of_hbm": (nx + ny) / t_f / 1e9 / (HBM / 1e12),
                    "bwd_us": t_b * 1e3, "bwd_TBps": (2 * nx + 2 * ny) / t_b / 1e9, "bwd_of_hbm": (2 * nx + 2 * ny) / t_b / 1e9 / (HBM / 1e12)})
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--batch", type=int, default=256)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_efficientnet.py measures on a CUDA device; none is visible")
    torch.backends.cudnn.benchmark = True
    res = {"card": card(), "batch": args.batch, "resolution": 224, "steps": args.steps}
    res["ours_captured_step"] = bench_ours(args.batch, args.steps, args.warmup)
    res["eager_torch_step"] = bench_eager(args.batch, args.steps, args.warmup)
    res["speedup_vs_eager"] = res["eager_torch_step"]["ms"] / res["ours_captured_step"]["ms"]
    res["dw5_kernels"] = bench_dw5(args.batch, 20)
    res["card_after"] = card()
    os.makedirs(args.outdir, exist_ok=True)
    with open(os.path.join(args.outdir, "efficientnet.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps(res))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""bench.py -- images/sec of a MobileViTv2-1.0 bf16 256x256 training step (BASELINE.json metric) on N H100s.

    python bench.py [--gpus N] [--steps K] [--warmup W] [--batch B] [--impl ours|reference]
    python -m torch.distributed.run --nnodes=1 --nproc-per-node N --master-addr 127.0.0.1 --master-port P bench.py --gpus N ...

One "step" = forward + cross-entropy(label_smoothing 0.1) + backward (+ DDP gradient all-reduce over NCCL at N > 1) +
GradScaler unscale + clip_grad_norm_(10) + AdamW step, per-GPU batch 128 (config/classification/imagenet/mobilevit_v2.yaml
:9,15 of the reference), synthetic ImageNet-shaped tensors, random-init weights.

Prints ONE JSON line (rank 0).  ``value`` = whole-job images/s with inputs resident in HBM; ``e2e`` = same metric with the
step's images+labels copied from pinned host memory and the loss read back inside the timed region; ``roofline`` =
algorithmic bytes of the pointwise-conv GEMM kernel family (the dominant kernel) / their CUDA-event time vs measured HBM
peak; ``cpu_baseline`` = the oracle (CPU restatement of the reference path) timed on a bounded sample on the host cores.
``--impl reference`` times that CPU path alone (the reference is pure Python/PyTorch; its nn.Module path == the oracle).
``--dump-outputs DIR`` writes what the last step of the first timed region computed -- the loss and the updated parameters -- as
float32 ``DIR/<name>.npy``; the inputs and the initial weights are seeded, so two builds can be compared output for output.
"""
import argparse
import json
import os
import subprocess
import sys
import threading
import time

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

_JSON_FD = None


def quiet_stdout():
    """The contract is ONE JSON line on stdout: route everything else that libraries print there (e.g. the "NCCL version ..." banner)
    to stderr by pointing fd 1 at fd 2 for the duration of the run; emit() writes the result to the saved original stdout."""
    global _JSON_FD
    if _JSON_FD is None:
        sys.stdout.flush()
        _JSON_FD = os.dup(1)
        os.dup2(2, 1)


def emit(line: dict):
    data = (json.dumps(line) + "\n").encode()
    if _JSON_FD is None:
        sys.stdout.write(data.decode())
        sys.stdout.flush()
    else:
        sys.stdout.flush()
        os.write(_JSON_FD, data)


METRIC = "images/sec training step, MobileViTv2-1.0 bf16 256x256"  # BASELINE.json metric (the --width 2.0 run is configs[3], named in config.workload)
RES, NCLS = 256, 1000


def measured_peaks():
    p = os.path.join(ROOT, "MEASURED_PEAKS.json")
    if os.path.exists(p):
        with open(p) as f:
            d = json.load(f)
        return float(d["hbm_gbs"]), "measured (MEASURED_PEAKS.json hbm_gbs)"
    return 3350.0, "fallback (H100 SXM data sheet, 3.35 TB/s)"


class ClockSampler:
    """nvidia-smi clocks / throttle reasons during the timed region."""

    def __init__(self, gpu_index=0):
        self.proc, self.lines, self.gpu = None, [], gpu_index

    def start(self):
        q = ("clocks.sm,clocks.max.sm,power.draw,clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
             "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap")
        try:
            self.proc = subprocess.Popen(["nvidia-smi", f"--id={self.gpu}", f"--query-gpu={q}", "--format=csv,noheader,nounits", "-lms", "100"],
                                         stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True)
            self.t = threading.Thread(target=self._read, daemon=True)
            self.t.start()
        except Exception:
            self.proc = None

    def _read(self):
        for line in self.proc.stdout:
            self.lines.append(line.strip())

    def stop(self):
        if self.proc is None:
            return {"sm_mhz": None, "sm_max_mhz": None, "reasons": ["nvidia-smi unavailable"]}
        self.proc.terminate()
        try:
            self.proc.wait(timeout=2)
        except Exception:
            pass
        sm, mx, reasons = [], None, set()
        for ln in self.lines:
            f = [x.strip() for x in ln.split(",")]
            if len(f) < 7:
                continue
            try:
                sm.append(float(f[0]))
                mx = float(f[1])
            except ValueError:
                continue
            for name, v in zip(["hw_slowdown", "hw_thermal_slowdown", "sw_thermal_slowdown", "sw_power_cap"], f[3:7]):
                if v.lower().startswith("active"):
                    reasons.add(name)
        sm.sort()
        return {"sm_mhz": sm[len(sm) // 2] if sm else None, "sm_max_mhz": mx, "reasons": sorted(reasons), "samples": len(sm)}


DUMP_MAX_PARAMS = 8 * 1024 * 1024  # 32 MB of float32: larger models dump a fixed seeded sample of their parameters


def output_snapshot(loss, model):
    """What a caller of the timed step receives: the step's loss and the updated parameters (flattened in model.parameters() order;
    beyond DUMP_MAX_PARAMS elements, the same seeded sample of positions on every run)."""
    with torch.no_grad():
        flat = torch.cat([p.detach().float().flatten() for p in model.parameters()])
        if flat.numel() > DUMP_MAX_PARAMS:
            idx = torch.randperm(flat.numel(), generator=torch.Generator().manual_seed(0))[:DUMP_MAX_PARAMS].sort().values
            flat = flat[idx.to(flat.device)]
        return {"loss": loss.detach().float().reshape(1).clone(), "params": flat.clone()}


def write_outputs(out_dir, outputs):
    import numpy as np
    os.makedirs(out_dir, exist_ok=True)
    for name, t in outputs.items():
        np.save(os.path.join(out_dir, name + ".npy"), t.cpu().numpy().astype(np.float32))


# ------------------------------------------------------------------------------------------------ CPU (reference) arm
ALGO_MB_PER_IMAGE = {1.0: 190.8, 2.0: 380.5}  # SURVEY.md 8d: 3 x (sum of conv/linear in+out activation elements) x 2 B


def workload_config(width, B, world):
    """The workload description BOTH arms print (identical dict => the driver's same_config check can pass)."""
    cfg_no = {1.0: 1, 2.0: 3}.get(width)
    return {"workload": f"MobileViTv2-{width:.1f} bf16 training step, synthetic ImageNet 256x256"
                        + (f" (BASELINE.json configs[{cfg_no}])" if cfg_no is not None else ""),
            "per_gpu_batch": B, "global_batch": B * world, "parallelism": f"dp{world}", "resolution": RES,
            "l2": "activations per step (>7 GB at batch 128) exceed the 50 MB L2; no explicit flush"}


def usable_cores():
    """Cores this process may really use: the affinity mask capped by the cgroup CPU quota (a container can expose 128 CPUs in its mask
    and be throttled to a handful; oversubscribing them made round 1's CPU numbers vary 21x between boxes)."""
    n = len(os.sched_getaffinity(0)) if hasattr(os, "sched_getaffinity") else (os.cpu_count() or 1)
    for path in ("/sys/fs/cgroup/cpu.max", "/sys/fs/cgroup/cpu/cpu.cfs_quota_us"):
        try:
            with open(path) as f:
                txt = f.read().split()
            if path.endswith("cpu.max"):
                quota, period = txt[0], float(txt[1])
            else:
                quota = txt[0]
                with open("/sys/fs/cgroup/cpu/cpu.cfs_period_us") as f:
                    period = float(f.read().split()[0])
            if quota not in ("max", "-1"):
                n = min(n, max(1, int(-(-float(quota) // period))))
            break
        except Exception:
            continue
    return max(1, n)


class CpuArm:
    """The reference's own nn.Module path restated by the oracle (fp32: the reference refuses AMP on CPU, engine/utils.py:31-32):
    forward + CE(label_smoothing 0.1) + backward + AdamW(lr 2e-3, wd 0.05) on the host cores."""

    def __init__(self, width=1.0):
        from oracle import cvnets_oracle as O
        self.O, self.width = O, width
        self.P = O.clone_params(O.seeded_fill_(O.mobilevit_v2_shapes(width), 0))
        self.opt = torch.optim.AdamW([v for v in self.P.values() if v.requires_grad], lr=2e-3, weight_decay=0.05)
        self.gen = torch.Generator().manual_seed(0)

    def batch(self, b):
        return torch.randn(b, 3, RES, RES, generator=self.gen), torch.randint(0, NCLS, (b,), generator=self.gen)

    def step(self, x, y):
        t0 = time.perf_counter()
        self.O.training_step(self.P, self.opt, x, y, width_multiplier=self.width)
        return time.perf_counter() - t0

    def calibrate_threads(self, budget_s=45.0):
        """Pick the torch thread count that is fastest on THIS box (hyper-threads / noisy neighbours make 'all of them' a bad default):
        one warm + one timed 2-image step per candidate, smallest first, stop when it gets slower or the budget is spent."""
        cores = usable_cores()
        cands = sorted({min(cores, c) for c in (4, 8, 16, 32, 64, cores)})
        x, y = self.batch(2)
        t_start, best, log = time.perf_counter(), None, []
        for c in cands:
            torch.set_num_threads(c)
            self.step(x, y)
            dt = min(self.step(x, y), self.step(x, y)) if (time.perf_counter() - t_start) < 0.5 * budget_s else self.step(x, y)
            ips = 2.0 / dt
            log.append((c, round(ips, 3)))
            if best is None or ips > best[1]:
                best = (c, ips)
            elif ips < 0.9 * best[1]:
                break
            if time.perf_counter() - t_start > budget_s:
                break
        torch.set_num_threads(best[0])
        return best[0], best[1], cores, log


def cpu_training_throughput(width, steps, warmup, budget_s, max_batch=128):
    """Bounded CPU measurement.  Thread count calibrated on this box; the per-step sample is sized from a probe at batch 8 (per-image cost
    grows with the batch on these hosts: a 2-image probe over-estimated the rate 3x in round 2's first run); every step is timed and the
    loop stops -- saying so in the line -- as soon as the wall-clock budget is spent.  Returns a dict."""
    arm = CpuArm(width)
    t0 = time.perf_counter()
    threads, probe_ips, cores, calib = arm.calibrate_threads(budget_s=min(40.0, 0.3 * budget_s))
    xb, yb = arm.batch(min(8, max_batch))
    arm.step(xb, yb)
    probe_ips = min(probe_ips, xb.shape[0] / arm.step(xb, yb))
    remaining = max(10.0, budget_s - (time.perf_counter() - t0))
    total = max(1, steps + warmup)
    batch = int(max(1, min(max_batch, 0.8 * probe_ips * remaining / total)))
    x, y = arm.batch(batch)
    t_loop, times, warm_done = time.perf_counter(), [], 0
    for i in range(total):
        dt = arm.step(x, y)
        left = remaining - (time.perf_counter() - t_loop)
        if i < warmup and left >= 2.0 * dt:  # untimed warm-up, as long as at least one timed step still fits afterwards
            warm_done += 1
        else:
            times.append(dt)
        if len(times) >= steps or left < 1.1 * dt:
            break
    dt = sum(times) / len(times)
    return {"ips": batch / dt, "ms": dt * 1e3, "threads": threads, "cores_available": cores, "batch": batch, "steps": len(times),
            "warmup": warm_done, "calibration": calib}


def run_reference_arm(args, rank, world):
    """`--impl reference`: the reference's own CPU implementation of the path (oracle port), on the box's host cores, wall-clock bounded
    (~2.5 minutes in total regardless of how slow the host is).  Under torchrun only rank 0 works."""
    if rank != 0:
        return
    r = cpu_training_throughput(args.width, args.steps, args.warmup, budget_s=args.cpu_budget)
    sample = (f"batch {r['batch']} of the per-GPU batch of {args.batch}, fwd+bwd+AdamW, fp32, {r['threads']} torch threads "
              f"(calibrated; {r['cores_available']} usable cores)")
    line = {
        "impl": "reference", "metric": METRIC, "value": r["ips"], "unit": "images/sec", "n_gpus": args.gpus, "steps": r["steps"],
        "warmup": r["warmup"], "ms_per_step": r["ms"], "higher_is_better": True, "scaling": "weak", "vs_baseline": None,
        "dtype": "fp32 (reference refuses AMP on CPU)", "data": "synthetic",
        "config": workload_config(args.width, args.batch, world),
        "requested": {"steps": args.steps, "warmup": args.warmup},
        "cpu_baseline": {"value": r["ips"], "unit": "images/sec", "cores": r["threads"], "kind": "port", "sample": sample,
                         "thread_calibration_img_s": r["calibration"]},
        "e2e": {"value": r["ips"], "unit": "images/sec", "h2d_bytes_per_step": 0, "d2h_bytes_per_step": 0},
        "gpu_launches": 0,
    }
    emit(line)


# ------------------------------------------------------------------------------------------- eager-GPU comparator
def gpu_eager_baseline(dev, B, width, steps, warmup):
    """SURVEY.md 8d / BASELINE.md 3: the reference modules' own GPU path = PyTorch eager (cuDNN / cuBLAS) under bf16 autocast +
    channels_last + GradScaler + clip_grad_norm_(10) + AdamW(fused), same batch, same step definition (protocol of the reference's
    main_benchmark.py:94-117 extended with backward + optimizer as engine/training_engine.py:257-312).  The reference cannot travel to
    the GPU box, so its restatement (the oracle, pinned to the reference by tests/golden) stands in.  Timed eagerly (what a reference
    user gets) and as ONE CUDA graph (host overhead removed: the stronger comparator)."""
    from oracle import cvnets_oracle as O
    P = O.clone_params(O.seeded_fill_(O.mobilevit_v2_shapes(width), 0), device=dev)
    for k, v in list(P.items()):
        if v.dim() == 4:
            P[k] = v.detach().contiguous(memory_format=torch.channels_last).requires_grad_(True)
    decay = [v for v in P.values() if v.requires_grad and v.dim() > 1]
    no_decay = [v for v in P.values() if v.requires_grad and v.dim() <= 1]
    params = decay + no_decay
    gen = torch.Generator(device=dev).manual_seed(99)
    x = torch.randn(B, 3, RES, RES, device=dev, generator=gen).contiguous(memory_format=torch.channels_last)
    y = torch.randint(0, NCLS, (B,), device=dev, generator=gen)

    def make(capturable):
        opt = torch.optim.AdamW([{"params": decay, "weight_decay": 0.05}, {"params": no_decay, "weight_decay": 0.0}], lr=2e-3,
                                betas=(0.9, 0.999), fused=True, capturable=capturable)
        scaler = torch.amp.GradScaler("cuda", enabled=True)

        def step():
            with torch.autocast("cuda", dtype=torch.bfloat16):
                logits = O.mobilevit_v2_forward(P, x, width_multiplier=width, training=True)
                loss = F.cross_entropy(logits, y, label_smoothing=0.1)
            opt.zero_grad(set_to_none=True)
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
            torch.nn.utils.clip_grad_norm_(params, 10.0)
            scaler.step(opt)
            scaler.update()
            return loss
        return step

    def timed(fn, n):
        torch.cuda.synchronize(dev)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        torch.cuda.synchronize(dev)
        return e0.elapsed_time(e1) / n

    out = {"what": "oracle restatement of the reference modules, torch eager bf16 autocast + channels_last + GradScaler + clip 10 + AdamW(fused)",
           "per_gpu_batch": B, "unit": "images/sec"}
    step = make(False)
    for _ in range(max(3, warmup)):
        step()
    ms = timed(step, steps)
    out.update({"value": B / (ms * 1e-3), "ms_per_step": ms, "steps": steps})
    try:
        gstep = make(True)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            for _ in range(3):
                gstep()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize(dev)
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            gstep()
        for _ in range(3):
            g.replay()
        gms = timed(g.replay, steps)
        out.update({"graphed_value": B / (gms * 1e-3), "graphed_ms_per_step": gms})
        del g
    except Exception as e:  # the comparator must never take the bench line down
        out["graphed_error"] = repr(e)[:200]
    del P
    torch.cuda.empty_cache()
    return out


# --------------------------------------------------------------------------------------------------------- our arm
class GemmTimer:
    """CUDA-event timing of every cvb_pw_gemm launch (the dominant kernel family) inside the timed region."""

    def __init__(self, ops):
        self.ops, self.records, self.enabled = ops, [], False
        self._orig = ops.pw_gemm

    def install(self):
        ops, timer = self.ops, self

        def timed_pw_gemm(A, W, N, **kw):
            if not timer.enabled:
                return timer._orig(A, W, N, **kw)
            s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            s.record()
            out = timer._orig(A, W, N, **kw)
            e.record()
            M, K = A.shape[0], kw.get("K") or A.shape[1]
            # algorithmic bytes (SURVEY.md 8d): input activation read once + output written once, bf16
            timer.records.append((s, e, 2.0 * M * (K + N), 2.0 * M * K * N, (M, N, K, kw.get("a_mode", 0), kw.get("e_mode", 0))))
            return out

        ops.pw_gemm = timed_pw_gemm
        import ml_cvnets_b200.functional as Fn
        Fn.ops.pw_gemm = timed_pw_gemm

    def summary(self):
        ms = sum(r[0].elapsed_time(r[1]) for r in self.records)
        byts = sum(r[2] for r in self.records)
        flops = sum(r[3] for r in self.records)
        return ms, byts, flops, len(self.records)

    def per_shape(self, steps):
        agg = {}
        for r in self.records:
            a = agg.setdefault(r[4], [0, 0.0, r[2]])
            a[0] += 1
            a[1] += r[0].elapsed_time(r[1])
        out = [{"M,N,K,a_mode,e_mode": list(k), "n_per_step": v[0] / steps, "us_each": 1e3 * v[1] / v[0], "GBps": v[2] / (v[1] / v[0]) / 1e6}
               for k, v in agg.items()]
        return sorted(out, key=lambda d: -d["us_each"] * d["n_per_step"])


class OpTimer:
    """Optional (--profile-ops): CUDA-event time of every C-ABI launch, aggregated per entry point (diagnostics only)."""

    NAMES = ["pw_gemm", "pw_wgrad", "dw_fwd", "dw_bwd", "stem_im2col", "bn_finalize", "bn_bwd_finalize", "bn_apply", "bn_bwd_reduce",
             "gn_finalize", "gn_bwd_apply", "linattn_fwd", "linattn_bwd", "global_pool_fwd", "global_pool_bwd", "unprep_grad"]

    def __init__(self, ops):
        self.ops, self.rec = ops, []

    def install(self):
        import ml_cvnets_b200.functional as Fn
        for name in self.NAMES:
            orig = getattr(self.ops, name)

            def wrapped(*a, _orig=orig, _name=name, **kw):
                s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                s.record()
                out = _orig(*a, **kw)
                e.record()
                shape = tuple(tuple(x.shape) for x in a if isinstance(x, torch.Tensor))[:2] + tuple(x for x in a if isinstance(x, int))[:5]
                self.rec.append((_name, s, e, shape))
                return out

            setattr(self.ops, name, wrapped)
            setattr(Fn.ops, name, wrapped)

    def summary(self, steps):
        agg, shp = {}, {}
        for name, s, e, shape in self.rec:
            t = s.elapsed_time(e)
            a = agg.setdefault(name, [0, 0.0])
            a[0] += 1
            a[1] += t
            if name in ("pw_wgrad", "dw_fwd", "dw_bwd"):
                b = shp.setdefault(name + str(shape), [0, 0.0])
                b[0] += 1
                b[1] += t
        out = {k: {"n_per_step": v[0] / steps, "ms_per_step": v[1] / steps} for k, v in sorted(agg.items(), key=lambda kv: -kv[1][1])}
        out["_by_shape"] = {k: {"n_per_step": v[0] / steps, "us_each": 1e3 * v[1] / v[0]} for k, v in sorted(shp.items(), key=lambda kv: -kv[1][1])[:40]}
        return out


def run_ours(args, rank, world, local_rank):
    import ml_cvnets_b200 as m
    from ml_cvnets_b200 import ops
    from ml_cvnets_b200 import dist as D

    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    torch.manual_seed(0 + rank)
    B = args.batch
    model = m.MobileViTv2(m.default_opts(width_multiplier=args.width)).to(dev).train()
    if args.no_pdl:
        ops.set_pdl_enabled(False)
    use_graph = not args.no_graph and not args.profile_ops
    ts = None
    if args.torch_optim:
        # A/B path (one GPU): the torch pipeline of round 1 -- F.cross_entropy, GradScaler, clip_grad_norm_, torch.optim.AdamW(fused)
        assert world == 1, "--torch-optim is a single-GPU comparison path"
        groups, _ = model.get_trainable_parameters(weight_decay=0.05, no_decay_bn_filter_bias=True)
        params = [p for p in model.parameters()]
        opt = torch.optim.AdamW(groups, lr=2e-3, betas=(0.9, 0.999), fused=True, capturable=use_graph)
        scaler = torch.amp.GradScaler("cuda", enabled=True)  # the reference enables it even for bf16 (main_train.py:114)

        def step(x, y):
            logits = model(x)
            loss = F.cross_entropy(logits.float(), y, label_smoothing=0.1)
            opt.zero_grad(set_to_none=True)
            scaler.scale(loss).backward()
            scaler.unscale_(opt)
            torch.nn.utils.clip_grad_norm_(params, 10.0)
            scaler.step(opt)
            scaler.update()
            return loss
    else:
        # the product path: engine.TrainStep = forward + cvb_ce loss + backward writing into one flat gradient buffer + bucketed NCCL
        # all-reduce overlapped with backward (N > 1) + two-launch unscale/clip/AdamW(+EMA)/scaler tail; no ATen kernel in the step
        ts = m.TrainStep(model, lr=2e-3, betas=(0.9, 0.999), weight_decay=0.05, no_decay_bn_filter_bias=True, max_norm=10.0, label_smoothing=0.1,
                         ema_momentum=(0.0005 if args.ema else None), n_buckets=args.buckets)
        step = ts._step

    gen = torch.Generator(device=dev).manual_seed(1234 + rank)
    x_dev = torch.randn(B, 3, RES, RES, device=dev, generator=gen)
    y_dev = torch.randint(0, NCLS, (B,), device=dev, generator=gen)

    def sync_all():
        torch.cuda.synchronize(dev)
        if world > 1:
            torch.distributed.barrier()
            torch.cuda.synchronize(dev)

    def max_over_ranks(ms):
        if world == 1:
            return ms
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        return float(t.item())

    for _ in range(max(args.warmup, 3)):
        step(x_dev, y_dev)
    # ---- whole training step as ONE CUDA graph: fwd + loss + bwd (+ bucketed NCCL all-reduce at N > 1) + optimizer tail.
    # Kernel arguments (incl. TMA tensor maps) are baked at capture; inputs live in static buffers.
    if use_graph:
        if ts is not None:
            ts.eager_steps = max(args.warmup, 3)
            ts.capture(x_dev, y_dev)
            static_x, static_y = ts.static_inputs
            launches_per_graph = ts.launches_per_step
            run_step = ts.step
        else:
            static_x, static_y = x_dev.clone(), y_dev.clone()
            torch.cuda.synchronize(dev)
            side = torch.cuda.Stream(device=dev)
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(2):
                    step(static_x, static_y)
            torch.cuda.current_stream().wait_stream(side)
            torch.cuda.synchronize(dev)
            graph = torch.cuda.CUDAGraph()
            model.zero_grad(set_to_none=True)
            launches_before_capture = ops.launch_count
            with torch.cuda.graph(graph):
                static_loss = step(static_x, static_y)
            launches_per_graph = ops.launch_count - launches_before_capture

            def run_step(x, y):
                if x is not static_x:
                    static_x.copy_(x, non_blocking=True)
                    static_y.copy_(y, non_blocking=True)
                graph.replay()
                return static_loss

        for _ in range(max(10, args.warmup)):  # settle the replay path (NCCL inside the graph needs more than a couple of replays)
            run_step(static_x, static_y)
    else:
        run_step = step
        launches_per_graph = None
    timer = GemmTimer(ops)
    if not args.no_kernel_timing and not use_graph:
        timer.install()
    optimer = None
    if args.profile_ops:
        optimer = OpTimer(ops)
        optimer.install()
    sampler = ClockSampler(local_rank)
    # ---------------- timed region 1: inputs resident in HBM
    # The sampler is started BEFORE the barrier: spawning nvidia-smi takes 10-100 ms of host time on rank 0; after the barrier that delay would
    # make every other rank wait at its first all-reduce inside ITS timed region and inflate the max over ranks.
    if rank == 0:
        sampler.start()
    sync_all()
    timer.enabled = not args.no_kernel_timing and not use_graph
    launches0 = ops.launch_count
    marks = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    marks[0].record()
    for i in range(args.steps):
        if args.profile_ops:
            torch.cuda._sleep(int(0.25 * 1.9e9))  # diagnostics only: queue the step behind a spin so op timings exclude launch gaps
        loss = run_step(static_x, static_y) if use_graph else step(x_dev, y_dev)
        if args.profile_ops:
            torch.cuda.synchronize(dev)
        marks[i + 1].record()
    ev0, ev1 = marks[0], marks[-1]
    sync_all()
    outputs = output_snapshot(loss, model) if args.dump_outputs else None
    per_step = sorted(marks[i].elapsed_time(marks[i + 1]) for i in range(args.steps))
    step_stats = {"min": per_step[0], "median": per_step[len(per_step) // 2], "p90": per_step[min(len(per_step) - 1, int(0.9 * len(per_step)))],
                  "max": per_step[-1], "note": "rank 0's CUDA-event time of each timed step"}
    if world > 1:  # slowest rank's view of the same statistics (a straggler shows up here, not only in the max-over-ranks total)
        step_stats["max_over_ranks"] = {"median": max_over_ranks(step_stats["median"]), "max": max_over_ranks(step_stats["max"])}
    timer.enabled = False
    launches = (launches_per_graph * args.steps) if use_graph else (ops.launch_count - launches0)
    op_ms = optimer.summary(args.steps) if optimer is not None else None
    if optimer is not None:
        optimer.rec = []
    clocks = sampler.stop() if rank == 0 else None
    ms_total = max_over_ranks(ev0.elapsed_time(ev1))
    ms_step = ms_total / args.steps
    value = world * B / (ms_step * 1e-3)
    final_loss = float(loss.detach())

    # ---------------- timed region 2: end to end (pinned host -> device every step, loss read back every step)
    nbuf = 2
    hx = [torch.randn(B, 3, RES, RES).pin_memory() for _ in range(nbuf)]
    hy = [torch.randint(0, NCLS, (B,)).pin_memory() for _ in range(nbuf)]
    dx = [torch.empty_like(x_dev) for _ in range(nbuf)]
    dy = [torch.empty_like(y_dev) for _ in range(nbuf)]
    copy_stream = torch.cuda.Stream(device=dev)
    ready = [torch.cuda.Event() for _ in range(nbuf)]
    consumed = [torch.cuda.Event() for _ in range(nbuf)]
    hloss = torch.zeros(1).pin_memory()

    def prefetch(i):
        b = i % nbuf
        with torch.cuda.stream(copy_stream):
            copy_stream.wait_event(consumed[b])
            dx[b].copy_(hx[b], non_blocking=True)
            dy[b].copy_(hy[b], non_blocking=True)
            ready[b].record(copy_stream)

    e2e_steps = args.steps
    for b in range(nbuf):
        consumed[b].record()
    sync_all()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    prefetch(0)
    for i in range(e2e_steps):
        b = i % nbuf
        if i + 1 < e2e_steps:
            prefetch(i + 1)
        torch.cuda.current_stream().wait_event(ready[b])
        loss = run_step(dx[b], dy[b])
        consumed[b].record()
        hloss.copy_(loss.detach().reshape(1), non_blocking=True)
        torch.cuda.current_stream().synchronize()  # the user reads the loss every step
        _ = float(hloss[0])
    e1.record()
    sync_all()
    e2e_ms = max_over_ranks(e0.elapsed_time(e1)) / e2e_steps
    e2e_value = world * B / (e2e_ms * 1e-3)
    h2d = world * (hx[0].numel() * 4 + hy[0].numel() * 8)
    d2h = world * 4

    if use_graph and not args.no_kernel_timing:
        # the dominant-kernel timing needs CUDA events around individual launches: a short eager pass right after the timed
        # region (same process, same tensors; kernels and shapes identical to the ones baked into the graph)
        timer.install()
        timer.enabled = True
        # eager launches are CPU-bound here; a GPU-side spin first lets the host queue the whole step so that the event pairs
        # bracket back-to-back kernel execution only (no launch gaps inside the measured intervals).  The spin is sized from the
        # measured host enqueue time of one eager step on THIS box (slow host cores otherwise leak gaps into the numbers).
        timer.enabled = False
        torch.cuda.synchronize(dev)
        t_h = time.perf_counter()
        step(x_dev, y_dev)
        host_s = time.perf_counter() - t_h
        torch.cuda.synchronize(dev)
        spin_s = min(2.0, 2.0 * host_s + 0.05)
        timer.enabled = True
        for _ in range(3):
            torch.cuda._sleep(int(spin_s * 2.0e9))
            step(x_dev, y_dev)
            torch.cuda.synchronize(dev)
        timer.enabled = False
    if rank != 0:
        return
    peak, peak_src = measured_peaks()
    family = None
    if timer.records:
        gms, gbytes, gflops, n = timer.summary()
        nsteps_t = 3 if use_graph else args.steps
        per_step_ms = gms / nsteps_t
        ach = gbytes / (gms * 1e-3) / 1e9
        family = {"kernel": "pw_gemm_* (all 1x1-conv / linear forward + input-gradient GEMMs), CUDA events around each launch in an eager pass "
                            "(includes ~5 us of event overhead per launch: a lower bound)", "bound": "hbm", "achieved": ach, "peak": peak,
                  "unit": "GB/s", "frac": ach / peak, "launches_per_step": n // nsteps_t, "kernel_ms_per_step": per_step_ms,
                  "share_of_step": per_step_ms / ms_step, "algorithmic_bytes_per_step": gbytes / nsteps_t, "tflops": gflops / (gms * 1e-3) / 1e12}
    # The dominant "kernel" of this path is the step itself: ONE CUDA-graph launch per step.
    # achieved = SURVEY.md 8d's algorithmic bytes per image x the images one launch processes / the launch's CUDA-event duration (the timed
    # region above).
    algo_mb = ALGO_MB_PER_IMAGE.get(args.width)
    roof = None
    if algo_mb:
        algo_bytes = algo_mb * 1e6 * B
        ach = algo_bytes / (ms_step * 1e-3) / 1e9
        roof = {"kernel": ("one CUDA-graph launch = the whole training step" if use_graph else "the whole training step (eager launches)"),
                "bound": "hbm", "achieved": ach, "peak": peak, "unit": "GB/s", "frac": ach / peak, "peak_source": peak_src,
                "algorithmic_bytes_per_launch": algo_bytes, "kernels_per_launch": launches // max(args.steps, 1)}
    cpu = None
    if not args.no_cpu_baseline and world == 1:
        r = cpu_training_throughput(args.width, 3, 1, budget_s=min(60.0, args.cpu_budget))
        cpu = {"value": r["ips"], "unit": "images/sec", "cores": r["threads"], "kind": "port",
               "sample": (f"oracle fp32 training step, batch {r['batch']} (of {B}), {r['warmup']} warm-up + {r['steps']} timed steps "
                          f"({r['ms']:.0f} ms each), {r['threads']} torch threads calibrated on this box ({r['cores_available']} usable cores)"),
               "thread_calibration_img_s": r["calibration"]}
    eager = None
    if not args.no_eager_baseline and world == 1:
        try:
            eager = gpu_eager_baseline(dev, B, args.width, args.steps, args.warmup)
            eager["ours_over_eager"] = value / eager["value"]
            if "graphed_value" in eager:
                eager["ours_over_graphed"] = value / eager["graphed_value"]
        except Exception as e:
            eager = {"error": repr(e)[:300]}
    step_frac = (value / world) * algo_mb * 1e6 / 1e9 / peak if algo_mb else None
    line = {
        "metric": METRIC, "value": value, "unit": "images/sec", "n_gpus": world, "steps": args.steps, "warmup": args.warmup,
        "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": workload_config(args.width, B, world),
        "impl_detail": {"grad_sync": ("none" if world == 1 else f"{args.buckets} flat fp32 NCCL all-reduce buckets issued as the backward of their modules finishes (overlapped), inside the CUDA graph"),
                        "optimizer": ("engine.TrainStep: cvb_ce loss, gradients written into one flat buffer, cvb_grad_norm + cvb_adamw_step (unscale, clip 10, AdamW, scaler update"
                                      + (", EMA 0.0005)" if args.ema else ")") if ts is not None else "torch: F.cross_entropy + GradScaler + clip_grad_norm_ 10 + AdamW(fused)"),
                        "execution": "one CUDA graph per step" if use_graph else "eager launches"},
        "step_ms": step_stats, "gpu_eager_baseline": eager,
        "clocks": clocks, "e2e": {"value": e2e_value, "unit": "images/sec", "h2d_bytes_per_step": h2d, "d2h_bytes_per_step": d2h,
                                  "ms_per_step": e2e_ms},
        "gpu_launches": launches, "roofline": roof, "roofline_gemm_family": family, "cpu_baseline": cpu,
        "step_roofline": {"algorithmic_mb_per_image": algo_mb, "frac_of_hbm_peak": step_frac, "peak_gbs": peak},
        "loss": final_loss,
    }
    if op_ms is not None:
        line["op_ms"] = op_ms
        if timer.records:
            line["gemm_shapes"] = timer.per_shape(3 if use_graph else args.steps)
    if outputs is not None:
        write_outputs(args.dump_outputs, outputs)
    emit(line)


# ------------------------------------------------------------------------------------- secondary workload: ViT-B/16 (BASELINE configs[2])
VIT_GFLOP_PER_IMAGE = {"base": 106.2, "small": 27.6, "tiny": 7.5}  # SURVEY.md 8d: 3 x 2 x forward GMAC (fwd + bwd)
CLIP_GFLOP_PER_PAIR = {"base": 123.8}  # image tower 17.708 GMAC + text tower (12 x 77 tokens x 3.15 M MAC + attention) 2.92 GMAC, x 6


def vit_eager_baseline(dev, B, mode, steps, warmup):
    """The reference's ViT path on this GPU: oracle restatement under torch bf16 autocast + GradScaler + clip + AdamW(fused), eager."""
    from oracle import cvnets_oracle as O
    P = O.clone_params(O.seeded_fill_(O.vit_shapes(mode), 0), device=dev)
    decay = [v for v in P.values() if v.requires_grad and v.dim() > 1]
    no_decay = [v for v in P.values() if v.requires_grad and v.dim() <= 1]
    opt = torch.optim.AdamW([{"params": decay, "weight_decay": 0.2}, {"params": no_decay, "weight_decay": 0.0}], lr=2e-3, fused=True)
    scaler = torch.amp.GradScaler("cuda", enabled=True)
    gen = torch.Generator(device=dev).manual_seed(99)
    x = torch.randn(B, 3, 224, 224, device=dev, generator=gen)
    y = torch.randint(0, NCLS, (B,), device=dev, generator=gen)

    def step():
        with torch.autocast("cuda", dtype=torch.bfloat16):
            loss = F.cross_entropy(O.vit_forward(P, x, mode=mode, training=True), y, label_smoothing=0.1)
        opt.zero_grad(set_to_none=True)
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(decay + no_decay, 1.0)
        scaler.step(opt)
        scaler.update()

    for _ in range(max(3, warmup)):
        step()
    torch.cuda.synchronize(dev)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        step()
    e1.record()
    torch.cuda.synchronize(dev)
    ms = e0.elapsed_time(e1) / steps
    del P
    torch.cuda.empty_cache()
    return {"what": "oracle restatement of the reference ViT, torch eager bf16 autocast + GradScaler + clip 1.0 + AdamW(fused)", "per_gpu_batch": B,
            "value": B / (ms * 1e-3), "unit": "images/sec", "ms_per_step": ms, "steps": steps}


def run_vit(args, rank, world, local_rank):
    """`--workload vit_<mode>`: ViT-B/16 training step (fwd + CE + bwd + clip + AdamW), bf16, 224x224, per-GPU batch 256 by default
    (examples/vit/classification/vit_base.yaml:13-14).  Tensor-bound: the roofline is dense-bf16 TFLOP/s."""
    import ml_cvnets_b200 as m
    from ml_cvnets_b200 import ops
    clip = args.workload.startswith("clip_")
    mode = args.workload.split("_", 1)[1].replace("b16", "base")
    dev = torch.device("cuda", local_rank)
    torch.cuda.set_device(dev)
    torch.manual_seed(rank)
    B = args.batch if args.batch != 128 else 256
    gen = torch.Generator(device=dev).manual_seed(1234 + rank)
    x_dev = torch.randn(B, 3, 224, 224, device=dev, generator=gen)
    if clip:
        # BASELINE.json configs[4]: CLIP ViT-B/16 image + text contrastive step (config/multi_modal_img_text/clip_vit.yaml); synthetic pairs,
        # tokens uniform in the vocabulary with the end-of-text id (the highest) at a random position
        model = m.CLIP(m.default_clip_opts(mode)).to(dev).train()
        y_dev = torch.randint(1, 49406, (B, 77), device=dev, generator=gen)
        y_dev[torch.arange(B, device=dev), torch.randint(1, 77, (B,), device=dev, generator=gen)] = 49407
        ts = m.TrainStep(model, lr=5e-4, weight_decay=0.2, max_norm=1.0, n_buckets=args.buckets,
                         forward_loss=lambda mod, im, tok, cfg: m.clip_contrastive_loss(*mod(im, tok), _cfg=cfg))
    else:
        model = m.VisionTransformer(m.default_vit_opts(mode)).to(dev).train()
        ts = m.TrainStep(model, lr=2e-3, weight_decay=0.2, max_norm=1.0, label_smoothing=0.1, ema_momentum=(0.0005 if args.ema else None), n_buckets=args.buckets)
        y_dev = torch.randint(0, NCLS, (B,), device=dev, generator=gen)

    def sync_all():
        torch.cuda.synchronize(dev)
        if world > 1:
            torch.distributed.barrier()
            torch.cuda.synchronize(dev)

    def max_over_ranks(ms):
        if world == 1:
            return ms
        t = torch.tensor([ms], device=dev, dtype=torch.float64)
        torch.distributed.all_reduce(t, op=torch.distributed.ReduceOp.MAX)
        return float(t.item())

    for _ in range(max(args.warmup, 3)):
        ts.step(x_dev, y_dev)
    if not args.no_graph:
        ts.capture(x_dev, y_dev)
        x_dev, y_dev = ts.static_inputs
        for _ in range(5):
            ts.step(x_dev, y_dev)
    sampler = ClockSampler(local_rank)
    if rank == 0:
        sampler.start()  # before the barrier (see run_ours)
    sync_all()
    n0 = ops.launch_count
    marks = [torch.cuda.Event(enable_timing=True) for _ in range(args.steps + 1)]
    marks[0].record()
    for i in range(args.steps):
        loss = ts.step(x_dev, y_dev)
        marks[i + 1].record()
    sync_all()
    outputs = output_snapshot(loss, model) if args.dump_outputs else None
    clocks = sampler.stop() if rank == 0 else None
    ms_step = max_over_ranks(marks[0].elapsed_time(marks[-1])) / args.steps
    per = sorted(marks[i].elapsed_time(marks[i + 1]) for i in range(args.steps))
    value = world * B / (ms_step * 1e-3)
    launches = (ts.launches_per_step * args.steps) if not args.no_graph else (ops.launch_count - n0)
    # end to end: pinned host -> device every step, loss read back every step
    hx, hy = torch.randn(B, 3, 224, 224).pin_memory(), y_dev.cpu().pin_memory()
    dx, dy = torch.empty_like(x_dev), torch.empty_like(y_dev)
    hloss = torch.zeros(1).pin_memory()
    sync_all()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(args.steps):
        dx.copy_(hx, non_blocking=True)
        dy.copy_(hy, non_blocking=True)
        loss = ts.step(dx, dy)
        hloss.copy_(loss.detach().reshape(1), non_blocking=True)
        torch.cuda.current_stream().synchronize()
        _ = float(hloss[0])
    e1.record()
    sync_all()
    e2e_ms = max_over_ranks(e0.elapsed_time(e1)) / args.steps
    if rank != 0:
        return
    peaks = {}
    try:
        with open(os.path.join(ROOT, "MEASURED_PEAKS.json")) as f:
            peaks = json.load(f)
    except Exception:
        pass
    peak_tf = float(peaks.get("bf16_tflops_sustained", 989.0))  # fallback: H100 SXM data sheet, dense bf16
    gflop = (CLIP_GFLOP_PER_PAIR if clip else VIT_GFLOP_PER_IMAGE).get(mode)
    ach = (value / world) * gflop / 1e3 if gflop else None
    eager = None
    if not args.no_eager_baseline and world == 1 and not clip:
        try:
            eager = vit_eager_baseline(dev, B, mode, max(3, args.steps // 2), 3)
            eager["ours_over_eager"] = value / eager["value"]
        except Exception as e:
            eager = {"error": repr(e)[:300]}
    if outputs is not None:
        write_outputs(args.dump_outputs, outputs)
    emit({
        "metric": (f"image-text pairs/sec contrastive training step, CLIP ViT-{mode}/16 bf16 224x224" if clip else
                   f"images/sec training step, ViT-{mode}/16 bf16 224x224"), "value": value, "unit": "images/sec", "n_gpus": world, "steps": args.steps,
        "warmup": args.warmup, "ms_per_step": ms_step, "higher_is_better": True, "scaling": "weak", "vs_baseline": None, "dtype": "bf16", "data": "synthetic",
        "config": {"workload": (f"CLIP ViT-{mode}/16 image + 12-layer text tower, contrastive loss with feature all-gather, fwd + bwd + clip + AdamW, "
                                "synthetic pairs (BASELINE.json configs[4])" if clip else
                                f"ViT-{mode}/16 bf16 forward + loss + backward + clip + AdamW, synthetic 224x224 (BASELINE.json configs[2])"), "per_gpu_batch": B,
                   "global_batch": B * world, "parallelism": f"dp{world}", "resolution": 224, "l2": "activations per step (> 10 GB) exceed the 50 MB L2"},
        "step_ms": {"min": per[0], "median": per[len(per) // 2], "max": per[-1]}, "clocks": clocks,
        "e2e": {"value": world * B / (e2e_ms * 1e-3), "unit": "images/sec", "h2d_bytes_per_step": world * (hx.numel() * 4 + hy.numel() * 8), "d2h_bytes_per_step": world * 4,
                "ms_per_step": e2e_ms},
        "gpu_launches": launches,
        "roofline": {"kernel": "whole step (one CUDA-graph launch): tensor-bound GEMMs + attention", "bound": "tensor", "achieved": ach, "peak": peak_tf,
                     "unit": "TFLOP/s", "frac": (ach / peak_tf) if ach else None, "peak_source": ("MEASURED_PEAKS.json bf16_tflops_sustained" if "bf16_tflops_sustained" in peaks else "H100 SXM data sheet"), "traffic": None,
                     "algorithmic_gflop_per_image": gflop},
        "gpu_eager_baseline": eager, "loss": float(loss.detach()),
    })


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--gpus", type=int, default=1)
    ap.add_argument("--steps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--batch", type=int, default=128, help="per-GPU batch (recipe: 128)")
    ap.add_argument("--workload", default="mobilevit_v2", help="mobilevit_v2 (the metric) | vit_b16 | vit_small (BASELINE.json configs[2] family) | clip_b16 (configs[4])")
    ap.add_argument("--width", type=float, default=1.0, help="MobileViTv2 width multiplier (1.0 = the metric config, 2.0 = BASELINE.json configs[3])")
    ap.add_argument("--cpu-budget", type=float, default=120.0, help="wall-clock bound (s) of the CPU arm / cpu_baseline sample")
    ap.add_argument("--no-eager-baseline", action="store_true", help="skip the eager-PyTorch-on-GPU comparator")
    ap.add_argument("--impl", default="ours", choices=["ours", "reference"])
    ap.add_argument("--no-cpu-baseline", action="store_true")
    ap.add_argument("--no-kernel-timing", action="store_true")
    ap.add_argument("--profile-ops", action="store_true", help="CUDA-event time per C-ABI entry point (diagnostics)")
    ap.add_argument("--torch-optim", action="store_true", help="A/B: torch loss/GradScaler/clip/AdamW instead of engine.TrainStep (1 GPU)")
    ap.add_argument("--ema", action="store_true", help="EMA of the weights (momentum 0.0005, the recipe's ema.enable) fused into the optimizer tail")
    ap.add_argument("--buckets", type=int, default=3, help="gradient all-reduce buckets (N > 1)")
    ap.add_argument("--no-pdl", action="store_true", help="diagnostics: plain stream-ordered launches instead of programmatic dependent launch")
    ap.add_argument("--no-graph", action="store_true", help="run the step eagerly instead of replaying one captured CUDA graph (N=1)")
    ap.add_argument("--dump-outputs", metavar="DIR", default=None,
                    help="write the loss and the updated parameters of the last timed step as float32 DIR/<name>.npy (rank 0)")
    args = ap.parse_args()
    rank, world, local_rank = int(os.environ.get("RANK", 0)), int(os.environ.get("WORLD_SIZE", 1)), int(os.environ.get("LOCAL_RANK", 0))
    quiet_stdout()
    if args.impl == "reference":
        run_reference_arm(args, rank, world)
        return
    if world > 1:
        os.environ.setdefault("MASTER_ADDR", "127.0.0.1")
        torch.distributed.init_process_group("nccl", device_id=torch.device("cuda", local_rank))
    try:
        if args.workload.startswith("vit_") or args.workload.startswith("clip_"):
            run_vit(args, rank, world, local_rank)
        else:
            run_ours(args, rank, world, local_rank)
    finally:
        if world > 1:
            torch.distributed.destroy_process_group()


if __name__ == "__main__":
    main()

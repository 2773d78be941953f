"""Gradient accumulation in TrainStep (-m gpu): ``accum_freq`` micro-batches per optimizer update, eager and captured.

  * cvb_grad_accumulate against torch's fp32 add, bit for bit, at ragged sizes and at sizes where every CTA loops three times;
  * the accumulated gradient is the in-order fp32 sum of the micro-batch gradients taken separately (MobileViTv2-1.0, EfficientNet-b0);
  * weights, momentum, step count, loss scale and EMA move once per window, and an EMA model evaluated inside a window does not change;
  * EfficientNet-b0 against the reference's accumulating loop (tests/golden/accum_fp32.pt);
  * an inf in one micro-batch skips the window's update and backs the loss scale off once; ``zero_grad()`` discards an open window;
  * captured replays equal eager calls bit for bit over a shuffled multi-shape sequence (RangeAugment, mixup, buffer EMA), with one update
    graph beside the per-shape graphs; accum_freq 1 is the plain step; data parallel on two GPUs."""
import copy
import os
import random
import socket

import pytest
import torch

import accum_ref as A
import efficientnet_ref as E
from oracle import cvnets_oracle as O

pytestmark = pytest.mark.gpu

AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True}


@pytest.fixture(scope="module")
def m():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as pkg
    return pkg


def rel_l2(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm().clamp_min(1e-30))


def _batch(shape, n_classes, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g), torch.randint(0, n_classes, (shape[0],), device="cuda", generator=g)


def _effnet(m, n_classes=16, **extra):
    torch.manual_seed(0)
    return m.EfficientNet(m.default_effnet_opts("b0", n_classes=n_classes, **extra)).cuda().train()


def _sgd(m, model, **kw):
    args = dict(optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None, label_smoothing=0.1, ema_momentum=0.0005)
    args.update(kw)
    return m.TrainStep(model, **args)


# ------------------------------------------------------------------------------------------------------------------ kernel
def _sizes():
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    per_pass = 4 * sms * 256 * 4  # the grid cap (4 CTAs per SM) x 256 threads x one float4 each
    return [1, 3, 4, 5, 1023, 4097, 3 * per_pass + 3, 3 * per_pass + 4 * 256 + 1]


@pytest.mark.parametrize("i", range(8))
def test_grad_accumulate_kernel_is_torch_add(m, i):
    from ml_cvnets_b200 import ops
    n = _sizes()[i]
    g = torch.Generator(device="cuda").manual_seed(100 + i)
    acc = torch.randn(n, device="cuda", generator=g)
    src = torch.randn(n, device="cuda", generator=g) * torch.exp2(torch.randint(-20, 20, (n,), device="cuda", generator=g).float())
    if n >= 4:  # subnormal operands and sums, signed zeros: an add that flushed them to zero would differ
        acc[:4] = torch.tensor([1e-39, -3e-40, 0.0, -0.0], device="cuda")
        src[:4] = torch.tensor([2e-39, 1e-40, -0.0, -0.0], device="cuda")
    want = torch.add(acc, src)
    ops.grad_accumulate(acc, src)
    torch.cuda.synchronize()
    assert torch.equal(acc.view(torch.int32), want.view(torch.int32))


def test_grad_accumulate_rejects_misaligned_or_mismatched(m):
    from ml_cvnets_b200 import _lib as L
    from ml_cvnets_b200 import ops
    a, b = torch.zeros(64, device="cuda"), torch.ones(64, device="cuda")
    with pytest.raises(L.CvbError, match="cvb_grad_accumulate"):
        ops.grad_accumulate(a[1:], b[1:])
    with pytest.raises(ValueError):
        ops.grad_accumulate(a, b[:32])
    with pytest.raises(ValueError):
        ops.grad_accumulate(a.double(), b.double())


# ------------------------------------------------------------------------------------------------------------------ summed gradients
def _mobilevit(m):
    torch.manual_seed(0)
    return m.MobileViTv2(m.default_opts(width_multiplier=1.0, n_classes=100)).cuda().train()


@pytest.mark.parametrize("k", [2, 3])
@pytest.mark.parametrize("model_name", ["mobilevit_v2", "efficientnet_b0"])
def test_accumulated_gradient_is_the_in_order_sum(m, model_name, k):
    """k micro-batches into one open window (accum_freq k + 1, so no update intervenes and the weights stay frozen) against the gradients of
    the same micro-batches taken one at a time on a twin whose steps cannot move its weights (lr 0), summed in order in fp32."""
    from ml_cvnets_b200 import ops
    make = _mobilevit if model_name == "mobilevit_v2" else _effnet
    res, B = (128, 4) if model_name == "mobilevit_v2" else (96, 6)
    batches = [_batch((B, 3, res, res), 16, 700 + j) for j in range(k)]
    base = make(m)
    twin = copy.deepcopy(base)
    acc_step = _sgd(m, base, accum_freq=k + 1, ema_momentum=None)
    one_step = _sgd(m, twin, lr=0.0, ema_momentum=None)
    ops.rng_seed(3)
    want = torch.zeros_like(one_step.ws.flat_g)
    for x, y in batches:
        one_step.step(x, y)
        want += one_step.ws.flat_g
    ops.rng_seed(3)
    for x, y in batches:
        acc_step.step(x, y)
        assert not acc_step.updated
    torch.cuda.synchronize()
    assert torch.isfinite(want).all() and float(want.abs().max()) > 0
    assert torch.equal(acc_step.grad_acc, want), rel_l2(acc_step.grad_acc, want)
    p = next(iter(acc_step.ws.params))
    o, n = acc_step.ws.offsets[id(p)]
    assert p.grad.data_ptr() == acc_step.grad_acc[o:o + n].data_ptr()  # p.grad are views of the accumulator


# ------------------------------------------------------------------------------------------------------------------ cadence
def _state(ts):
    torch.cuda.synchronize()
    return {"params": ts.opt.flat_p.clone(), "momentum": ts.opt.momentum_buffer.clone(), "step": ts.opt.step_count.clone(),
            "scale": ts.opt.scale.clone(), "ema": ts.opt.ema.clone(), "ema_buffers": ts.ema_buffers.clone()}


def test_state_moves_once_per_window_captured(m):
    """accum_freq 3, captured at one shape: inside a window nothing the update owns moves and the EMA model's evaluation is unchanged; the
    window's third call applies the update once (step count + 1) and clears the accumulator."""
    x, y = _batch((8, 3, 96, 96), 16, 1)
    ts = _sgd(m, _effnet(m), accum_freq=3, ema_momentum=0.3, ema_buffers=True)
    ts.capture(x, y)  # three eager warm-up calls: exactly one window
    assert ts._window == 0 and ts.updated
    ev = m.EvalStep(ts.ema_model())
    xe, ye = _batch((16, 3, 96, 96), 16, 2)

    def ema_logits():
        ev.update(xe, ye)
        torch.cuda.synchronize()
        return ev.logits.clone()

    for w in range(2):
        before, logits_before = _state(ts), ema_logits()
        for call in range(3):
            ts.step(*_batch((8, 3, 96, 96), 16, 10 * w + call))
            now = _state(ts)
            if call < 2:
                assert not ts.updated
                for k, v in before.items():
                    assert torch.equal(now[k], v), (w, call, k)
                assert torch.equal(ema_logits(), logits_before), (w, call)
                assert float(ts.grad_acc.abs().max()) > 0
            else:
                assert ts.updated
                assert float(now["step"][0]) == float(before["step"][0]) + 1
                for k in ("params", "momentum", "ema", "ema_buffers"):
                    assert not torch.equal(now[k], before[k]), (w, k)
                assert not torch.equal(ema_logits(), logits_before)
                assert int(torch.count_nonzero(ts.grad_acc)) == 0


# ------------------------------------------------------------------------------------------------------------------ reference
@pytest.fixture(scope="module")
def fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "accum_fp32.pt"), weights_only=False)


def _errors(fx, P0, losses, micro, windows):
    """rel-L2 against the fixture of the losses and of what each step moved -- running statistics after every micro-batch, parameters,
    momentum and EMA after every window -- each compared as its change from the start (the momentum starts at zero)."""
    def moved(keys, src, want):
        s0 = A.flat_sample([P0[k] for k in keys])
        return rel_l2(A.flat_sample([src[k] for k in keys]) - s0, want - s0)

    errs = {f"loss {j}": abs(a - b) / abs(b) for j, (a, b) in enumerate(zip(losses, fx["losses"]))}
    errs.update({f"running stats {j}": moved(fx["bn_keys"], st, fx["micro"][j]) for j, st in enumerate(micro)})
    for w, ((params, mom, ema), want) in enumerate(zip(windows, fx["windows"])):
        errs[f"params {w}"] = moved(fx["param_keys"], params, want["params"])
        errs[f"momentum {w}"] = rel_l2(A.flat_sample([mom[k] for k in fx["param_keys"]]), want["momentum"])
        errs[f"ema {w}"] = moved(fx["ema_keys"], ema, want["ema"])
    return errs


def test_against_the_reference_loop(m, fx):
    """EfficientNet-b0, accum_freq 2, two windows, against the reference's loop (make_golden_accum.py), bounded as the EfficientNet parity
    tests bound theirs: activations are bf16 at every layer boundary, so each quantity is held to its tolerance (losses 2e-2, the rest 5e-2
    rel-L2) or to 3x the error of the fp32 restatement run under bf16 autocast on the same micro-batches, whichever is larger.  At 64 x 64 and
    8 images the seeded network's early-layer gradients move by about 0.2 under bf16 alone, and the second window compounds the first."""
    c = fx["cfg"]
    P0 = O.seeded_fill_(E.efficientnet_shapes(c["mode"], c["n_classes"]), c["param_seed"])
    xs = [O.seeded_input((c["batch"], 3, c["crop"], c["crop"]), seed).cuda() for seed in c["x_seeds"]]
    ys = [y.cuda() for y in fx["targets"]]
    hp = dict(lr=c["lr"], momentum=c["momentum"], weight_decay=c["weight_decay"], label_smoothing=c["label_smoothing"])
    with torch.autocast("cuda", dtype=torch.bfloat16):
        a_losses, a_micro, a_windows = A.train_windows(O.clone_params(P0, device="cuda"), xs, ys, accum_freq=c["accum_freq"],
                                                       ema_momentum=c["ema_momentum"], mode=c["mode"], **hp)
    auto = _errors(fx, P0, a_losses, a_micro, a_windows)

    model = m.EfficientNet(m.default_effnet_opts(c["mode"], n_classes=c["n_classes"]))
    model.load_state_dict(P0, strict=True)
    model = model.cuda().train()
    ts = m.TrainStep(model, optimizer="sgd", nesterov=True, max_norm=None, ema_momentum=c["ema_momentum"], ema_buffers=True,
                     accum_freq=c["accum_freq"], **hp)
    named = dict(model.named_parameters())
    losses, micro, windows = [], [], []
    for x, y in zip(xs, ys):
        losses.append(float(ts.step(x, y).detach()))
        micro.append({k: v.clone() for k, v in model.state_dict().items()})
        if ts.updated:
            mom = {}
            for k, p in named.items():
                o, n = ts.ws.offsets[id(p)]
                mom[k] = ts.opt.momentum_buffer[o:o + n].view_as(p).clone()
            ema = {k: v.clone() for k, v in ts.ema_model().state_dict().items()}  # views of the live EMA: snapshot them
            windows.append(({k: p.detach().clone() for k, p in named.items()}, mom, ema))
    assert len(windows) == len(fx["windows"]) == 2
    errs = _errors(fx, P0, losses, micro, windows)
    print({k: f"{v:.3g} (autocast {auto[k]:.3g})" for k, v in errs.items()})
    for k, v in errs.items():
        assert v <= max(2e-2 if k.startswith("loss") else 5e-2, 3.0 * auto[k]), (k, v, auto[k])


# ------------------------------------------------------------------------------------------------------------------ inf, zero_grad
def test_inf_in_one_micro_batch_skips_the_window(m):
    """Window 1 is clean; window 2's second micro-batch holds an inf pixel.  Its update is skipped (parameters, momentum and step count stay),
    the loss scale is halved once and the growth tracker reset, and the EMA takes its skipped-step update as the reference's does."""
    ts = _sgd(m, _effnet(m), accum_freq=2, ema_momentum=0.1)
    ts.step(*_batch((4, 3, 64, 64), 16, 20))
    ts.step(*_batch((4, 3, 64, 64), 16, 21))
    assert ts.updated
    before = _state_no_buffers(ts)
    ts.step(*_batch((4, 3, 64, 64), 16, 22))
    x, y = _batch((4, 3, 64, 64), 16, 23)
    x[1, 0, 5, 7] = float("inf")
    ts.step(x, y)
    assert ts.updated
    now = _state_no_buffers(ts)
    assert torch.equal(now["params"], before["params"]) and torch.equal(now["momentum"], before["momentum"])
    assert float(now["step"][0]) == float(before["step"][0]) == 1.0
    assert float(now["scale"][0]) == 0.5 * float(before["scale"][0]) and float(now["scale"][1]) == 0.0
    assert float(ts.opt.stats[1]) > 0  # the window's count of non-finite gradient elements
    assert torch.allclose(now["ema"], before["ema"] * 0.9 + 0.1 * before["params"], rtol=1e-6, atol=1e-7)
    assert int(torch.count_nonzero(ts.grad_acc)) == 0


def _state_no_buffers(ts):
    torch.cuda.synchronize()
    return {"params": ts.opt.flat_p.clone(), "momentum": ts.opt.momentum_buffer.clone(), "step": ts.opt.step_count.clone(),
            "scale": ts.opt.scale.clone(), "ema": ts.opt.ema.clone()}


def test_zero_grad_discards_an_open_window(m):
    """One micro-batch, zero_grad(), then a full window equals that window alone, bit for bit (the BatchNorm statistics saw the discarded
    micro-batch, as the reference's do; in training mode they do not enter the gradients)."""
    batches = [_batch((6, 3, 64, 64), 16, 30 + j) for j in range(3)]
    runs = []
    for discard in (True, False):
        ts = _sgd(m, _effnet(m), accum_freq=2)
        if discard:
            ts.step(*batches[0])
            assert not ts.updated and float(ts.grad_acc.abs().max()) > 0
            ts.zero_grad()
            assert ts._window == 0 and int(torch.count_nonzero(ts.grad_acc)) == 0
        ts.step(*batches[1])
        assert not ts.updated
        ts.step(*batches[2])
        assert ts.updated
        runs.append(_state_no_buffers(ts))
        del ts
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), k


# ------------------------------------------------------------------------------------------------------------------ capture
SHAPES = ((64, 12), (96, 6), (128, 4))


def _aug_step(m, accum_freq):
    model = _effnet(m, **AUG)
    na = m.NeuralAugmentationLoss(target_value=(40, 5), curriculum_method="cosine", period=20)
    return _sgd(m, model, aug_loss=na, ema_buffers=True, accum_freq=accum_freq), model


def test_captured_windows_equal_eager_calls_bitwise(m):
    """EfficientNet-b0 + RangeAugment, mixup drawn per call, buffer EMA, accum_freq 2 over three shapes: capture (9 eager warm-up calls, so
    the window is open when capture ends) and a shuffled sequence of 11 calls whose windows mix shapes, against a TrainStep making the same
    calls eagerly.  Losses, loss parts, parameters, momentum, EMAs and running statistics agree bit for bit; the graphs are one per shape plus
    one update graph, in a pool at most 1.05x that of the same capture without accumulation."""
    from ml_cvnets_b200 import ops
    examples = [_batch((B, 3, c, c), 16, 800 + c) for c, B in SHAPES]
    rnd = random.Random(4)
    order = [rnd.randrange(len(SHAPES)) for _ in range(11)]
    seq = [_batch((SHAPES[i][1], 3, SHAPES[i][0], SHAPES[i][0]), 16, 8000 + k) for k, i in enumerate(order)]
    torch.manual_seed(5)
    sampler = m.engine.MixingSampler(cutmix_alpha=None)
    mixes = [sampler.sample(SHAPES[i][0], SHAPES[i][0]) for i in order]
    runs, updates = [], []
    for captured in (True, False):
        ts, model = _aug_step(m, 2)
        ops.rng_seed(9)
        if captured:
            ts.capture_shapes(examples)
            assert len(ts.captured_shapes) == len(SHAPES) and ts._update_graph is not None and ts.launches_per_update >= 3
            pool = ts.graph_pool_bytes()
        else:
            for _ in range(3):
                for x, y in examples:
                    ts.step(x, y)
        assert ts._window == 1
        losses, parts, upd = [], [], []
        for k, ((x, y), (kind, lam, box)) in enumerate(zip(seq, mixes)):
            ts.set_mix(kind, lam, box)
            ts.set_epoch(k // 2)
            losses.append(ts.step(x, y).clone())
            parts.append(ts.loss_parts.clone())
            upd.append(ts.updated)
        torch.cuda.synchronize()
        updates.append(upd)
        runs.append({"losses": torch.stack(losses), "parts": torch.stack(parts), "params": ts.opt.flat_p.clone(),
                     "momentum": ts.opt.momentum_buffer.clone(), "ema": ts.opt.ema.clone(), "ema_buffers": ts.ema_buffers.clone(),
                     "buffers": ts.ws.flat_buffers().clone(), "acc": ts.grad_acc.clone()})
        del ts, model
    print("order", order, "updates", updates[0], "losses", runs[0]["losses"].tolist())
    assert updates[0] == updates[1] == [k % 2 == 0 for k in range(len(seq))]
    assert torch.isfinite(runs[0]["losses"]).all()
    for k in runs[0]:
        assert torch.equal(runs[0][k], runs[1][k]), (k, rel_l2(runs[0][k], runs[1][k]))
    ts1, _ = _aug_step(m, 1)
    ts1.capture_shapes(examples)
    pool1 = ts1.graph_pool_bytes()
    del ts1
    print(f"graph pool: accum_freq 2 {pool} B, accum_freq 1 {pool1} B ({pool / pool1:.4f}x)")
    assert pool <= 1.05 * pool1


def test_accum_freq_one_is_the_plain_step(m):
    from ml_cvnets_b200 import ops
    x, y = _batch((8, 3, 96, 96), 16, 40)
    runs = []
    for kw in ({}, {"accum_freq": 1}):
        ts = _sgd(m, _effnet(m), **kw)
        assert ts.grad_acc is None and ts.opt.flat_g is ts.ws.flat_g
        assert ts.ws.params[0].grad.data_ptr() == ts.ws.flat_g.data_ptr()
        ops.rng_seed(1)
        ts.capture(x, y)
        assert ts._update_graph is None and ts.launches_per_update is None
        losses = [ts.step(x, y).clone() for _ in range(3)]
        assert ts.updated
        torch.cuda.synchronize()
        runs.append((ts.launches_per_shape, torch.stack(losses), ts.opt.flat_p.clone(), ts.opt.ema.clone()))
        del ts
    assert runs[0][0] == runs[1][0]
    for a, b in zip(runs[0][1:], runs[1][1:]):
        assert torch.equal(a, b)


# ------------------------------------------------------------------------------------------------------------------ data parallel
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _ddp_worker(rank, world, port, q):
    import torch.distributed as dist
    import ml_cvnets_b200 as m
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        P = O.seeded_fill_(O.mobilevit_v2_shapes(0.5), 7)
        shards = [[_batch((4, 3, 128, 128), 1000, 900 + 10 * r + j) for r in range(world)] for j in range(3)]

        def fresh():
            model = m.MobileViTv2(m.default_opts(width_multiplier=0.5))
            model.load_state_dict(P, strict=True)
            return model.cuda().eval()  # running statistics: the exchange itself is checked tightly

        ref = None
        for j in range(2):  # the single-process gradient of the concatenated micro-batches, summed over the two micro-batches
            for x, y in shards[j]:
                one = m.TrainStep(fresh(), lr=0.0, weight_decay=0.0, data_parallel=False)
                one.step(x, y)
                ref = one.ws.flat_g.clone() if ref is None else ref + one.ws.flat_g
        ref = ref / world
        ts = m.TrainStep(fresh(), lr=0.0, weight_decay=0.0, n_buckets=3, accum_freq=3)
        ts.capture(*shards[0][rank])
        ts.zero_grad()
        for j in range(2):
            ts.step(*shards[j][rank])
        err = float((ts.grad_acc / world - ref).norm() / ref.norm())
        ts.step(*shards[2][rank])
        assert ts.updated
        ts.set_lr(1e-3)
        for k in range(6):
            ts.step(*shards[k % 3][rank])
        flat = ts.opt.flat_p.clone()
        gathered = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(gathered, flat)
        drift = max(float((g - gathered[0]).abs().max()) for g in gathered)
        torch.cuda.synchronize()
        q.put((rank, err, drift))
    except BaseException as e:  # the parent must never wait for a result that will not come
        q.put((rank, repr(e)[:500], -1.0))
    q.close()
    q.join_thread()
    # a captured CUDA graph that contains NCCL kernels is still alive here: leave without the collective shutdown
    os._exit(0)


def test_data_parallel_accumulation():
    """Two ranks, accum_freq 3, captured: the all-reduced accumulator after two micro-batches against the single-process gradient of the
    concatenated micro-batches (5e-3 rel-L2, as the data-parallel exchange is bounded elsewhere); after two more windows the ranks' parameters
    are bit-identical."""
    if not torch.cuda.is_available() or torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 CUDA devices")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    world, port = 2, _free_port()
    procs = [ctx.Process(target=_ddp_worker, args=(r, world, port, q)) for r in range(world)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in range(world)]
    for p in procs:
        p.join(timeout=30)
        if p.is_alive():
            p.terminate()
    for rank, err, drift in res:
        assert not isinstance(err, str), f"rank {rank} failed: {err}"
        print(f"rank {rank}: accumulated gradient rel-L2 vs the single-process sum {err:.3g}; drift {drift:.3g}")
        assert err <= 5e-3
        assert drift == 0.0

"""Classification validation on the GPU (-m gpu): cvb_cls_metrics against an fp64 restatement (tests/eval_ref.py, pinned to the reference on
the CPU by test_eval_cpu.py) with negative controls; cvb_ema_update as TrainStep(ema_buffers=True) runs it, eager and captured; the EMA twin
of TrainStep.ema_model(); and EvalStep: weight refresh under interleaved captured train / eval graphs, padding invariance of the ragged
batch, captured against eager on the recipes' models, and data parallel."""
import os
import socket

import pytest
import torch

import eval_ref as E

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def m():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as pkg
    return pkg


def _bits(t):
    return t.detach().contiguous().view(torch.int32 if t.element_size() == 4 else torch.int16 if t.element_size() == 2 else torch.int64)


def _equal(a, b):
    return a.shape == b.shape and torch.equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------------------- cvb_cls_metrics
def _logits(B, C, seed, ties=False):
    """bf16 [B, C] view (row stride a multiple of 8 past C, like the classifier's padded output) and int64 targets with every 5th row
    ignored.  ties=False: the target's logit is unique in its row (torch.topk's choice among tied classes cannot matter); ties=True:
    logits from {0, .., 4}, so targets tie at the k-th place."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    ld = (C + 7) // 8 * 8 + 8
    full = torch.randn(B, ld, device="cuda", generator=g).mul_(3.0)
    if ties:
        full = torch.randint(0, 5, (B, ld), device="cuda", generator=g).float()
    full = full.to(torch.bfloat16)
    L = full[:, :C]
    y = torch.randint(0, C, (B,), device="cuda", generator=g)
    if not ties:
        lt = L.gather(1, y[:, None]).float()
        dup = (L.float() == lt) & (torch.arange(C, device="cuda")[None, :] != y[:, None])
        L[dup] = (lt - lt.abs() * 0.05 - 0.05).expand(-1, C)[dup].to(torch.bfloat16)
    if B > 1:
        y[::5] = -1
    return L, y


def _run_metrics(ops, L, y, ignore_index=-1):
    acc = torch.zeros(1, device="cuda", dtype=torch.float64)
    cnt = torch.zeros(3, device="cuda", dtype=torch.int64)
    scratch = torch.zeros(max(y.shape[0], 1), device="cuda")
    ticket = torch.zeros(1, device="cuda", dtype=torch.int32)
    ops.cls_metrics(L, y, acc, cnt, scratch, ticket, ignore_index)
    torch.cuda.synchronize()
    return acc, cnt


def _matches(acc, cnt, want, rel=1e-6):
    t1, t5, n = cnt.tolist()
    return (t1, t5, n) == (want["top1"], want["top5"], want["n"]) and abs(float(acc) - want["loss_sum"]) <= rel * max(abs(want["loss_sum"]), 1e-30)


@pytest.mark.parametrize("C", [3, 8, 1000, 10450])
@pytest.mark.parametrize("B", [1, 7, 100, 4096])
def test_cls_metrics_against_fp64(m, B, C):
    from ml_cvnets_b200 import ops
    L, y = _logits(B, C, 1000 * B + C)
    want = E.cls_metrics(L, y)
    acc, cnt = _run_metrics(ops, L, y)
    assert _matches(acc, cnt, want), (acc.item(), cnt.tolist(), want)
    # tie-free targets: exact against torch.topk (the reference's top_k_accuracy)
    keep = y != -1
    k = min(5, C)
    top = L[keep].float().topk(k, 1).indices
    hit = top == y[keep][:, None]
    assert cnt.tolist()[:2] == [int(hit[:, :1].sum()), int(hit.sum()) if C >= 5 else int(keep.sum())]
    # two runs agree bit for bit (4096 rows: each warp of the 256 CTAs takes two rows, and the last CTA folds all of them)
    acc2, cnt2 = _run_metrics(ops, L, y)
    assert _equal(acc, acc2) and torch.equal(cnt, cnt2)


@pytest.mark.parametrize("C", [3, 10, 1000])
def test_cls_metrics_ties_follow_the_rank_rule(m, C):
    from ml_cvnets_b200 import ops
    L, y = _logits(512, C, 7 + C, ties=True)
    want = E.cls_metrics(L, y)
    acc, cnt = _run_metrics(ops, L, y)
    assert _matches(acc, cnt, want)
    if C >= 5:  # the rule counts ties for the target: strictly more hits than "the target must beat every tied class"
        strict = int(((L > L.gather(1, y.clamp(min=0)[:, None])) | ((L == L.gather(1, y.clamp(min=0)[:, None]))
                                                                  & (torch.arange(C, device="cuda") != y[:, None]))).sum(1)[y != -1].lt(1).sum())
        assert cnt.tolist()[0] > strict


def test_cls_metrics_negative_controls(m):
    """A target shifted by one class, a dropped last row and a counted pad row must each fail the check the real call passes."""
    from ml_cvnets_b200 import ops
    L, y = _logits(100, 1000, 5)
    y[-1] = 3
    want = E.cls_metrics(L, y)
    assert _matches(*_run_metrics(ops, L, y), want)
    shifted = torch.where(y >= 0, (y + 1) % 1000, y)
    assert not _matches(*_run_metrics(ops, L, shifted), want)
    assert not _matches(*_run_metrics(ops, L[:-1], y[:-1]), want)
    assert int(y[0]) == -1  # row 0 is a pad row: counting it must fail the check
    padded = y.clone()
    padded[0] = 0
    assert not _matches(*_run_metrics(ops, L, padded), want)


def test_cls_metrics_wrapper_and_accumulation(m):
    """Calls add into the accumulators; a label outside [0, C) gives a NaN loss."""
    from ml_cvnets_b200 import ops
    L, y = _logits(64, 100, 11)
    acc = torch.zeros(1, device="cuda", dtype=torch.float64)
    cnt = torch.zeros(3, device="cuda", dtype=torch.int64)
    scratch, ticket = torch.zeros(64, device="cuda"), torch.zeros(1, device="cuda", dtype=torch.int32)
    for _ in range(3):
        ops.cls_metrics(L, y, acc, cnt, scratch, ticket)
    want = E.cls_metrics(L, y)
    assert cnt.tolist() == [3 * want["top1"], 3 * want["top5"], 3 * want["n"]]
    assert float(acc) == pytest.approx(3 * want["loss_sum"], rel=1e-6) and int(ticket) == 0
    bad = y.clone()
    bad[1] = 100
    a2, _ = _run_metrics(ops, L, bad)
    assert torch.isnan(a2).all()


# ------------------------------------------------------------------------------------------------------------- buffer EMA
def _mv2(m, width=0.5):
    torch.manual_seed(0)
    return m.MobileViTv2(m.default_opts(width, n_classes=10)).cuda().train()


def _b0(m, **kw):
    torch.manual_seed(0)
    return m.EfficientNet(m.default_effnet_opts("b0", n_classes=10, **kw)).cuda().train()


def _sgd(m, model, **kw):
    return m.TrainStep(model, optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None, label_smoothing=0.1, **kw)


def _data(B, res, seed, n_classes=10):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B, 3, res, res, device="cuda", generator=g), torch.randint(0, n_classes, (B,), device="cuda", generator=g)


@pytest.mark.parametrize("captured", [False, True])
@pytest.mark.parametrize("kind", ["mobilevit_v2", "efficientnet"])
def test_buffer_ema_follows_the_oracle_bitwise(m, kind, captured):
    model = _mv2(m) if kind == "mobilevit_v2" else _b0(m)
    step = _sgd(m, model, ema_momentum=0.1, ema_buffers=True)
    flat = step.ws.flat_buffers()
    assert _equal(step.ema_buffers, flat)
    bufs = [b for b in model.buffers() if b.is_floating_point()]
    assert all(b.data_ptr() >= flat.data_ptr() and b.data_ptr() < flat.data_ptr() + flat.numel() * 4 for b in bufs)
    batches = [_data(8, 128, 40 + i) for i in range(5)]
    if captured:
        step.capture(*batches[0])
    ref = step.ema_buffers.clone()
    for x, y in batches:
        step(x, y)
        torch.cuda.synchronize()
        ref = E.ema_flat(ref, flat.clone(), 0.1)
        assert _equal(step.ema_buffers, ref)
    sd = step.state_dict()
    assert _equal(sd["ema_buffers"], ref)


def test_ema_buffers_off_is_the_current_step_bitwise(m):
    """EfficientNet-b0 (a bitwise deterministic step): with ema_buffers=False the step is the parent's -- same losses, parameters and
    parameter EMA as with the buffer EMA on -- and its captured graph has exactly one launch fewer (the buffer EMA's)."""
    runs = {}
    for on in (False, True):
        model = _b0(m)
        step = _sgd(m, model, ema_momentum=0.1, ema_buffers=on)
        batches = [_data(8, 96, 60 + i) for i in range(4)]
        step.capture(*batches[0])
        losses = [step(x, y).clone() for x, y in batches]
        torch.cuda.synchronize()
        runs[on] = (torch.stack(losses), step.opt.flat_p.clone(), step.opt.ema.clone(), step.launches_per_step, set(step.state_dict()))
    (l0, p0, e0, n0, k0), (l1, p1, e1, n1, k1) = runs[False], runs[True]
    assert _equal(l0, l1) and _equal(p0, p1) and _equal(e0, e1)
    assert n1 == n0 + 1
    assert "ema_buffers" not in k0 and k1 == k0 | {"ema_buffers"}


def test_ema_buffers_state_round_trip(m):
    model = _b0(m)
    step = _sgd(m, model, ema_momentum=0.1, ema_buffers=True)
    for i in range(2):
        step(*_data(8, 96, 70 + i))
    sd = step.state_dict()
    step2 = _sgd(m, _b0(m), ema_momentum=0.1, ema_buffers=True)
    step2.load_state_dict(sd)
    assert _equal(step2.ema_buffers, step.ema_buffers) and _equal(step2.opt.ema, step.opt.ema)
    with pytest.raises(ValueError, match="ema_momentum"):
        _sgd(m, _b0(m), ema_buffers=True)


# ------------------------------------------------------------------------------------------------------------- EMA twin
def _prep_ranges(model):
    from ml_cvnets_b200.engine import EvalStep
    out = []
    for prep in EvalStep(model)._prepared():
        for e in prep._entries:
            out.append((e[1].data_ptr(), e[1].data_ptr() + e[1].numel() * e[1].element_size()))
    return out


@pytest.mark.parametrize("kind", ["mobilevit_v2", "efficientnet"])
def test_ema_twin_state_logits_and_caches(m, kind):
    build = (lambda: _mv2(m)) if kind == "mobilevit_v2" else (lambda: _b0(m))
    model = build()
    step = _sgd(m, model, ema_momentum=0.1, ema_buffers=True)
    flat = step.ws.flat_buffers()
    ref = step.ema_buffers.clone()
    x = _data(16, 128, 80)[0]
    with torch.no_grad():
        model.eval()
        model(x)  # the live model's eval caches exist before the twin is made (deepcopy copies them)
        model.train()
    for i in range(5):
        step(*_data(8, 128, 90 + i))
        ref = E.ema_flat(ref, flat.clone(), 0.1)
    twin = step.ema_model()
    assert twin is step.ema_model() and not twin.training
    assert all(not p.requires_grad and p.grad is None for p in twin.parameters())
    sd, live_sd = twin.state_dict(), model.state_dict()
    assert list(sd) == list(live_sd)
    ema_p = step.opt.ema_parameters(model)
    o = 0
    for k, v in sd.items():
        if k in ema_p:
            assert _equal(v, ema_p[k]), k
        elif v.is_floating_point():
            assert _equal(v.reshape(-1), ref[o:o + v.numel()]), k
            o += v.numel()
        else:
            assert torch.equal(v, live_sd[k]), k  # num_batches_tracked: the live counter
    assert o == ref.numel()
    # its eval logits are those of a fresh model loaded with its state_dict
    fresh = build()
    fresh.load_state_dict({k: v.clone() for k, v in sd.items()})
    fresh.eval()
    with torch.no_grad():
        lt, lf = twin(x).clone(), fresh(x).clone()
    assert _equal(lt, lf)
    # its kernel-layout weight caches are its own
    mine, live = _prep_ranges(twin), _prep_ranges(model)
    assert mine and live
    assert not any(a < d and c < b for a, b in mine for c, d in live)


# ------------------------------------------------------------------------------------------------------------- EvalStep
def test_interleaved_captured_train_and_eval_read_current_weights(m, monkeypatch):
    from ml_cvnets_b200.engine import EvalStep
    model = _b0(m)
    step = _sgd(m, model, ema_momentum=0.1, ema_buffers=True)
    step.capture(*_data(8, 96, 100))
    evs = {"live": EvalStep(model).capture(batch=16, crop=(96, 96)), "ema": EvalStep(step.ema_model()).capture(batch=16, crop=(96, 96))}
    xv, yv = _data(16, 96, 101)

    def fresh_logits(src):
        f = _b0(m)
        f.load_state_dict({k: v.clone() for k, v in src.state_dict().items()})
        f.eval()
        with torch.no_grad():
            return f(xv).clone()

    for i in range(3):
        step(*_data(8, 96, 110 + i))
        for name, ev in evs.items():
            ev.update(xv, yv)
            got = ev.logits.clone()
            assert _equal(got, fresh_logits(ev.model)), (name, i)
    assert model.training
    for ev in evs.values():
        monkeypatch.setattr(ev, "_refresh", lambda force=False: None)
    step(*_data(8, 96, 120))
    for name, ev in evs.items():
        ev.update(xv, yv)
        assert not _equal(ev.logits.clone(), fresh_logits(ev.model)), name


def test_eval_graphs_contain_no_weight_refresh(m, monkeypatch):
    from ml_cvnets_b200 import ops
    from ml_cvnets_b200.engine import EvalStep
    model = _mv2(m).eval()
    ev = EvalStep(model)
    calls = []
    orig = ops.PreparedWeights.prepare

    def counting(self, force=True):
        n0 = ops.launch_count
        orig(self, force)
        if torch.cuda.is_current_stream_capturing() and ops.launch_count != n0:
            calls.append(self)

    monkeypatch.setattr(ops.PreparedWeights, "prepare", counting)
    ev.capture(batch=8, crop=(128, 128))
    assert not calls


@pytest.mark.parametrize("kind", ["mobilevit_v2", "efficientnet"])
def test_ragged_batch_in_the_captured_graph_is_padding_invariant(m, kind):
    from ml_cvnets_b200.engine import EvalStep
    model = (_mv2(m) if kind == "mobilevit_v2" else _b0(m)).eval()
    cap = EvalStep(model).capture(batch=100, crop=(128, 128))
    eag = EvalStep(model)
    xf, yf = _data(100, 128, 130)
    cap.update(xf, yf)  # the pad rows of the next batch then hold real images of this one
    cap.reset()
    x, y = _data(37, 128, 131)
    cap.update(x, y)
    eag.update(x, y)
    assert _equal(cap.logits[:37], eag.logits)
    assert _equal(cap.loss_sum, eag.loss_sum) and torch.equal(cap.counts, eag.counts)
    assert cap.compute() == eag.compute()
    with pytest.raises(ValueError, match="exceeds"):
        cap.update(*_data(101, 128, 132))
    with pytest.raises(ValueError, match="no CUDA graph"):
        cap.update(*_data(4, 96, 133))


AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True, "model.learn_augmentation.lr_multiplier": 1.0}
N_CLS = 100


def _recipe_case(m, kind):
    """(model, oracle shapes, oracle eval forward, crop) of a recipe's classifier with seeded weights (the parity tests' inputs)."""
    import efficientnet_ref as EF
    from oracle import cvnets_oracle as O
    if kind == "mobilevit_v2":
        return (m.MobileViTv2(m.default_opts(1.0, n_classes=N_CLS)), O.mobilevit_v2_shapes(1.0, n_classes=N_CLS),
                lambda P, x: O.mobilevit_v2_forward(P, x, width_multiplier=1.0, training=False), 256)
    if kind == "efficientnet_ra":
        return (m.EfficientNet(m.default_effnet_opts("b0", n_classes=N_CLS, **AUG)), EF.efficientnet_shapes("b0", n_classes=N_CLS),
                lambda P, x: EF.efficientnet_forward(P, x, mode="b0", training=False), 224)
    if kind == "mobilevit_v1_s":
        return (m.MobileViT(m.default_mit_opts("small", n_classes=N_CLS)), O.mobilevit_v1_shapes("small", n_classes=N_CLS),
                lambda P, x: O.mobilevit_v1_forward(P, x, mode="small", training=False), 256)
    return (m.VisionTransformer(m.default_vit_opts("tiny", n_classes=N_CLS)), O.vit_shapes("tiny", n_classes=N_CLS),
            lambda P, x: O.vit_forward(P, x, mode="tiny", training=False), 224)


@pytest.mark.parametrize("kind", ["mobilevit_v2", "efficientnet_ra", "mobilevit_v1_s", "vit_tiny"])
def test_captured_equals_eager_and_agrees_with_the_oracle(m, kind):
    from ml_cvnets_b200.engine import EvalStep
    from oracle import cvnets_oracle as O
    model, shapes, fwd, res = _recipe_case(m, kind)
    P = O.seeded_fill_(shapes, 17)
    missing, unexpected = model.load_state_dict(P, strict=False)
    assert not unexpected and all(k.startswith("neural_augmentor.") for k in missing)
    model = model.cuda().train()
    batches = [O.seeded_input((b, 3, res, res), 200 + b).cuda() for b in (100, 37)]
    Pc = O.clone_params(P, requires_grad=False, device="cuda")
    with torch.no_grad():
        targets = [fwd(Pc, x).argmax(1) for x in batches]  # the fp32 oracle's top-1: top1 below is the agreement with it
    cap, eag = EvalStep(model).capture(batch=100, crop=(res, res)), EvalStep(model)
    for x, y in zip(batches, targets):
        cap.update(x, y)
        eag.update(x, y)
    assert model.training  # restored after every pass
    got, want = cap.compute(), eag.compute()
    assert got == want, (got, want)
    assert got["top1"] >= 95.0, got
    assert cap.graph_pool_bytes() > 0


# ------------------------------------------------------------------------------------------------------------- data parallel
def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _ddp_worker(rank, world, port, q):
    import torch.distributed as dist
    import ml_cvnets_b200 as pkg
    from ml_cvnets_b200.engine import EvalStep
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank))
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    try:
        model = _mv2(pkg).eval()
        x, y = _data(32, 128, 300)
        ev = EvalStep(model).capture(batch=16, crop=(128, 128))
        ev.update(x[16 * rank:16 * (rank + 1)], y[16 * rank:16 * (rank + 1)])
        shard = ev.compute()
        single = None
        if rank == 0:
            ev1 = EvalStep(model)
            ev1.world = 1
            ev1.update(x, y)
            single = ev1.compute()
        q.put((rank, shard, single))
    finally:
        dist.destroy_process_group()


def test_data_parallel_compute_equals_single_gpu(m):
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_ddp_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=600) for _ in procs)
    for p in procs:
        p.join(timeout=60)
    (_, s0, single), (_, s1, _) = res
    assert s0 == s1
    assert s0["top1"] == single["top1"] and s0["top5"] == single["top5"]
    assert s0["loss"] == pytest.approx(single["loss"], rel=1e-12)

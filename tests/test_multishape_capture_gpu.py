"""Several captured input shapes in one TrainStep (-m gpu): the variable-batch sampler's (crop, batch) pairs each replayed from their own CUDA
graph, with one model, one optimizer state and one step arena shared by all of them.

  * EfficientNet-b0 with SGD-Nesterov and stochastic depth: captured replays in a random order equal eager steps in that order, bit for bit;
  * ViT-tiny with AdamW, EMA, mixup / cutmix and stochastic depth: within the run-to-run bound of an eager ViT run;
  * CLIP with RangeAugment at global batches that are not multiples of 8: the contrastive loss against an fp32 restatement, and the captured
    multi-shape step against the eager one;
  * guard rails (uncaptured shape, no arena re-plan, launch counts), the shared graph memory pool, and data parallel replay on two GPUs."""
import os
import random
import socket

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

STREAMING = 2  # cvb_set_mha_impl mode: the streaming attention kernels, whose backward is bitwise reproducible


@pytest.fixture(scope="module")
def m():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as pkg
    return pkg


def _batch(shape, n_classes, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(*shape, device="cuda", generator=g), torch.randint(0, n_classes, (shape[0],), device="cuda", generator=g)


def _effnet(m, sd=0.2):
    torch.manual_seed(0)
    return m.EfficientNet(m.default_effnet_opts("b0", n_classes=16, **{"model.classification.efficientnet.stochastic_depth_prob": sd})).cuda()


def _sgd_step(m, model):
    return m.TrainStep(model, optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None, label_smoothing=0.1,
                       ema_momentum=0.0005)


# (crop, batch) pairs scaled by area like the sampler's table: crop^2 * batch ~ constant
EFF_SMALL = ((64, 16), (96, 7), (128, 4))
EFF_MEM = ((64, 64), (96, 28), (128, 16))


def _warmup_passes(warmup=3):
    return max(warmup, 3)


def test_efficientnet_replays_equal_eager_steps_bitwise(m):
    """Capture three shapes, replay a fixed random order of 10 steps with repeats; a second TrainStep runs the identical sequence eagerly,
    capture's warm-up passes included.  Losses, parameters, buffers, momentum and EMA must agree bit for bit (the B0 step is deterministic)."""
    from ml_cvnets_b200 import ops
    examples = [_batch((B, 3, c, c), 16, 100 + c) for c, B in EFF_SMALL]
    rnd = random.Random(3)
    order = [rnd.randrange(len(EFF_SMALL)) for _ in range(10)]
    seq = [_batch((EFF_SMALL[i][1], 3, EFF_SMALL[i][0], EFF_SMALL[i][0]), 16, 1000 + k) for k, i in enumerate(order)]
    runs = []
    for captured in (True, False):
        model = _effnet(m)
        ts = _sgd_step(m, model)
        ops.rng_seed(7)
        if captured:
            ts.capture_shapes(examples)
        else:
            for _ in range(_warmup_passes()):
                for x, y in examples:
                    ts.step(x, y)
        losses = [ts.step(x, y).clone() for x, y in seq]
        torch.cuda.synchronize()
        runs.append((torch.stack(losses), ts.opt.flat_p.clone(), ts.opt.momentum_buffer.clone(), ts.opt.ema.clone(),
                     torch.cat([b.detach().flatten().float() for b in model.buffers()])))
        del ts, model
    print("orders", order, "losses", runs[0][0].tolist())
    assert torch.isfinite(runs[0][0]).all()
    for name, a, b in zip(("losses", "params", "momentum", "ema", "buffers"), runs[0], runs[1]):
        assert torch.equal(a, b), (name, float((a - b).abs().max()))


def test_vit_tiny_with_mixing_and_stochastic_depth_follows_eager(m):
    """ViT-tiny, AdamW + EMA, mixup / cutmix drawn per step by MixingSampler, stochastic depth 0.1, crops 128 / 192 / 224: the captured run and
    the eager run take the same first (eager) step exactly, then every parameter stays within AdamW's noise bound 2.5 * lr * steps (ViT steps
    are not bitwise reproducible: the LayerNorm-gain reductions depend on arrival order in their last bits)."""
    from ml_cvnets_b200 import _lib as L
    from ml_cvnets_b200 import ops
    lib = L.load()
    shapes = ((128, 12), (192, 5), (224, 4))
    lr = 1e-3
    examples = [_batch((B, 3, c, c), 100, 200 + c) for c, B in shapes]
    rnd = random.Random(5)
    order = [rnd.randrange(len(shapes)) for _ in range(8)]
    seq = [_batch((shapes[i][1], 3, shapes[i][0], shapes[i][0]), 100, 2000 + k) for k, i in enumerate(order)]
    torch.manual_seed(11)
    sampler = m.engine.MixingSampler()
    mixes = [sampler.sample(shapes[i][0], shapes[i][0]) for i in order]
    old = lib.cvb_set_mha_impl(STREAMING)
    runs = []
    try:
        for captured in (True, False):
            torch.manual_seed(0)
            model = m.VisionTransformer(m.default_vit_opts("tiny", n_classes=100, **{"model.classification.vit.stochastic_dropout": 0.1}))
            model = model.cuda().train()
            ts = m.TrainStep(model, lr=lr, weight_decay=0.05, max_norm=10.0, label_smoothing=0.1, ema_momentum=0.0005)
            ops.rng_seed(1234)
            first = float(ts.step(*examples[0]))
            steps = 1
            if captured:
                ts.capture_shapes(examples)
            else:
                for _ in range(_warmup_passes()):
                    for x, y in examples:
                        ts.step(x, y)
            steps += _warmup_passes() * len(examples)
            losses = []
            for (x, y), (kind, lam, box) in zip(seq, mixes):
                ts.set_mix(kind, lam, box)
                losses.append(float(ts.step(x, y)))
            steps += len(seq)
            torch.cuda.synchronize()
            runs.append((first, losses, ts.opt.flat_p.clone(), ts.opt.ema.clone()))
            del ts, model
    finally:
        lib.cvb_set_mha_impl(old)
    print("mixes", [k for k, _, _ in mixes], "losses", runs[0][1], runs[1][1])
    assert runs[0][0] == runs[1][0]
    assert all(torch.isfinite(torch.tensor(r[1])).all() for r in runs)
    assert max(abs(a - b) for a, b in zip(runs[0][1], runs[1][1])) <= 2e-2
    assert float((runs[0][2] - runs[1][2]).abs().max()) <= 2.5 * lr * steps
    assert float((runs[0][3] - runs[1][3]).abs().max()) <= 2.5 * lr * steps


# ------------------------------------------------------------------------------------------------------------------ CLIP
def _contrastive_ref(img, txt, ls):
    """contrastive_loss_clip.py:56-97 on one rank, fp32: logits = clamp(exp(logit_scale), 0, 100) * features products, labels arange."""
    s = torch.clamp(ls.exp(), 0, 100.0)
    lab = torch.arange(img.shape[0], device=img.device)
    return 0.5 * (F.cross_entropy(s * img @ txt.t(), lab) + F.cross_entropy(s * txt @ img.t(), lab))


@pytest.mark.parametrize("G", [13, 21, 5, 16])
def test_contrastive_loss_at_any_global_batch(m, G):
    d = 64
    g = torch.Generator(device="cuda").manual_seed(G)
    img0 = F.normalize(torch.randn(G, d, device="cuda", generator=g), dim=-1).bfloat16()
    txt0 = F.normalize(torch.randn(G, d, device="cuda", generator=g), dim=-1).bfloat16()
    ls0 = torch.tensor(2.3, device="cuda")
    img, txt, ls = img0.clone().requires_grad_(True), txt0.clone().requires_grad_(True), ls0.clone().requires_grad_(True)
    loss = m.clip_contrastive_loss(img, txt, ls)
    loss.backward()
    I, T, lr_ = img0.float().requires_grad_(True), txt0.float().requires_grad_(True), ls0.clone().requires_grad_(True)
    ref = _contrastive_ref(I, T, lr_)
    ref.backward()
    rel = lambda a, b: float((a.float() - b).norm() / b.norm())  # noqa: E731
    errs = (abs(float(loss) - float(ref)) / abs(float(ref)), rel(img.grad, I.grad), rel(txt.grad, T.grad),
            abs(float(ls.grad) - float(lr_.grad)) / abs(float(lr_.grad)))
    print(f"G={G}: loss / d img / d txt / d logit_scale relative errors {errs}")
    assert errs[0] <= 5e-3 and errs[1] <= 2e-2 and errs[2] <= 2e-2 and errs[3] <= 2e-2, errs


AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True}


def _clip(m):
    torch.manual_seed(0)
    opts = m.default_clip_opts("tiny", projection_dim=64, text_dim=128, text_layers=2, text_heads=4, vocab_size=1000, context_length=16, **AUG)
    return m.CLIP(opts).cuda().train()


def _clip_batch(B, crop, seed, L=16):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(1, 998, (B, L), generator=g)
    tok[torch.arange(B), torch.randint(2, L, (B,), generator=g)] = 999
    x = torch.rand(B, 3, crop, crop, generator=g)
    return x.cuda(), tok.cuda()


def _clip_forward_loss(m):
    def fl(model, im, tok, cfg):
        img, txt, scale, x_aug = model(im, tok)
        return m.clip_contrastive_loss(img, txt, scale, _cfg=cfg), x_aug
    return fl


def test_clip_range_augment_multishape_capture_follows_eager(m):
    """CLIP + RangeAugment (forward_loss, aug_loss) at batches 13 and 21: captured replays in a random order against eager steps in that order."""
    from ml_cvnets_b200 import _lib as L
    from ml_cvnets_b200 import ops
    lib = L.load()
    shapes = ((96, 13), (64, 21))
    lr = 1e-4
    examples = [_clip_batch(B, c, 300 + c) for c, B in shapes]
    rnd = random.Random(9)
    order = [rnd.randrange(len(shapes)) for _ in range(8)]
    seq = [_clip_batch(shapes[i][1], shapes[i][0], 3000 + k) for k, i in enumerate(order)]
    old = lib.cvb_set_mha_impl(STREAMING)
    runs = []
    try:
        for captured in (True, False):
            model = _clip(m)
            na = m.NeuralAugmentationLoss(target_value=(40, 10), curriculum_method="cosine", period=20)
            ts = m.TrainStep(model, lr=lr, weight_decay=0.2, max_norm=1.0, aug_loss=na, forward_loss=_clip_forward_loss(m))
            ops.rng_seed(77)
            first = float(ts.step(*examples[0]))
            steps = 1
            if captured:
                ts.capture_shapes(examples)
            else:
                for _ in range(_warmup_passes()):
                    for ex in examples:
                        ts.step(*ex)
            steps += _warmup_passes() * len(examples)
            losses = []
            for k, ex in enumerate(seq):
                ts.set_epoch(k)
                losses.append(float(ts.step(*ex)))
            steps += len(seq)
            torch.cuda.synchronize()
            runs.append((first, losses, ts.opt.flat_p.clone()))
            del ts, model
    finally:
        lib.cvb_set_mha_impl(old)
    print("losses", runs[0][1], runs[1][1])
    assert runs[0][0] == runs[1][0]
    assert all(torch.isfinite(torch.tensor(r[1])).all() for r in runs)
    assert max(abs(a - b) for a, b in zip(runs[0][1], runs[1][1])) <= 2e-2
    assert float((runs[0][2] - runs[1][2]).abs().max()) <= 2.5 * lr * steps


# ------------------------------------------------------------------------------------------------------------------ guard rails
def test_guard_rails(m):
    from ml_cvnets_b200 import ops
    examples = [_batch((B, 3, c, c), 16, 400 + c) for c, B in EFF_SMALL]
    # single-shape capture: the launch count is the one the same shape gets in a multi-shape capture, and equals a steady eager step's
    ts1 = _sgd_step(m, _effnet(m))
    ts1.capture(*examples[2])
    single = ts1.launches_per_step
    assert ts1.launches_per_shape == {tuple(tuple(t.shape) for t in examples[2]): single}
    assert len(ts1.static_inputs) == 2 and ts1.static_inputs[0].shape == examples[2][0].shape
    del ts1
    ts0 = _sgd_step(m, _effnet(m))
    for _ in range(3):
        ts0.step(*examples[2])
    n0 = ops.launch_count
    ts0.step(*examples[2])
    eager = ops.launch_count - n0
    del ts0
    ts = _sgd_step(m, _effnet(m))
    ts.capture_shapes(examples)
    assert set(ts.captured_shapes) == {tuple(tuple(t.shape) for t in ex) for ex in examples}
    key = tuple(tuple(t.shape) for t in examples[2])
    print("launches: single capture", single, "multi", ts.launches_per_shape, "eager", eager)
    assert ts.launches_per_shape[key] == single and ts.launches_per_step == max(ts.launches_per_shape.values())
    ptrs = (ts.ws._buf32.data_ptr(), ts.ws._buf64.data_ptr())
    for x, y in examples + examples[::-1]:
        loss = ts.step(x, y)
    torch.cuda.synchronize()
    assert torch.isfinite(loss)
    assert (ts.ws._buf32.data_ptr(), ts.ws._buf64.data_ptr()) == ptrs and ts.ws.frozen
    x, y = _batch((5, 3, 64, 64), 16, 1)
    with pytest.raises(ValueError, match="captured"):
        ts.step(x, y)
    with pytest.raises(AssertionError):
        ts.capture(*examples[0])


def test_shared_pool_memory(m):
    """Three EfficientNet shapes in one pool reserve at most 1.25x what the most demanding shape's graph reserves on its own."""
    examples = [_batch((B, 3, c, c), 16, 500 + c) for c, B in EFF_MEM]
    single = []
    for ex in examples:
        ts = _sgd_step(m, _effnet(m))
        ts.capture(*ex)
        single.append(ts.graph_pool_bytes())
        del ts
        torch.cuda.empty_cache()
    ts = _sgd_step(m, _effnet(m))
    ts.capture_shapes(examples)
    multi = ts.graph_pool_bytes()
    print(f"graph pool bytes: single shapes {single}, all three {multi} ({multi / max(single):.3f}x the largest)")
    assert 0 < multi <= 1.25 * max(single)


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
    from oracle import cvnets_oracle as O
    try:
        shapes = ((128, 8), (256, 2))
        shards = {s: [_batch((s[1], 3, s[0], s[0]), 1000, 600 + 10 * r + s[0]) for r in range(world)] for s in shapes}
        P = O.seeded_fill_(O.mobilevit_v2_shapes(0.5), 7)

        def fresh():
            model = m.MobileViTv2(m.default_opts(width_multiplier=0.5))
            model.load_state_dict(P, strict=True)
            return model.cuda().eval()  # running statistics: the exchange itself is checked tightly

        def reference(s):
            tot = None
            for x, y in shards[s]:
                ts = m.TrainStep(fresh(), lr=0.0, weight_decay=0.0, data_parallel=False)
                ts.step(x, y)
                tot = ts.ws.flat_g.clone() if tot is None else tot + ts.ws.flat_g
            return tot / world

        refs = {s: reference(s) for s in shapes}
        ts = m.TrainStep(fresh(), lr=0.0, weight_decay=0.0, n_buckets=3)
        ts.capture_shapes([shards[s][rank] for s in shapes])
        errs = []
        for s in shapes + shapes[::-1]:
            ts.step(*shards[s][rank])
            errs.append(float((ts.ws.flat_g / world - refs[s]).norm() / refs[s].norm()))
        ts.set_lr(1e-3)
        for s in (shapes[0], shapes[1], shapes[1], shapes[0]):
            ts.step(*shards[s][rank])
        flat = ts.opt.flat_p.clone()
        gathered = [torch.empty_like(flat) for _ in range(world)]
        dist.all_gather(gathered, flat)
        drift = max(float((g - gathered[0]).abs().max()) for g in gathered)
        torch.cuda.synchronize()
        q.put((rank, errs, len(ts.ws._bucket_range), drift))
    except BaseException as e:  # the parent must never wait for a result that will not come
        q.put((rank, repr(e)[:500], -1, -1.0))
    q.close()
    q.join_thread()
    # a captured CUDA graph that contains NCCL kernels is still alive here: leave without the collective shutdown
    os._exit(0)


def test_data_parallel_multishape_replay():
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
    for rank, errs, n_fire, drift in res:
        assert not isinstance(errs, str), f"rank {rank} failed: {errs}"
        print(f"rank {rank}: rel-L2 vs the single-GPU gradient of the concatenated batch per replay {errs}; buckets {n_fire}; drift {drift:.3g}")
        assert all(e <= 5e-3 for e in errs), errs
        assert n_fire == 3
        assert drift == 0.0

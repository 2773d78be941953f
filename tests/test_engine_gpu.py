"""engine.TrainStep / cross_entropy / FlatAdamW / StepWorkspace (-m gpu): the fused step against the torch pipeline the reference runs
(engine/training_engine.py:257-312: F.cross_entropy -> GradScaler.scale().backward() -> unscale_ -> clip_grad_norm_ -> AdamW -> update)."""
import copy

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as m
    return m


def rel_l2(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


@pytest.mark.parametrize("B,C,smoothing,ignore", [(128, 1000, 0.1, False), (7, 1000, 0.0, False), (33, 37, 0.2, True), (4, 8, 0.1, True)])
def test_cross_entropy_matches_torch(pkg, B, C, smoothing, ignore):
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + C)
    logits = (3 * torch.randn(B, C, device="cuda", generator=g)).bfloat16()
    y = torch.randint(0, C, (B,), device="cuda", generator=g)
    if ignore:
        y[::3] = -1
    ours_in = logits.clone().requires_grad_(True)
    ref_in = logits.float().requires_grad_(True)
    loss = pkg.cross_entropy(ours_in, y, label_smoothing=smoothing, ignore_index=-1)
    ref = F.cross_entropy(ref_in, y, ignore_index=-1, label_smoothing=smoothing)
    assert abs(float(loss) - float(ref)) <= 2e-5 * max(1.0, abs(float(ref))), (float(loss), float(ref))
    gscale = torch.tensor(3.0, device="cuda")
    loss.backward(gscale)
    ref.backward(gscale)
    # dlogits are stored in bf16 (they feed the bf16 classifier GEMMs): bf16 rounding is the tolerance
    assert rel_l2(ours_in.grad, ref_in.grad) <= 4e-3
    assert float((ours_in.grad.float() - ref_in.grad).abs().max()) <= 2 ** -8 * float(ref_in.grad.abs().max()) + 1e-8


def _small_model(pkg, seed=11, width=0.5):
    model = pkg.MobileViTv2(pkg.default_opts(width_multiplier=width))
    model.load_state_dict(O.seeded_fill_(O.mobilevit_v2_shapes(width), seed), strict=True)
    return model.cuda().train()


def test_train_step_gradients_match_autograd_path(pkg):
    """Workspace mode (gradients written in place, Functions return None) == the plain autograd path of the same kernels, bitwise.

    Both paths launch the same kernels with the same rounding points, and every multi-CTA reduction is order-independent (fp64 partial sums,
    fp64 weight-gradient scratch), so repeated autograd runs and the three workspace steps (step 0 plans the arena, step 1 builds the
    descriptor tables, step 2 runs fully planned) must all produce the same gradient bits."""
    B, res = 16, 128
    x = O.seeded_input((B, 3, res, res), 5).cuda()
    y = (torch.arange(B, device="cuda") * 37) % 1000
    scale = 65536.0
    refs = []
    for _ in range(2):
        ref = _small_model(pkg)
        logits = ref(x)
        (pkg.cross_entropy(logits, y, label_smoothing=0.1) * scale).backward()
        refs.append(ref)
    ref, ref2 = refs
    for (k, p), (_, q) in zip(ref.named_parameters(), ref2.named_parameters()):
        assert torch.equal(p.grad, q.grad), f"autograd path, two runs: {k} differs in {int((p.grad != q.grad).sum())} elements"
    model = _small_model(pkg)
    ts = pkg.TrainStep(model, lr=0.0, weight_decay=0.0)  # lr 0: parameters stay put, gradients can be compared after the step
    for it in range(3):
        loss = ts.step(x, y)
        bad = [k for (k, p), (_, q) in zip(model.named_parameters(), ref.named_parameters()) if not torch.equal(p.grad, q.grad)]
        assert not bad, f"step {it}: {len(bad)} workspace gradients differ from the autograd path's, e.g. {bad[:5]}"
    assert abs(float(loss) - float(F.cross_entropy(logits.float(), y, label_smoothing=0.1))) < 2e-2
    assert int(model.conv_1.block.norm.num_batches_tracked) == 3


def test_lazy_module_boundaries_match_materialised_outputs(pkg):
    """functional.LazyBN: handing module outputs over pre-BatchNorm (normalised by the consumer's load mode, BN-backward sums taken in the
    consumer's input-gradient epilogue) is the same forward computation as materialising them: logits and BatchNorm running statistics are
    bitwise equal.  The gradients differ at one rounding point: the lazy path applies the activation derivative to the consumer's fp32
    accumulator and rounds dz to bf16 once, the materialised path rounds the gradient of the activated output to bf16 first and then
    bn_bwd_reduce rounds dz again (measured: whole-gradient rel-L2 8.6e-3 at this shape).  Each path is bitwise reproducible run to run."""
    B, res = 16, 128
    x = O.seeded_input((B, 3, res, res), 6).cuda()
    y = (torch.arange(B, device="cuda") * 41) % 1000
    out = {}
    for fuse in (True, False, True):
        model = _small_model(pkg)
        model.fuse_boundaries = fuse
        logits = model(x)
        pkg.cross_entropy(logits, y, label_smoothing=0.1).backward()
        out.setdefault(fuse, []).append((logits.detach().float().clone(), torch.cat([p.grad.flatten() for p in model.parameters()]).clone(),
                                         {k: b.clone() for k, b in model.named_buffers()}))
    (la, ga, ba), (la2, ga2, ba2) = out[True]
    (lb, gb, bb), = out[False]
    assert torch.equal(la2, la) and torch.equal(ga2, ga), "lazy path: two runs differ"
    assert all(torch.equal(ba2[k], ba[k]) for k in ba), "lazy path: two runs leave different buffers"
    e_g = rel_l2(ga, gb)
    print(f"lazy vs materialised: whole-gradient rel-L2 {e_g:.3g}")
    assert torch.equal(la, lb), f"logits: lazy vs materialised rel-L2 {rel_l2(la, lb):.3g}"
    assert e_g <= 1e-2
    for k in ba:
        assert torch.equal(ba[k], bb[k]), k


def test_train_step_matches_torch_pipeline_and_graph_replay(pkg):
    """Three optimizer steps: TrainStep eager == TrainStep captured, bitwise (loss trajectory and parameters), and both follow the torch
    pipeline run on the same kernels (loss trajectory within 3e-2: torch computes the loss from bf16 logits in fp32, unscales, clips and
    updates with its own kernels, and AdamW's first updates turn those last-bit differences into +-lr steps)."""
    B, res = 16, 128
    xs = [O.seeded_input((B, 3, res, res), 100 + i).cuda() for i in range(4)]
    ys = [(torch.arange(B, device="cuda") * (i + 3)) % 1000 for i in range(4)]
    # torch pipeline
    ref = _small_model(pkg)
    groups, _ = ref.get_trainable_parameters(weight_decay=0.05, no_decay_bn_filter_bias=True)
    opt = torch.optim.AdamW(groups, lr=2e-3, betas=(0.9, 0.999))
    scaler = torch.amp.GradScaler("cuda", enabled=True)
    ref_losses = []
    for x, y in zip(xs, ys):
        loss = F.cross_entropy(ref(x).float(), y, label_smoothing=0.1)
        opt.zero_grad(set_to_none=True)
        scaler.scale(loss).backward()
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(list(ref.parameters()), 10.0)
        scaler.step(opt)
        scaler.update()
        ref_losses.append(float(loss))
    # eager TrainStep
    m1 = _small_model(pkg)
    t1 = pkg.TrainStep(m1, lr=2e-3, weight_decay=0.05, max_norm=10.0, label_smoothing=0.1)
    l1 = [float(t1.step(x, y)) for x, y in zip(xs, ys)]
    # captured TrainStep: the warm-up steps inside capture() use lr = 0 so that the trajectory starts from the same weights
    m2 = _small_model(pkg)
    t2 = pkg.TrainStep(m2, lr=0.0, weight_decay=0.0, max_norm=10.0, label_smoothing=0.1)
    sd0 = {k: v.clone() for k, v in m2.state_dict().items()}
    t2.capture(xs[0], ys[0])
    m2.load_state_dict(sd0)  # undo the BatchNorm running-stat updates of the warm-up steps
    t2.opt.exp_avg.zero_(); t2.opt.exp_avg_sq.zero_(); t2.opt.step_count.zero_(); t2.opt.scale.copy_(torch.tensor([65536.0, 0.0]))
    t2.opt.wd.copy_(t1.opt.wd)
    t2.set_lr(2e-3)
    l2 = [float(t2.step(x, y)) for x, y in zip(xs, ys)]
    print("losses: eager", l1, "captured", l2, "torch pipeline", ref_losses)
    assert l1 == l2, (l1, l2)
    assert abs(l1[0] - ref_losses[0]) <= 2e-3 * abs(l1[0]), (l1, ref_losses)
    for a, r in zip(l1, ref_losses):
        assert abs(a - r) <= 3e-2 * abs(r), (l1, ref_losses)
    for (k, p), (_, q) in zip(m1.named_parameters(), m2.named_parameters()):
        assert torch.equal(p, q), k
    for (k, p), (_, q) in zip(m1.named_buffers(), m2.named_buffers()):
        assert torch.equal(p, q), k


def test_ema_and_lr_schedule_and_state_dict(pkg):
    B, res = 4, 64
    x = O.seeded_input((B, 3, res, res), 9).cuda()
    y = torch.arange(B, device="cuda")
    model = _small_model(pkg)
    mom = 0.05
    ts = pkg.TrainStep(model, lr=1e-3, ema_momentum=mom)
    ema_ref = {k: p.detach().clone() for k, p in model.named_parameters()}
    for it in range(3):
        ts.set_lr(1e-3 * (it + 1))
        ts.step(x, y)
        for k, p in model.named_parameters():  # cvnets/misc/averaging_utils.py:55
            ema_ref[k] = ema_ref[k] * (1.0 - mom) + mom * p.detach()
    ema = ts.opt.ema_parameters(model)
    for k, v in ema_ref.items():
        assert rel_l2(ema[k], v) <= 1e-5, k
    assert abs(float(ts.opt.hp[0]) - 3e-3) < 1e-9
    sd = ts.state_dict()
    assert float(sd["step"]) == 3.0
    ts2 = pkg.TrainStep(_small_model(pkg), lr=5.0, ema_momentum=mom)
    ts2.load_state_dict(sd)
    assert torch.equal(ts2.opt.exp_avg, ts.opt.exp_avg) and abs(float(ts2.opt.hp[0]) - 3e-3) < 1e-9


def test_eval_after_train_step_sees_new_weights(pkg):
    """ADVICE r1: raw-pointer / replayed optimizer updates do not bump Tensor._version; eval-mode weight caches must still refresh."""
    B, res = 4, 64
    x = O.seeded_input((B, 3, res, res), 9).cuda()
    y = torch.arange(B, device="cuda")
    model = _small_model(pkg)
    ts = pkg.TrainStep(model, lr=5e-2)
    ts.capture(x, y)
    model.eval()
    with torch.no_grad():
        a = model(x).float().clone()
    model.train()
    for _ in range(3):
        ts.step(x, y)
    model.eval()
    with torch.no_grad():
        b = model(x).float()
        fresh = pkg.MobileViTv2(pkg.default_opts(width_multiplier=0.5)).cuda().eval()
        fresh.load_state_dict(model.state_dict(), strict=True)
        c = fresh(x).float()
    assert rel_l2(b, c) <= 1e-3, "eval forward used stale bf16 weight copies"
    assert rel_l2(a, b) > 1e-2, "weights did not move?"


@pytest.mark.parametrize("kind", ["mixup", "cutmix"])
def test_batch_mixing_fused_into_stem_gather_and_loss(pkg, kind):
    """SURVEY.md 8f row 3: RandomMixup / RandomCutmix (data/transforms/image_torch.py:99-137, :290-342) applied inside the stem's gather and
    the loss kernels == the reference's formulation (mixed images + soft targets) computed with torch."""
    from ml_cvnets_b200 import ops
    B, H, W, C = 6, 32, 48, 1000
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(B, 3, H, W, device="cuda", generator=g)
    y = torch.randint(0, C, (B,), device="cuda", generator=g)
    lam, box = (0.3, (0, 0, 0, 0)) if kind == "mixup" else (1.0 - (30 - 10) * (20 - 4) / (W * H), (10, 4, 30, 20))
    mix = torch.tensor([1.0 if kind == "mixup" else 2.0, lam, *box], device="cuda", dtype=torch.float32)
    rolled = x.roll(1, 0)
    if kind == "mixup":
        xm = x * lam + rolled * (1.0 - lam)
    else:
        xm = x.clone()
        x1, y1, x2, y2 = box
        xm[:, :, y1:y2, x1:x2] = rolled[:, :, y1:y2, x1:x2]
    a, b = ops.stem_im2col(x, mix=mix).float(), ops.stem_im2col(xm).float()
    assert float((a - b).abs().max()) <= 2 ** -7 * float(b.abs().max()) and rel_l2(a, b) <= 1e-3  # at most a bf16 ulp (fma vs mul+add)
    logits = (3 * torch.randn(B, C, device="cuda", generator=g)).bfloat16()
    soft = F.one_hot(y, C).float() * lam + F.one_hot(y.roll(1, 0), C).float() * (1.0 - lam)
    ref_in = logits.float().requires_grad_(True)
    ref = F.cross_entropy(ref_in, soft, label_smoothing=0.1)
    ref.backward()
    ours_in = logits.clone().requires_grad_(True)
    from types import SimpleNamespace
    loss = pkg.cross_entropy(ours_in, y, _cfg=SimpleNamespace(label_smoothing=0.1, ignore_index=-1, scale=None, mix=mix))
    loss.backward()
    assert abs(float(loss) - float(ref)) <= 2e-5 * abs(float(ref)), (float(loss), float(ref))
    assert rel_l2(ours_in.grad, ref_in.grad) <= 4e-3
    # end to end through TrainStep (eval-mode BatchNorm keeps the comparison free of batch-statistics amplification)
    model = _small_model(pkg).eval()
    ts = pkg.TrainStep(model, lr=0.0, weight_decay=0.0)
    xs, ys = O.seeded_input((8, 3, 64, 64), 77).cuda(), torch.arange(8, device="cuda") * 7
    if kind == "cutmix":
        lam2, box2 = 1.0 - (40 - 8) * (50 - 20) / (64 * 64), (8, 20, 40, 50)
    else:
        lam2, box2 = 0.65, (0, 0, 0, 0)
    ts.set_mix(kind, lam2, box2)
    l_mixed = float(ts.step(xs, ys))
    rolled = xs.roll(1, 0)
    xm = xs * lam2 + rolled * (1 - lam2) if kind == "mixup" else xs.clone()
    if kind == "cutmix":
        xm[:, :, box2[1]:box2[3], box2[0]:box2[2]] = rolled[:, :, box2[1]:box2[3], box2[0]:box2[2]]
    with torch.no_grad():
        lg = model(xm).float()
    softs = F.one_hot(ys, 1000).float() * lam2 + F.one_hot(ys.roll(1, 0), 1000).float() * (1 - lam2)
    l_ref = float(F.cross_entropy(lg, softs, label_smoothing=0.1))
    ts.set_mix(None)
    l_plain = float(ts.step(xs, ys))
    assert abs(l_mixed - l_ref) <= 3e-3 * abs(l_ref), (l_mixed, l_ref)
    assert abs(l_plain - l_ref) > 1e-4  # the mixing really changed the step

"""RangeAugment on the GPU: the kernels of csrc/neural_aug.cu against the fp32 restatement (tests/range_augment_ref.py) fed the kernels' own
draws, the draws' statistics, the stem input gradient against torch, the drop-in models under a plain ``loss.backward()``, a TrainStep with the
composite loss, and bitwise run-to-run reproducibility of the augmented training step."""
import math

import pytest
import torch
import torch.nn.functional as F

import range_augment_ref as R

pytestmark = pytest.mark.gpu

AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True, "model.learn_augmentation.lr_multiplier": 1.0}


@pytest.fixture(scope="module")
def m():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as pkg
    return pkg


def _key(seed):
    return torch.tensor([seed * 0x9E3779B1 + 12345], device="cuda", dtype=torch.int64)


def _draws(ops, key, B, H, W, enabled=7):
    tab = torch.empty(4 + 3 * B, device="cuda", dtype=torch.float32)
    ops.na_plan(key, B, enabled, tab)
    return tab, R.draws_from_kernels(tab, ops.na_noise(key, B, H, W))


def _raw(enabled=7, seed=0):
    g = torch.Generator().manual_seed(seed)
    init = {"brightness": (0.5, 1.5), "contrast": (0.5, 1.5), "noise": (0.0, 0.1)}
    out = {}
    for k, name in enumerate(R.NAMES):
        if enabled >> k & 1:
            out[name] = tuple(torch.tensor(v + 0.4 * float(torch.randn((), generator=g)), device="cuda") for v in init[name])
    return out


def _flat6(raw):
    return [raw[n][i] if n in raw else None for n in R.NAMES for i in (0, 1)]


def _image(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, 3, H, W, generator=g)
    x[0, :, :3] = 0.0
    x[-1, :, -3:] = 1.0
    return x.cuda()


MIXES = {"plain": None, "mixup": [1.0, 0.3, 0, 0, 0, 0], "cutmix": [2.0, 0.75, 3, 5, 20, 17]}


@pytest.mark.parametrize("mix", list(MIXES))
@pytest.mark.parametrize("B,H,W,enabled", [(6, 24, 32, 7), (5, 32, 24, 7), (1, 16, 16, 7), (8, 32, 32, 3), (7, 24, 24, 5)])
def test_forward_kernels_against_oracle(m, mix, B, H, W, enabled):
    ops = m.ops
    x = _image(B, H, W, B * 100 + H)
    mixv = None if MIXES[mix] is None else torch.tensor(MIXES[mix], device="cuda")
    raw = _raw(enabled, seed=B)
    for seed in range(4):
        key = _key(seed + 7 * B)
        tab, draws = _draws(ops, key, B, H, W, enabled)
        mu = torch.zeros(2, 3 * B, device="cuda", dtype=torch.float64)
        coef = torch.empty(3 * B, 3, device="cuda")
        sq = torch.empty(B, 3, device="cuda", dtype=torch.float64)
        ops.na_stats(x, mixv, key, bool(enabled & 4), mu)
        xm = R.mixed(x, MIXES[mix] or [0, 1, 0, 0, 0, 0])
        torch.testing.assert_close(mu[0].view(B, 3), xm.double().mean(dim=[2, 3]), atol=1e-6, rtol=1e-6)
        ops.na_compose(tab, mu, _flat6(raw), B, coef)
        y = ops.na_apply(x, mixv, key, coef, bool(enabled & 4), sq)
        ref = R.augment(xm, raw, draws)
        torch.testing.assert_close(y, ref, atol=2e-5, rtol=1e-4)
        torch.testing.assert_close(sq, ((y.double() - xm.double()) ** 2).sum(dim=[2, 3]), atol=1e-9, rtol=1e-6)  # fp32 squares, fp64 sums


@pytest.mark.parametrize("B,H,W", [(6, 24, 32), (3, 32, 32), (1, 16, 16)])
@pytest.mark.parametrize("mix", ["plain", "mixup", "cutmix"])
def test_backward_kernels_against_autograd(m, B, H, W, mix):
    """bwd_reduce (against an fp64 restatement) and param_grad (against autograd of the oracle on the same draws), with the loss term."""
    ops = m.ops
    x = _image(B, H, W, 5 + B)
    mixv = None if MIXES[mix] is None else torch.tensor(MIXES[mix], device="cuda")
    xm = R.mixed(x, MIXES[mix] or [0, 1, 0, 0, 0, 0])
    raw = _raw(7, seed=B + 1)
    key = _key(99 + B)
    tab, draws = _draws(ops, key, B, H, W)
    mu = torch.zeros(2, 3 * B, device="cuda", dtype=torch.float64)
    coef = torch.empty(3 * B, 3, device="cuda")
    sq = torch.empty(B, 3, device="cuda", dtype=torch.float64)
    ops.na_stats(x, mixv, key, True, mu)
    ops.na_compose(tab, mu, _flat6(raw), B, coef)
    y = ops.na_apply(x, mixv, key, coef, True, sq)
    dY = torch.randn(B, 3, H, W, device="cuda", generator=torch.Generator("cuda").manual_seed(B))
    g_sq = torch.rand(B, 3, device="cuda", dtype=torch.float64) * 1e-3
    red = torch.zeros(3 * B, 3, device="cuda", dtype=torch.float64)
    ops.na_bwd_reduce(dY, g_sq, x, mixv, key, coef, True, red)
    eps = ops.na_noise(key, B, H, W).double()
    A, Bc, C = [coef[:, i].double().view(B, 3, 1, 1) for i in range(3)]
    pre = A * xm.double() + Bc + C * eps
    g = torch.where((pre >= 0) & (pre <= 1), dY.double() + 2 * g_sq.view(B, 3, 1, 1) * (pre.clamp(0, 1) - xm.double()), torch.zeros_like(pre))
    ref_red = torch.stack([(g * xm.double()).sum([2, 3]), g.sum([2, 3]), (g * eps).sum([2, 3])], -1).view(3 * B, 3)
    torch.testing.assert_close(red, ref_red, atol=1e-4, rtol=1e-5)
    grads = [torch.zeros((), device="cuda") if p is not None else None for p in _flat6(raw)]
    ops.na_param_grad(tab, mu, red, _flat6(raw), B, grads)
    params = {n: tuple(p.clone().requires_grad_(True) for p in raw[n]) for n in raw}
    yo = R.augment(xm, params, draws)
    total = (yo * dY).sum() + (g_sq.float() * ((yo - xm) ** 2).sum([2, 3])).sum()
    ref = torch.autograd.grad(total, [p for n in R.NAMES for p in params[n]])
    for i, (a, b) in enumerate(zip([g for g in grads if g is not None], ref)):
        torch.testing.assert_close(a, b, atol=2e-3 * max(1.0, float(b.abs())), rtol=2e-3, msg=lambda msg, i=i: f"param {i}: {msg}")


@pytest.mark.parametrize("B", [1, 7, 64])
def test_loss_kernels(m, B):
    ops = m.ops
    H, W = 16, 24
    sq = torch.rand(B, 3, device="cuda", dtype=torch.float64) * 3.0
    table = torch.tensor([R.psnr_to_mse(p) for p in (40.0, 30.0, 10.0)], device="cuda")
    ce = torch.tensor(2.5, device="cuda")
    for epoch in (0, 1, 2, 9):
        step = torch.tensor([epoch], device="cuda", dtype=torch.int64)
        loss, parts = torch.empty((), device="cuda"), torch.empty(2, device="cuda")
        ops.na_loss_fwd(sq, H, W, table, step, 100.0, loss, w_na=0.7, ce=ce, w_ce=1.3, parts=parts)
        t = float(table[min(epoch, 2)])
        sq_t = sq.float().sum(1).clone().requires_grad_(True)
        mse = sq_t * 65025.0 / (3 * H * W)
        na = F.smooth_l1_loss(mse, torch.full_like(mse, t)) * (100.0 / 65025.0)
        torch.testing.assert_close(parts[1], na.detach(), atol=1e-6, rtol=1e-5)
        torch.testing.assert_close(loss, 1.3 * ce + 0.7 * na.detach(), atol=1e-6, rtol=1e-5)
        (gref,) = torch.autograd.grad(0.7 * na, sq_t)
        gout, gscale, g_ce = torch.tensor(2.0, device="cuda"), torch.tensor(8.0, device="cuda"), torch.empty((), device="cuda")
        g_sq = ops.na_loss_bwd(sq, H, W, table, step, 100.0, gout, gscale, w_na=0.7, g_ce=g_ce, w_ce=1.3)
        torch.testing.assert_close(g_sq.float(), (16.0 * gref).view(B, 1).expand(B, 3), atol=1e-9, rtol=1e-5)
        assert float(g_ce) == pytest.approx(2.6)


def _stem_weight(C0, seed):
    g = torch.Generator().manual_seed(seed)
    w = (torch.randn(C0, 3, 3, 3, generator=g) * 0.3).cuda()
    Ws = torch.zeros(C0, 32, device="cuda", dtype=torch.bfloat16)
    Ws[:, :27] = w.reshape(C0, 27).to(torch.bfloat16)
    return w, Ws


@pytest.mark.parametrize("C0", [16, 32, 40, 64])
@pytest.mark.parametrize("B,H,W", [(1, 32, 32), (3, 18, 22), (5, 64, 48), (64, 112, 112)])
def test_stem_input_gradient(m, C0, B, H, W):
    Ho, Wo = H // 2, W // 2
    g = torch.Generator("cuda").manual_seed(C0 + B)
    dz = torch.randn(B * Ho * Wo, C0, device="cuda", generator=g).to(torch.bfloat16)
    y = torch.randn(B * Ho * Wo, C0, device="cuda", generator=g).to(torch.bfloat16)
    coef = torch.randn(3, C0, device="cuda", generator=g) * 0.5
    w, Ws = _stem_weight(C0, C0)
    dX = m.ops.stem_dgrad(dz, y, coef, Ws, B, Ho, Wo)
    dy = (coef[0] * dz.float() + coef[1] * y.float() + coef[2]).to(torch.bfloat16).float()
    dy4 = dy.view(B, Ho, Wo, C0).permute(0, 3, 1, 2)
    w4 = Ws[:, :27].float().view(C0, 3, 3, 3)
    ref = torch.nn.grad.conv2d_input((B, 3, H, W), w4, dy4, stride=2, padding=1)
    # dy is rounded to bf16 after a fused multiply-add in the kernel and after separate roundings here: a rounding may flip by one bf16 ulp
    # (2^-8 relative) in either, so each contribution may differ by that much
    bound = torch.nn.grad.conv2d_input((B, 3, H, W), w4.abs(), dy4.abs(), stride=2, padding=1) * 2.0 ** -8 + 1e-4
    assert ((dX - ref).abs() <= bound).all(), float(((dX - ref).abs() - bound).max())
    assert float((dX - ref).abs().mean()) < 1e-5 * max(1.0, float(ref.abs().mean()))  # flips are rare: the bulk agrees to fp32 summation order


def test_draw_statistics(m):
    from scipy import stats
    ops = m.ops
    B, H, W = 10, 8, 8
    counts = torch.zeros(3, B)
    orders, us = set(), []
    for seed in range(600):
        tab = torch.empty(4 + 3 * B, device="cuda")
        ops.na_plan(_key(seed), B, 7, tab)
        t = tab.cpu()
        orders.add(tuple(int(v) for v in t[:3]))
        assert int(t[3]) == 3
        rows = t[4:].view(3, B)
        sel = rows >= 0
        assert (sel.sum(1) == B // 2).all()  # exactly max(1, B // 2) distinct samples per augmentation
        counts += sel.float()
        us.append(rows[sel])
    assert len(orders) == 6
    expect = 600 * (B // 2) / B
    assert ((counts - expect).abs() < 5 * math.sqrt(expect)).all(), counts
    u = torch.cat(us).numpy()
    assert (u >= 0).all() and (u < 1).all()
    assert stats.kstest(u, "uniform").pvalue > 1e-4
    eps = ops.na_noise(_key(3), 16, 64, 64)
    assert abs(float(eps.mean())) < 0.01 and abs(float(eps.var()) - 1.0) < 0.02
    tab = torch.empty(4 + 3, device="cuda")
    ops.na_plan(_key(1), 1, 7, tab)
    assert (tab[4:] >= 0).all()  # B = 1: the one sample is always augmented


def test_graph_replay_draws_fresh_values(m):
    ops = m.ops
    ops.rng_seed(5, device="cuda")
    B = 8
    tab = torch.empty(4 + 3 * B, device="cuda")
    ops.na_plan(ops.rng_next("cuda"), B, 7, tab)  # warm the module
    torch.cuda.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        key = ops.rng_next("cuda")
        ops.na_plan(key, B, 7, tab)
    seen = []
    for _ in range(3):
        graph.replay()
        torch.cuda.synchronize()
        seen.append(tab.clone())
    assert not torch.equal(seen[0], seen[1]) and not torch.equal(seen[1], seen[2])


def _effnet(m, seed=0, **extra):
    from ml_cvnets_b200.models_effnet import default_effnet_opts
    torch.manual_seed(seed)
    return m.EfficientNet(default_effnet_opts("b0", n_classes=10, **AUG, **extra)).cuda().train()


def _mit(m, seed=0):
    from ml_cvnets_b200.models_mit import default_mit_opts
    torch.manual_seed(seed)
    return m.MobileViT(default_mit_opts("xx_small", n_classes=10, **{"model.classification.classifier_dropout": 0.0, "model.classification.mit.dropout": 0.0,
                                                                      "model.classification.mit.attn_dropout": 0.0}, **AUG)).cuda().train()


def _replay_draws(m, state, B, H, W):
    """The draws of the first key drawn from generator state ``state`` (the augmentor's, when nothing before it draws)."""
    st, key = state.clone(), torch.empty(1, device="cuda", dtype=torch.int64)
    m._lib.load().cvb_rng_next(st.data_ptr(), key.data_ptr(), torch.cuda.current_stream().cuda_stream)
    return _draws(m.ops, key, B, H, W)[1]


@pytest.mark.parametrize("kind", ["efficientnet", "mobilevit"])
def test_dropin_model_with_reference_loss(m, kind):
    """Plain loss.backward() through the drop-in model with the reference's NeuralAugmentation loss restated in torch on
    out["augmented_tensor"]: the augmentor's gradients equal the oracle augmentor's on the same draws and the same upstream gradient."""
    model = _effnet(m) if kind == "efficientnet" else _mit(m)
    B, H, W = 4, 64, 64
    x = _image(B, H, W, 11)
    y = torch.tensor([1, 2, 3, 4], device="cuda")
    m.ops.rng_seed(17, device="cuda")
    state = m.ops._RNG[torch.device("cuda", torch.cuda.current_device())].clone()
    out = model(x)
    assert set(out) == {"augmented_tensor", "logits"}
    x_aug = out["augmented_tensor"]
    x_aug.retain_grad()
    t = R.psnr_to_mse(30.0)
    loss = F.cross_entropy(out["logits"].float(), y, label_smoothing=0.1) + R.na_loss(x_aug, x, t)
    loss.backward()
    draws = _replay_draws(m, state, B, H, W)
    aug = model.neural_augmentor
    raw = {n: tuple(p.detach().clone().requires_grad_(True) for p in (getattr(aug, n)._low, getattr(aug, n)._high)) for n in R.NAMES}
    ref_aug = R.augment(x, raw, draws)
    torch.testing.assert_close(x_aug.detach(), ref_aug.detach(), atol=2e-5, rtol=1e-4)
    # the upstream gradient reaching x_aug is the stem's input gradient plus the loss term; push it through the oracle
    ref = torch.autograd.grad(ref_aug, [p for n in R.NAMES for p in raw[n]], grad_outputs=x_aug.grad)
    ours = [p.grad for p in aug.raw_parameters()]
    for i, (a, b) in enumerate(zip(ours, ref)):
        torch.testing.assert_close(a, b, atol=1e-3 * max(1.0, float(b.abs())), rtol=2e-3, msg=lambda msg, i=i: f"param {i}: {msg}")
    model.eval()
    out = model(x)
    assert out["augmented_tensor"] is None and out["logits"].shape == (B, 10)


def rel_l2(a, b):
    a, b = a.detach().float().flatten(), b.detach().float().flatten()
    return float((a - b).norm() / (b.norm() + 1e-20))


def cosine(a, b):
    a, b = a.detach().float().flatten(), b.detach().float().flatten()
    return float(torch.dot(a, b) / (a.norm() * b.norm() + 1e-20))


def _model_case(m, kind):
    """(drop-in model, oracle parameter shapes, oracle forward) of one conv-stem classifier with the augmentor, 10 classes, dropouts 0."""
    import efficientnet_ref as E
    from oracle import cvnets_oracle as O
    from ml_cvnets_b200.models_effnet import default_effnet_opts
    from ml_cvnets_b200.models_mit import default_mit_opts
    if kind == "efficientnet":
        return (m.EfficientNet(default_effnet_opts("b0", n_classes=10, **AUG)), E.efficientnet_shapes("b0", n_classes=10),
                lambda P, x: E.efficientnet_forward(P, x, mode="b0"))
    if kind == "mobilevit":
        opts = default_mit_opts("xx_small", n_classes=10, **{"model.classification.classifier_dropout": 0.0, "model.classification.mit.dropout": 0.0,
                                                               "model.classification.mit.attn_dropout": 0.0}, **AUG)
        return m.MobileViT(opts), O.mobilevit_v1_shapes("xx_small", n_classes=10), lambda P, x: O.mobilevit_v1_forward(P, x, mode="xx_small")
    return (m.MobileViTv2(m.default_opts(0.5, n_classes=10, **AUG)), O.mobilevit_v2_shapes(0.5, n_classes=10),
            lambda P, x: O.mobilevit_v2_forward(P, x, width_multiplier=0.5))


@pytest.mark.parametrize("kind,mix", [("efficientnet", "mixup"), ("efficientnet", "cutmix"), ("mobilevit", "mixup"), ("mobilevit_v2", "mixup")])
def test_trainstep_step_against_oracle(m, kind, mix):
    """One TrainStep step (SGD, lr 0 so the gradients stay readable) with RangeAugment, batch mixing and the NA loss, against the fp32 oracle on the
    step's own draws: augmented_tensor, logits, CE, L_na, the image gradient the stem hands the augmentor, the six augmentor gradients and the
    whole gradient.  Fixed bounds or 1.15x the error of the same oracle under torch bf16 autocast, whichever is larger.  MobileViTv2's stem hands
    its output to the next module pre-BatchNorm (lazy boundary); EfficientNet's and MobileViT's materialise it: both stem backward cases run."""
    from oracle import cvnets_oracle as O
    model, shapes, fwd = _model_case(m, kind)
    P = O.seeded_fill_(shapes, 61)
    P.update(R.seeded_aug_params(62))
    model.load_state_dict(P, strict=True)
    model = model.cuda().train()
    # EfficientNet at 8 x 128^2: at 4 x 64^2 its last stage's train-mode BatchNorms normalise 16 values per channel, which puts both bf16 paths
    # (ours and torch autocast) 15-20 % off fp32 in the logits and measures that amplification rather than the step
    B, H, W = (8, 128, 128) if kind == "efficientnet" else (4, 64, 64)
    x = _image(B, H, W, 21)
    y = torch.tensor([0, 3, 5, 7, 1, 9, 2, 4][:B], device="cuda")
    mixv = [1.0, 0.3, 0, 0, 0, 0] if mix == "mixup" else [2.0, 1.0 - (40 - 8) * (50 - 20) / (H * W), 8, 20, 40, 50]
    na = m.NeuralAugmentationLoss(target_value=(40, 10), curriculum_method="cosine", period=10)
    step = m.TrainStep(model, optimizer="sgd", lr=0.0, weight_decay=0.0, label_smoothing=0.1, max_norm=None, aug_loss=na)
    step.set_mix(mix, mixv[1], tuple(int(v) for v in mixv[2:]))
    step.set_epoch(4)
    got = {}

    def hook(mod, inp, out):
        got["logits"], got["x_aug"] = out["logits"].detach().float().clone(), out["augmented_tensor"].detach().clone()
        out["augmented_tensor"].register_hook(lambda g: got.__setitem__("dx", g.detach().clone()))

    handle = model.register_forward_hook(hook)
    m.ops.rng_seed(23, device="cuda")
    state = m.ops._RNG[torch.device("cuda", torch.cuda.current_device())].clone()
    scale = float(step.opt.scale[0])  # the loss scale of this step: the flat gradient holds scale * d loss / d p
    loss = step(x, y)
    torch.cuda.synchronize()
    handle.remove()
    ce, lna = step.loss_parts.tolist()
    grads = [p.grad.detach().clone() / scale for p in model.parameters()]
    draws = _replay_draws(m, state, B, H, W)
    xm = R.mixed(x, mixv)
    soft = R.mixed_targets(y, 10, mixv)
    t = float(na.table[4])

    def oracle(autocast):
        Pc = O.clone_params(P, device="cuda")
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            xa = R.augment(xm, R.raw_from(Pc), draws)
            logits = fwd(Pc, xa).float()
        ce_r = F.cross_entropy(logits, soft, label_smoothing=0.1)
        na_r = R.na_loss(xa, xm, t)
        (dx,) = torch.autograd.grad(ce_r, xa, retain_graph=True)
        (ce_r + na_r).backward()
        names = [k for k, _ in model.named_parameters()]
        return dict(x_aug=xa.detach(), logits=logits.detach(), ce=float(ce_r), na=float(na_r), dx=dx, grads=[Pc[k].grad for k in names])

    ref, auto = oracle(False), oracle(True)
    # the image the augmentor saw is the batch mixed once; the stem did not mix it again (that would change the logits far beyond bf16 error)
    torch.testing.assert_close(got["x_aug"], ref["x_aug"], atol=2e-5, rtol=1e-4)
    assert lna == pytest.approx(ref["na"], rel=1e-4, abs=1e-7)
    assert float(loss) == pytest.approx(ce + lna, rel=1e-6)
    e_log, a_log = rel_l2(got["logits"], ref["logits"]), rel_l2(auto["logits"], ref["logits"])
    e_dx, a_dx = rel_l2(got["dx"] / scale, ref["dx"]), rel_l2(auto["dx"], ref["dx"])
    ours_a, ref_a, auto_a = torch.stack(grads[:6]), torch.stack(ref["grads"][:6]), torch.stack(auto["grads"][:6])
    e_a, a_a = rel_l2(ours_a, ref_a), rel_l2(auto_a, ref_a)
    ours_g, ref_g, auto_g = (torch.cat([g.flatten() for g in gs]) for gs in (grads, ref["grads"], auto["grads"]))
    e_g, a_g = rel_l2(ours_g, ref_g), rel_l2(auto_g, ref_g)
    c_g, ac_g = cosine(ours_g, ref_g), cosine(auto_g, ref_g)
    print(f"[{kind} {mix}] ours/autocast rel-L2 vs fp32: logits {e_log:.4g}/{a_log:.4g} ce {ce:.5f}/{auto['ce']:.5f} (fp32 {ref['ce']:.5f}) "
          f"dx {e_dx:.4g}/{a_dx:.4g} aug {e_a:.4g}/{a_a:.4g} grad {e_g:.4g}/{a_g:.4g} cos {c_g:.5f}/{ac_g:.5f}")
    assert e_log <= max(8e-2, 1.15 * a_log), f"logits rel-L2 {e_log:.4g} (autocast {a_log:.4g})"
    if mix == "mixup":
        with torch.no_grad():
            twice = fwd(O.clone_params(P, requires_grad=False, device="cuda"), R.mixed(ref["x_aug"], mixv))
        assert e_log < 0.5 * rel_l2(twice, ref["logits"]), "the logits look like those of an image mixed twice"
    assert abs(ce - ref["ce"]) <= max(2e-2 * abs(ref["ce"]), 1.15 * abs(auto["ce"] - ref["ce"])), (ce, ref["ce"], auto["ce"])
    assert e_dx <= max(0.1, 1.15 * a_dx), f"stem input gradient rel-L2 {e_dx:.4g} (autocast {a_dx:.4g})"
    assert e_a <= max(5e-2, 1.15 * a_a), f"augmentor gradients {ours_a.tolist()} vs {ref_a.tolist()} (autocast {auto_a.tolist()})"
    assert e_g <= max(0.2, 1.15 * a_g), f"whole-gradient rel-L2 {e_g:.4g} (autocast {a_g:.4g})"
    assert 1 - c_g <= max(0.02, 1.15 * (1 - ac_g)), f"whole-gradient cosine {c_g:.5f} (autocast {ac_g:.5f})"


@pytest.mark.parametrize("optimizer", ["sgd", "adamw"])
def test_flat_optimizers_decay_sampler_parameters(m, optimizer):
    """The reference's no_decay_bn_filter_bias exempts len(shape) == 1 only (cvnets/misc/common.py:122-176): the 0-dim sampler parameters get the
    weight decay in the flat optimizers' per-element table, the BatchNorm parameters do not.  A step without aug_loss still trains (the NA
    output simply has no gradient); aug_loss with a model that has no augmentor is an error."""
    model = _effnet(m)
    step = m.TrainStep(model, optimizer=optimizer, lr=0.01, weight_decay=4e-5, label_smoothing=0.1)
    for p in model.neural_augmentor.parameters():
        o, _ = step.ws.offsets[id(p)]
        assert float(step.opt.wd[o]) == pytest.approx(4e-5)
    o, k = step.ws.offsets[id(model.conv_1.block.norm.weight)]
    assert float(step.opt.wd[o:o + k].abs().max()) == 0.0
    x, y = _image(4, 64, 64, 3), torch.tensor([1, 2, 3, 4], device="cuda")
    assert math.isfinite(float(step(x, y)))
    for p in model.neural_augmentor.parameters():
        assert torch.isfinite(p.grad).all()
    from ml_cvnets_b200.models_effnet import default_effnet_opts
    plain = m.EfficientNet(default_effnet_opts("b0", n_classes=10)).cuda().train()
    with pytest.raises(ValueError, match="augmentor"):
        m.TrainStep(plain, optimizer="sgd", aug_loss=m.NeuralAugmentationLoss(target_value=(40, 10), period=10))(x, y)


def _run_steps(m, n_eager, n_replay, x, y):
    model = _effnet(m, seed=3)
    m.ops.rng_seed(31, device="cuda")
    na = m.NeuralAugmentationLoss(target_value=(40, 10), period=20)
    step = m.TrainStep(model, optimizer="sgd", lr=0.05, weight_decay=4e-5, label_smoothing=0.1, aug_loss=na)
    step.set_mix("cutmix", 0.75, (8, 4, 40, 36))
    for e in range(n_eager):
        step.set_epoch(e)
        step(x, y)
    if n_replay:
        step.capture(x, y, warmup=n_eager)
        for e in range(n_replay):
            step.set_epoch(n_eager + e)
            step(x, y)
    torch.cuda.synchronize()
    return torch.cat([p.detach().flatten() for p in model.parameters()]), step.loss_parts.clone()


def test_reproducible_steps(m):
    """Three SGD steps with RangeAugment and cutmix end in the same bits eager, eager again, and replayed from a CUDA graph.  At 16 x 96 x 96
    each per-plane reduction CTA loops over 36 chunks of its plane."""
    B, H, W = 16, 96, 96
    x = _image(B, H, W, 41)
    y = torch.arange(B, device="cuda") % 10
    a, la = _run_steps(m, 6, 0, x, y)
    b, lb = _run_steps(m, 6, 0, x, y)
    c, lc = _run_steps(m, 3, 3, x, y)
    assert torch.equal(a, b) and torch.equal(la, lb)
    assert torch.equal(a, c) and torch.equal(la, lc)

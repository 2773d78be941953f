"""MobileViT-v1 at the variable-batch sampler's crops (-m gpu): small-head attention past 256 tokens, bilinear unfold / fold of maps that are
not multiples of the patch, and the models end to end at every (crop, batch) pair of the recipes.

* mha forward / backward at head dims 16 - 60 and S = 257 / 324 / 400 and each head dim's longest sequence (the mma.sync kernels' shared
  memory): against fp32 torch, twice with equal bits, at grids of >= 3 CTAs per SM, writes checked with guard bands; one past each limit the
  call returns its error.
* patch_permute in all four directions on 5x5, 7x7, 9x9 and 5x7 maps: against fp64 F.interpolate plus the reference's reshapes (and its
  autograd for the transposes), the adjoint identity, and the permutation's bits at multiples of the patch.
* XXS / XS / S against the real reference's fixtures at 160 - 320 px; TrainStep captured over the recipe's pairs at the recipe's batches,
  replays bitwise equal to eager steps; RangeAugment with gradient accumulation; EvalStep at the odd crops; S refuses the 192 pair."""
import os
import random
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_sample import at_sample  # noqa: E402
from mit_multiscale_ref import FIXTURES, PATCH, RECIPE_PAIRS, S_PAIRS, fixture_name, fold, mobilevit_v1_forward, unfold  # noqa: E402
from oracle import cvnets_oracle as O  # noqa: E402
from test_kernels_gpu import close  # noqa: E402
from write_guard import Guarded  # noqa: E402

pytestmark = pytest.mark.gpu

BF, F32 = torch.bfloat16, torch.float32
HDS = (16, 20, 24, 30, 36, 48, 60)
LN2 = 0.6931471805599453


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as m
    return m


@pytest.fixture(scope="module")
def lib(pkg):
    return pkg._lib.load()


def S():
    return torch.cuda.current_stream().cuda_stream


def _limit(hd, backward=True):
    from ml_cvnets_b200 import ops
    return ops.mha_max_seq(hd, backward)


def _mha_cases():
    out = []
    for hd in HDS:
        smax = _limit(hd)
        out += [(hd, s) for s in sorted({257, 324, 400, smax}) if s <= smax]
    return out


# ------------------------------------------------------------------------------------------------------------ attention
def _mha_ref32(qkv, dO, n, S_, H, hd, scale):
    """fp32 softmax attention of the first n sequences: O, LSE (base 2), dQKV"""
    x = qkv[:n * S_].float().view(n, S_, 3, H, hd).permute(2, 0, 3, 1, 4).requires_grad_(True)
    s = (x[0] @ x[1].transpose(-1, -2)) * scale
    lse = torch.logsumexp(s, -1)
    o = torch.softmax(s, -1) @ x[2]
    o2 = o.transpose(1, 2).reshape(n * S_, H * hd)
    o2.backward(dO[:n * S_].float())
    dqkv = x.grad.permute(1, 3, 0, 2, 4).reshape(n * S_, 3 * H * hd)
    return o2.detach(), (lse / LN2).detach(), dqkv


@pytest.mark.parametrize("hd,S_", _mha_cases())
def test_mha_long_small_heads(lib, hd, S_):
    H = 4
    B = -(-3 * torch.cuda.get_device_properties(0).multi_processor_count // H)  # >= 3 CTAs per SM
    C = H * hd
    g = torch.Generator(device="cuda").manual_seed(hd * 1000 + S_)
    qkv = torch.randn(B * S_, 3 * C, device="cuda", generator=g).to(BF)
    dO = torch.randn(B * S_, C, device="cuda", generator=g).to(BF)
    scale = hd ** -0.5
    runs = []
    for _ in range(2):
        O_ = Guarded((B * S_, C), BF, ld=C + 8)
        LSE = Guarded((B * H * S_,), F32)
        DQ = Guarded((B * S_, 3 * C), BF, ld=3 * C + 16)
        lib.cvb_mha_fwd(qkv.data_ptr(), qkv.stride(0), B, S_, H, hd, scale, None, None, O_.ptr, O_.ld, LSE.ptr, S())
        dOp = torch.zeros(B * S_, O_.ld, device="cuda", dtype=BF)  # the backward reads O and dO at one pitch
        dOp[:, :C] = dO
        lib.cvb_mha_bwd(qkv.data_ptr(), qkv.stride(0), O_.ptr, dOp.data_ptr(), O_.ld, LSE.ptr, B, S_, H, hd, scale, None, None, DQ.ptr, DQ.ld, S())
        torch.cuda.synchronize()
        runs.append((O_.check("mha O"), LSE.check("mha LSE"), DQ.check("mha dQKV")))
    for name, a, b in zip(("O", "LSE", "dQKV"), runs[0], runs[1]):
        assert torch.equal(a, b), f"{name} differs between two runs"
    o, lse, dq = runs[0]
    n = max(1, min(B, (1 << 26) // (H * S_ * S_)))
    ro, rl, rd = _mha_ref32(qkv, dO, n, S_, H, hd, scale)
    close(o[:n * S_], ro, what="mha O")
    lse = lse.view(B, H, S_)[:n]
    assert float((lse - rl).abs().max()) <= 1e-4 * float(rl.abs().max()) + 1e-4
    close(dq[:n * S_], rd, rtol=3e-2, atol=2e-2 * float(rd.abs().max()) + 1e-6, what="mha dQKV")


@pytest.mark.parametrize("hd", HDS)
def test_mha_refuses_past_the_limit(pkg, lib, hd):
    """one token past the shared-memory limit the call returns its error (no launch); the backward's limit is the lower one"""
    from ml_cvnets_b200 import ops
    for backward in (False, True):
        smax = _limit(hd, backward)
        S_, H = smax + 1, 4  # 4 heads: leading dimensions that are multiples of 8 at every head dim
        qkv = torch.zeros(S_, 3 * H * hd, device="cuda", dtype=BF)
        O_, LSE = torch.zeros(S_, H * hd, device="cuda", dtype=BF), torch.zeros(1, H, S_, device="cuda")
        if not backward:
            with pytest.raises(pkg._lib.CvbError, match=f"too long for head_dim {hd}.*S <= {smax} in the forward"):
                ops.mha_fwd(qkv, 1, S_, H, hd, 1.0)
        else:
            with pytest.raises(pkg._lib.CvbError, match=f"too long for head_dim {hd}.*S <= {smax} in the backward"):
                ops.mha_bwd(qkv, O_, O_, LSE, 1, S_, H, hd, 1.0)
    enc = pkg.TransformerEncoder(pkg.default_mit_opts("xx_small"), 4 * hd, 8 * hd, num_heads=4).cuda() if (4 * hd) % 8 == 0 else None
    if enc is not None:
        with pytest.raises(NotImplementedError, match=f"S <= {_limit(hd)}"):
            enc(torch.randn(1, _limit(hd) + 1, 4 * hd, device="cuda"))


# ------------------------------------------------------------------------------------------------------------ unfold / fold
MAPS = ((5, 5), (7, 7), (9, 9), (5, 7))
CS = (96, 144, 240)


def _grid(H, W):
    return -(-H // PATCH) * PATCH, -(-W // PATCH) * PATCH


def _run(lib, X, B, H, W, C, direction):
    """one cvb_patch_permute call into a guard-banded output"""
    Hn, Wn = _grid(H, W)
    rows = B * (Hn * Wn if direction in (0, 3) else H * W)
    out = Guarded((rows, C), BF)
    lib.cvb_patch_permute(X.data_ptr(), out.ptr, B, H, W, C, PATCH, PATCH, direction, S())
    torch.cuda.synchronize()
    return out.check(f"patch_permute direction {direction}")


def _map_rows(x4):   # [B, C, H, W] -> [B*H*W, C]
    return x4.permute(0, 2, 3, 1).reshape(-1, x4.shape[1])


def _rows_map(r, B, H, W):
    return r.view(B, H, W, -1).permute(0, 3, 1, 2)


@pytest.mark.parametrize("C", CS)
@pytest.mark.parametrize("H,W", MAPS)
def test_patch_permute_resized(lib, H, W, C):
    B = 3
    Hn, Wn = _grid(H, W)
    N = (Hn // PATCH) * (Wn // PATCH)
    g = torch.Generator(device="cuda").manual_seed(H * 100 + W + C)
    xm = torch.randn(B * H * W, C, device="cuda", generator=g).to(BF)        # a feature map
    xt = torch.randn(B * PATCH * PATCH * N, C, device="cuda", generator=g).to(BF)  # tokens
    outs = {}
    for d, X in ((0, xm), (1, xt), (2, xt), (3, xm)):
        a, b = _run(lib, X, B, H, W, C, d), _run(lib, X, B, H, W, C, d)
        assert torch.equal(a, b), f"direction {d} differs between two runs"
        outs[d] = a
    # fp64 reference: the reference's unfolding / folding with F.interpolate, and its autograd for the transposes
    x4 = _rows_map(xm.double(), B, H, W).requires_grad_(True)
    t, info = unfold(x4)
    assert info[4:] == (Hn, Wn)
    close(outs[0], t.reshape(-1, C).detach(), what="unfold")
    t.backward(xt.double().view(t.shape))
    close(outs[2], _map_rows(x4.grad), what="unfold transpose")
    tt = xt.double().view(B * PATCH * PATCH, N, C).requires_grad_(True)
    fm = fold(tt, (B, C, H, W, Hn, Wn))
    close(outs[1], _map_rows(fm.detach()), what="fold")
    fm.backward(_rows_map(xm.double(), B, H, W))
    close(outs[3], tt.grad.reshape(-1, C), what="fold transpose")
    # <A x, y> = <x, A^T y> on positive inputs (no cancellation)
    pm, pt = xm.float().abs().to(BF), xt.float().abs().to(BF)
    for fwd, adj, x, y in ((0, 2, pm, pt), (1, 3, pt, pm)):
        ax, aty = _run(lib, x, B, H, W, C, fwd), _run(lib, y, B, H, W, C, adj)
        lhs, rhs = float((ax.double() * y.double()).sum()), float((x.double() * aty.double()).sum())
        assert abs(lhs - rhs) <= 5e-3 * abs(lhs), (fwd, adj, lhs, rhs)


@pytest.mark.parametrize("H,W", [(6, 6), (8, 10)])
def test_patch_permute_transposes_at_multiples(lib, H, W):
    """at multiples of the patch the transposes are the permutations, bit for bit: UNFOLD_T = FOLD, FOLD_T = UNFOLD"""
    B, C = 2, 144
    g = torch.Generator(device="cuda").manual_seed(H * W)
    xm = torch.randn(B * H * W, C, device="cuda", generator=g).to(BF)
    xt = torch.randn(B * H * W, C, device="cuda", generator=g).to(BF)
    assert torch.equal(_run(lib, xt, B, H, W, C, 2), _run(lib, xt, B, H, W, C, 1))
    assert torch.equal(_run(lib, xm, B, H, W, C, 3), _run(lib, xm, B, H, W, C, 0))
    assert torch.equal(_run(lib, _run(lib, xm, B, H, W, C, 0), B, H, W, C, 1), xm)


# ------------------------------------------------------------------------------------------------------------ models
def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / b.norm())


@pytest.mark.parametrize("mode,crop", FIXTURES)
def test_model_against_reference_fixture(pkg, golden_dir, mode, crop):
    """eval logits at 1 x crop^2 and a train step at batch 2 against the real reference's fp32 record, bounded by the resize-aware oracle
    under bf16 autocast (the bounds of test_mobilevit_v1_modes_gpu.py)"""
    fx = torch.load(os.path.join(golden_dir, fixture_name(mode, crop)), weights_only=False)
    opts = pkg.default_mit_opts(mode, **{"model.classification.mit.dropout": 0.0, "model.classification.classifier_dropout": 0.0})
    model = pkg.MobileViT(opts)
    model.load_state_dict(O.seeded_fill_(O.mobilevit_v1_shapes(mode), fx["seed"]), strict=True)
    model = model.cuda().eval()
    x1 = O.seeded_input((1, 3, crop, crop), fx["eval_x_seed"]).cuda()
    with torch.no_grad():
        ev = model(x1)
        Pa = O.clone_params(O.seeded_fill_(O.mobilevit_v1_shapes(mode), fx["seed"]), requires_grad=False, device="cuda")
        with torch.autocast("cuda", dtype=torch.bfloat16):
            eva = mobilevit_v1_forward(Pa, x1, mode=mode, training=False)
    e, ea = rel_l2(ev, fx["eval_logits"]), rel_l2(eva, fx["eval_logits"])
    print(f"[{mode} @ {crop}] eval logits rel-L2 vs the reference: ours {e:.4g}, torch-autocast {ea:.4g}")
    assert e <= max(3e-2, 1.5 * ea)
    model.train()
    x = O.seeded_input((fx["batch"], 3, crop, crop), fx["x_seed"]).cuda()
    logits = model(x)
    loss = F.cross_entropy(logits.float(), fx["labels"].cuda(), label_smoothing=0.1)
    loss.backward()
    Pt = O.clone_params(O.seeded_fill_(O.mobilevit_v1_shapes(mode), fx["seed"]), device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        lt = mobilevit_v1_forward(Pt, x, mode=mode, training=True)
        F.cross_entropy(lt, fx["labels"].cuda(), label_smoothing=0.1).backward()
    et, eta = rel_l2(logits, fx["logits"]), rel_l2(lt, fx["logits"])
    print(f"[{mode} @ {crop}] train logits rel-L2: ours {et:.4g}, torch-autocast {eta:.4g}; loss {float(loss):.5f} vs {float(fx['loss']):.5f}")
    assert et <= max(5e-2, 1.5 * eta)
    named = dict(model.named_parameters())
    total = sum(n * n for n in fx["grad_norms"].values()) ** 0.5
    bad = []
    for k, g in fx["grads"].items():
        if fx["grad_norms"][k] < 1e-3 * total:
            continue
        eo, eau = rel_l2(*at_sample(named[k].grad, g)), rel_l2(*at_sample(Pt[k].grad, g))
        if eo > max(0.1, 2.0 * eau):
            bad.append((k, eo, eau))
    assert not bad, bad[:8]


def _batch(B, crop, seed, n_classes=1000):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return torch.randn(B, 3, crop, crop, device="cuda", generator=g), torch.randint(0, n_classes, (B,), device="cuda", generator=g)


def _mit(pkg, mode, **extra):
    torch.manual_seed(0)
    return pkg.MobileViT(pkg.default_mit_opts(mode, **extra)).cuda().train()


def _adamw(pkg, model, **kw):
    return pkg.TrainStep(model, lr=2e-3, weight_decay=0.01, max_norm=None, label_smoothing=0.1, ema_momentum=0.0005, **kw)


def _captured_vs_eager(pkg, build, pairs, seq_len, seed, mixes=False, n_classes=1000):
    """one TrainStep captured over ``pairs`` and replayed over a random sequence of them, a second one running the same sequence eagerly
    (capture's warm-up passes included): losses, parameters and EMA must agree bit for bit"""
    from ml_cvnets_b200 import ops
    examples = [_batch(B, c, 100 + c, n_classes) for c, B in pairs]
    rnd = random.Random(seed)
    order = [rnd.randrange(len(pairs)) for _ in range(seq_len)]
    seq = [_batch(pairs[i][1], pairs[i][0], 1000 + k, n_classes) for k, i in enumerate(order)]
    torch.manual_seed(seed)
    sampler = pkg.engine.MixingSampler()
    draws = [sampler.sample(pairs[i][0], pairs[i][0]) if mixes else None for i in order]
    runs = []
    for captured in (True, False):
        model, ts = build()
        ops.rng_seed(7)
        if captured:
            ts.capture_shapes(examples)
        else:
            for _ in range(3):
                for x, y in examples:
                    ts.step(x, y)
        losses = []
        for (x, y), mix in zip(seq, draws):
            if mix is not None:
                ts.set_mix(*mix)
            losses.append(ts.step(x, y).clone())
        torch.cuda.synchronize()
        runs.append((torch.stack(losses), ts.opt.flat_p.clone(), ts.opt.ema.clone()))
        del ts, model
        torch.cuda.empty_cache()
    print("order", [pairs[i][0] for i in order], "losses", runs[0][0].tolist())
    assert torch.isfinite(runs[0][0]).all()
    for name, a, b in zip(("losses", "params", "ema"), runs[0], runs[1]):
        assert torch.equal(a, b), (name, float((a.float() - b.float()).abs().max()))


def test_xxs_captured_over_the_recipe_pairs(pkg):
    """XXS at all five pairs (160 x 327 ... 320 x 81), the recipe's dropouts, mixup / cutmix drawn by MixingSampler"""
    def build():
        model = _mit(pkg, "xx_small")
        return model, _adamw(pkg, model)
    _captured_vs_eager(pkg, build, RECIPE_PAIRS, 10, 3, mixes=True)


def test_small_captured_over_its_pairs(pkg):
    """S at the four pairs it trains on (the 192 pair refuses, test_small_refuses_the_192_pair)"""
    def build():
        model = _mit(pkg, "small")
        return model, _adamw(pkg, model)
    _captured_vs_eager(pkg, build, S_PAIRS, 6, 4)


AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True}


def test_range_augment_with_accumulation_at_odd_crops(pkg):
    """XXS with RangeAugment (aug_loss) and accum_freq 2 at 160 / 288 px (the resized maps): captured replays equal eager steps bitwise"""
    def build():
        model = _mit(pkg, "xx_small", n_classes=10, **AUG)
        na = pkg.NeuralAugmentationLoss(target_value=(40, 10), curriculum_method="cosine", period=10)
        return model, _adamw(pkg, model, aug_loss=na, accum_freq=2)
    _captured_vs_eager(pkg, build, [(160, 12), (288, 4)], 6, 5, n_classes=10)


def test_eval_step_at_odd_crops(pkg):
    """EvalStep captured at 160 / 288 / 320 counts what the eager pass counts"""
    model = _mit(pkg, "xx_small").eval()
    res = {}
    for captured in (True, False):
        ev = pkg.EvalStep(model)
        for crop in (160, 288, 320):
            if captured:
                ev.capture(batch=16, crop=(crop, crop))
            for k in range(2):
                ev.update(*_batch(16 - 5 * k, crop, 50 + crop + k))
        res[captured] = ev.compute()
    print(res)
    assert res[True] == res[False]


def test_small_refuses_the_192_pair(pkg):
    """MobileViT-S over the full table: the 192 pair's 144 tokens of width 144 raise NotImplementedError during capture's warm-up, before any
    graph is captured"""
    model = _mit(pkg, "small")
    ts = _adamw(pkg, model)
    with pytest.raises(NotImplementedError, match="S == C"):
        ts.capture_shapes([_batch(B, c, 100 + c) for c, B in RECIPE_PAIRS])
    assert not ts.captured_shapes

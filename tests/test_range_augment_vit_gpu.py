"""RangeAugment on the ViT / CLIP recipes on the GPU: the conv stem's image gradient (cvb_patch_stem_dgrad) against torch, one TrainStep step of
ViT-tiny and of a small CLIP with the augmentor against the fp32 oracle on the step's own draws, ViT-B/16 at the recipes' crops, a captured CLIP
step with fresh draws, and the unchanged outputs of models without the augmentor."""
import math

import pytest
import torch
import torch.nn.functional as F

import range_augment_ref as R
from test_range_augment_gpu import AUG, _image, _replay_draws, cosine, rel_l2

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def m():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as pkg
    return pkg


def _stem_case(C0, B, H, W, seed):
    Ho, Wo = H // 4, W // 4
    g = torch.Generator("cuda").manual_seed(seed)
    dz = torch.randn(B * Ho * Wo, C0, device="cuda", generator=g).to(torch.bfloat16)
    y = torch.randn(B * Ho * Wo, C0, device="cuda", generator=g).to(torch.bfloat16)
    coef = torch.randn(3, C0, device="cuda", generator=g) * 0.5
    w = torch.randn(C0, 3, 4, 4, device="cuda", generator=g) * 0.2
    Wp = w.permute(0, 2, 3, 1).reshape(C0, 48).to(torch.bfloat16).contiguous()  # patch columns (u, v, ci), as cvb_im2col orders them
    return dz, y, coef, w, Wp


SHAPES = [(1, 16, 16), (3, 32, 48), (2, 160, 256), (8, 64, 128), (64, 320, 320), (256, 224, 224)]


@pytest.mark.parametrize("C0", [32, 48, 96, 192, 320])
@pytest.mark.parametrize("B,H,W", SHAPES)
def test_patch_stem_input_gradient(m, C0, B, H, W):
    dz, y, coef, w, Wp = _stem_case(C0, B, H, W, C0 + B + H)
    dX = m.ops.patch_stem_dgrad(dz, y, coef, Wp, B, H // 4, W // 4)
    assert dX.dtype == torch.float32 and dX.shape == (B, 3, H, W) and dX.is_contiguous()
    dy = (coef[0] * dz.float() + coef[1] * y.float() + coef[2]).to(torch.bfloat16).float()
    dy4 = dy.view(B, H // 4, W // 4, C0).permute(0, 3, 1, 2)
    w4 = Wp.float().view(C0, 4, 4, 3).permute(0, 3, 1, 2)
    prev = torch.backends.cudnn.allow_tf32
    torch.backends.cudnn.allow_tf32 = False
    try:
        ref = torch.nn.grad.conv2d_input((B, 3, H, W), w4, dy4, stride=4, padding=1)
    finally:
        torch.backends.cudnn.allow_tf32 = prev
    assert rel_l2(dX, ref) <= 4e-3, rel_l2(dX, ref)
    assert torch.count_nonzero(dX[:, :, -1, :]) == 0 and torch.count_nonzero(dX[:, :, :, -1]) == 0
    assert torch.isfinite(dX).all()


@pytest.mark.parametrize("C0", [192, 320])
def test_patch_stem_input_gradient_is_bitwise_reproducible(m, C0):
    """At 64 x 224^2 each warp of the persistent grid handles about nine patch tiles, so the result must not depend on which warp took which."""
    B, H, W = 64, 224, 224
    dz, y, coef, _, Wp = _stem_case(C0, B, H, W, 5)
    a = m.ops.patch_stem_dgrad(dz, y, coef, Wp, B, H // 4, W // 4)
    b = m.ops.patch_stem_dgrad(dz, y, coef, Wp, B, H // 4, W // 4)
    assert torch.equal(a, b)


def test_patch_stem_rejects_bad_widths(m):
    dz, y, coef, _, Wp = _stem_case(48, 1, 16, 16, 1)
    with pytest.raises(RuntimeError, match="multiple of 16"):  # the library's CvbError
        m.ops.patch_stem_dgrad(dz[:, :40].contiguous(), y[:, :40].contiguous(), coef[:, :40].contiguous(), Wp[:40], 1, 4, 4)


def _vit(m, mode="tiny", n_classes=10, aug=True):
    opts = m.default_vit_opts(mode, n_classes=n_classes, **(AUG if aug else {}))
    model = m.VisionTransformer(opts)
    model.emb_dropout.p = 0.0  # the oracle has no positional-embedding dropout ('tiny' trains with 0.1)
    return model


def _clip_opts(m, aug=True):
    return m.default_clip_opts("tiny", projection_dim=64, text_dim=128, text_layers=2, text_heads=4, vocab_size=1000, context_length=16,
                               **(AUG if aug else {}))


def _tokens(B, L=16, seed=0):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(1, 998, (B, L), generator=g)
    tok[torch.arange(B), torch.randint(2, L, (B,), generator=g)] = 999
    return tok.cuda()


def _clip_forward_loss(m):
    def fl(model, im, tok, cfg):
        img, txt, scale, x_aug = model(im, tok)
        return m.clip_contrastive_loss(img, txt, scale, _cfg=cfg), x_aug
    return fl


@pytest.mark.parametrize("kind,mix", [("vit", "mixup"), ("vit", "cutmix"), ("clip", "mixup"), ("clip", "cutmix")])
def test_trainstep_step_against_oracle(m, kind, mix, monkeypatch):
    """One TrainStep step (SGD, lr 0) with RangeAugment, batch mixing and the NA loss against the fp32 oracle on the step's own draws: augmented
    image, logits / features, both loss terms, the stem's image gradient, the six sampler gradients and the whole gradient.  Fixed bounds or
    1.15x the error of the same oracle under torch bf16 autocast, whichever is larger.  The stem's image gradient must come from
    cvb_patch_stem_dgrad, once per step."""
    calls = []
    real = m.ops.patch_stem_dgrad
    monkeypatch.setattr(m.ops, "patch_stem_dgrad", lambda *a, **k: calls.append(1) or real(*a, **k))
    from oracle import cvnets_oracle as O
    from vit_multiscale_ref import vit_forward_any_size
    B = 4 if kind == "vit" else 8  # the contrastive loss takes batches of multiples of 8
    if kind == "vit":
        model = _vit(m)
        P = O.seeded_fill_(O.vit_shapes("tiny", n_classes=10), 71)
        H = W = 64
    else:
        model = m.CLIP(_clip_opts(m))
        model.image_encoder.emb_dropout.p = 0.0
        P = O.seeded_fill_(O.clip_shapes("tiny", proj=64, text_dim=128, text_layers=2, vocab=1000, ctx=16), 71)
        H = W = 224  # the oracle's CLIP reads the 196-entry positional table as is
    pre = "" if kind == "vit" else "image_encoder."
    P.update({pre + k: v for k, v in R.seeded_aug_params(72).items()})
    model.load_state_dict(P, strict=True)
    model = model.cuda().train()
    x = _image(B, H, W, 31)
    y = torch.tensor([0, 3, 5, 7], device="cuda") if kind == "vit" else _tokens(B)
    mixv = [1.0, 0.3, 0, 0, 0, 0] if mix == "mixup" else [2.0, 1.0 - (40 - 8) * (50 - 20) / (H * W), 8, 20, 40, 50]
    na = m.NeuralAugmentationLoss(target_value=(40, 20), curriculum_method="cosine", period=10)
    kw = {} if kind == "vit" else {"forward_loss": _clip_forward_loss(m)}
    step = m.TrainStep(model, optimizer="sgd", lr=0.0, weight_decay=0.0, label_smoothing=0.1, max_norm=None, aug_loss=na, **kw)
    step.set_mix(mix, mixv[1], tuple(int(v) for v in mixv[2:]))
    step.set_epoch(4)
    got = {}
    enc = model if kind == "vit" else model.image_encoder

    def hook(mod, inp, out):
        got["out"], got["x_aug"] = out["logits"].detach().float().clone(), out["augmented_tensor"].detach().clone()
        out["augmented_tensor"].register_hook(lambda g: got.__setitem__("dx", g.detach().clone()))

    handle = enc.register_forward_hook(hook)
    m.ops.rng_seed(29, device="cuda")
    state = m.ops._RNG[torch.device("cuda", torch.cuda.current_device())].clone()
    scale = float(step.opt.scale[0])
    loss = step(x, y)
    torch.cuda.synchronize()
    handle.remove()
    assert len(calls) == 1, "the stem's image gradient did not go through cvb_patch_stem_dgrad"
    main, lna = step.loss_parts.tolist()
    names = [k for k, _ in model.named_parameters()]
    grads = [p.grad.detach().clone() / scale for p in model.parameters()]
    draws = _replay_draws(m, state, B, H, W)
    xm = R.mixed(x, mixv)
    t = float(na.table[4])

    def oracle(autocast):
        Pc = O.clone_params(P, device="cuda")
        raw = R.raw_from({k[len(pre):]: v for k, v in Pc.items() if k.startswith(pre + "neural_augmentor.")})
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            xa = R.augment(xm, raw, draws)
            if kind == "vit":
                out = vit_forward_any_size(Pc, xa, mode="tiny").float()
            else:
                img, txt = O.clip_forward(Pc, xa, y, vit_mode="tiny", text_layers=2, text_heads=4)
                out = img.float()
        if kind == "vit":
            main_r = F.cross_entropy(out, R.mixed_targets(y, 10, mixv), label_smoothing=0.1)
        else:
            main_r = O.clip_loss(img.float(), txt.float(), Pc["logit_scale"])
        na_r = R.na_loss(xa, xm, t)
        (dx,) = torch.autograd.grad(main_r, xa, retain_graph=True)
        (main_r + na_r).backward()
        return dict(x_aug=xa.detach(), out=out.detach(), main=float(main_r), na=float(na_r), dx=dx, grads=[Pc[k].grad for k in names])

    ref, auto = oracle(False), oracle(True)
    torch.testing.assert_close(got["x_aug"], ref["x_aug"], atol=2e-5, rtol=1e-4)
    assert lna == pytest.approx(ref["na"], rel=1e-4, abs=1e-7)
    assert float(loss) == pytest.approx(main + lna, rel=1e-6)
    e_out, a_out = rel_l2(got["out"], ref["out"]), rel_l2(auto["out"], ref["out"])
    e_dx, a_dx = rel_l2(got["dx"] / scale, ref["dx"]), rel_l2(auto["dx"], ref["dx"])
    ia = [i for i, k in enumerate(names) if "neural_augmentor." in k]
    ours_a, ref_a, auto_a = (torch.stack([gs[i] for i in ia]) for gs in (grads, ref["grads"], auto["grads"]))
    e_a, a_a = rel_l2(ours_a, ref_a), rel_l2(auto_a, ref_a)
    used = [i for i, g in enumerate(ref["grads"]) if g is not None]
    ours_g, ref_g, auto_g = (torch.cat([gs[i].flatten() for i in used]) for gs in (grads, ref["grads"], auto["grads"]))
    e_g, a_g = rel_l2(ours_g, ref_g), rel_l2(auto_g, ref_g)
    c_g, ac_g = cosine(ours_g, ref_g), cosine(auto_g, ref_g)
    print(f"[{kind} {mix}] ours/autocast rel-L2 vs fp32: out {e_out:.4g}/{a_out:.4g} loss {main:.5f}/{auto['main']:.5f} (fp32 {ref['main']:.5f}) "
          f"dx {e_dx:.4g}/{a_dx:.4g} aug {e_a:.4g}/{a_a:.4g} grad {e_g:.4g}/{a_g:.4g} cos {c_g:.5f}/{ac_g:.5f}")
    assert e_out <= max(8e-2, 1.15 * a_out), f"logits / features rel-L2 {e_out:.4g} (autocast {a_out:.4g})"
    assert abs(main - ref["main"]) <= max(2e-2 * abs(ref["main"]), 1.15 * abs(auto["main"] - ref["main"])), (main, ref["main"], auto["main"])
    assert e_dx <= max(0.1, 1.15 * a_dx), f"stem image gradient rel-L2 {e_dx:.4g} (autocast {a_dx:.4g})"
    assert e_a <= max(5e-2, 1.15 * a_a), f"sampler gradients {ours_a.tolist()} vs {ref_a.tolist()} (autocast {auto_a.tolist()})"
    assert e_g <= max(0.2, 1.15 * a_g), f"whole-gradient rel-L2 {e_g:.4g} (autocast {a_g:.4g})"
    assert 1 - c_g <= max(0.02, 1.15 * (1 - ac_g)), f"whole-gradient cosine {c_g:.5f} (autocast {ac_g:.5f})"


@pytest.mark.parametrize("H,W", [(160, 160), (320, 320), (192, 256)])
def test_vit_b16_crops(m, H, W):
    """ViT-B/16 with the augmentor, one eager step at each of the recipes' crop shapes: finite loss parts, the sampler parameters learn."""
    torch.manual_seed(0)
    model = m.VisionTransformer(m.default_vit_opts("base", n_classes=100, **AUG)).cuda().train()
    na = m.NeuralAugmentationLoss(target_value=(40, 20), curriculum_method="cosine", period=10)
    step = m.TrainStep(model, lr=1e-4, weight_decay=0.2, max_norm=1.0, label_smoothing=0.1, aug_loss=na)
    step.set_mix("mixup", 0.7)
    x = _image(8, H, W, H + W)
    step(x, torch.arange(8, device="cuda"))
    torch.cuda.synchronize()
    assert all(math.isfinite(v) for v in step.loss_parts.tolist())
    for p in model.neural_augmentor.parameters():
        assert torch.isfinite(p.grad).all() and float(p.grad.abs()) > 0


def test_captured_clip_step_draws_fresh_values(m):
    """A captured CLIP + augmentor step draws fresh augmentations at every replay and keeps its loss parts finite; the flat optimizer decays the
    sampler parameters."""
    torch.manual_seed(0)
    model = m.CLIP(_clip_opts(m)).cuda().train()
    na = m.NeuralAugmentationLoss(target_value=(40, 20), curriculum_method="cosine", period=10)
    step = m.TrainStep(model, lr=1e-4, weight_decay=0.2, max_norm=1.0, aug_loss=na, forward_loss=_clip_forward_loss(m))
    for p in model.image_encoder.neural_augmentor.parameters():  # the reference decays the 0-dim sampler parameters (parameter_list)
        o, _ = step.ws.offsets[id(p)]
        assert float(step.opt.wd[o]) == pytest.approx(0.2)
    x, tok = _image(8, 224, 224, 3), _tokens(8)
    step.capture(x, tok)
    seen = []
    for e in range(3):
        step.set_epoch(e)
        step(x, tok)
        torch.cuda.synchronize()
        seen.append(step.loss_parts.clone())
    assert all(torch.isfinite(s).all() for s in seen)
    assert not torch.equal(seen[0][1], seen[1][1]) and not torch.equal(seen[1][1], seen[2][1])


def test_forward_loss_tuple_needs_aug_loss(m):
    model = m.CLIP(_clip_opts(m)).cuda().train()
    step = m.TrainStep(model, lr=1e-4, forward_loss=_clip_forward_loss(m))
    with pytest.raises(ValueError, match="aug_loss"):
        step(_image(8, 224, 224, 1), _tokens(8))


def test_models_without_augmentor_are_unchanged(m):
    vit = _vit(m, aug=False).cuda().train()
    assert vit.neural_augmentor is None
    x = _image(2, 64, 64, 2)
    assert isinstance(vit(x), torch.Tensor)
    clip = m.CLIP(_clip_opts(m, aug=False)).cuda().train()
    out = clip(_image(2, 224, 224, 2), _tokens(2))
    assert isinstance(out, tuple) and len(out) == 3
    aug_vit = _vit(m).cuda().eval()
    out = aug_vit(x)
    assert out["augmented_tensor"] is None and out["logits"].shape == (2, 10)
    aug_clip = m.CLIP(_clip_opts(m)).cuda().eval()
    img, txt, scale, x_aug = aug_clip(_image(2, 224, 224, 2), _tokens(2))
    assert x_aug is None and img.shape == (2, 64)

"""The ViT-H/16 recipes on the GPU (-m gpu): the 1280-channel LayerNorm backward, ViT-H against the real reference at the sampler's crops,
and recomputing gradient checkpointing of the encoder stacks -- bitwise equivalence with the plain path, its memory saving, the workspace's
per-layer reporting, and a captured CLIP ViT-H + RangeAugment step."""
import math
import os
import sys
from collections import Counter

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_sample import at_sample  # noqa: E402
from vit_huge_ref import vit_huge_forward, vit_huge_shapes  # noqa: E402
from test_kernels_gpu import bf, close, close_stat, rnd  # noqa: E402
from test_modules_gpu import rel_l2  # noqa: E402
from test_range_augment_gpu import AUG, _image  # noqa: E402
from test_reproducible_gpu import ln_bwd_ctas, passes, zeros64  # noqa: E402

pytestmark = pytest.mark.gpu

STREAMING = 2  # cvb_set_mha_impl mode: the streaming kernels (deterministic backward) for every head_dim-64 shape
CKPT = "model.classification.gradient_checkpointing"


@pytest.fixture(scope="module")
def m():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as pkg
    return pkg


# ------------------------------------------------------------------------------------------------ LayerNorm backward past 1024 channels
@pytest.mark.parametrize("C", [1280, 1152])
def test_ln_bwd_wide_rows(m, C):
    """The 5-chunk cvb_ln_bwd instantiation against an fp64 restatement, with every capped CTA looping over >= 3 groups of 8 rows."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    M = 8 * (3 * 4 * sms + 5)
    passes(math.ceil(M / 8), ln_bwd_ctas(M, sms))
    X = bf(rnd(M, C, seed=1701) * 1.5 + 0.3)
    V = bf(rnd(M, C, seed=1702))
    R = bf(rnd(M, C, seed=1703))
    gamma = 1 + 0.2 * rnd(C, seed=1704)
    ln = m.ops.ln_stats(X, 1e-6)
    col, cs = zeros64(2, C), zeros64(C)
    DX = m.ops.ln_bwd(V, X, ln, gamma, col, DRES=R, col_sum=cs)
    xh = (X.double() - ln[0].double()[:, None]) * ln[1].double()[:, None]
    v = V.double()
    g = v * gamma.double()
    ref = ln[1].double()[:, None] * (g - g.mean(1, keepdim=True) - xh * (g * xh).mean(1, keepdim=True)) + R.double()
    close(DX, ref, what="ln_bwd dx")
    close_stat(col[0], v.sum(0), "dbeta", rtol=5e-3)
    close_stat(col[1], (v * xh).sum(0), "dgamma", rtol=5e-3)
    close_stat(cs, DX.double().sum(0), "col_sum", rtol=5e-3)


def test_ln_bwd_rejects_wider_rows(m):
    X = bf(rnd(16, 1288, seed=1705))
    ln = m.ops.ln_stats(X, 1e-6)
    with pytest.raises(RuntimeError, match="1288"):
        m.ops.ln_bwd(X, X, ln, torch.ones(1288, device="cuda"), zeros64(2, 1288))


def test_standalone_layer_norm_1280(m):
    """LayerNorm(1280) on [N, S, C] (ViT-H's post_transformer_norm): forward and backward against fp32 torch."""
    ln = m.LayerNorm(1280, eps=1e-6).cuda()
    with torch.no_grad():
        ln.weight.copy_(1 + 0.2 * rnd(1280, seed=1706))
        ln.bias.copy_(0.1 * rnd(1280, seed=1707))
    x = bf(rnd(3, 197, 1280, seed=1708) * 2 + 0.5)
    gy = bf(rnd(3, 197, 1280, seed=1709))
    xg = x.clone().requires_grad_(True)
    y = ln(xg)
    y.backward(gy)
    xr = x.float().requires_grad_(True)
    w, b = ln.weight.detach().clone().requires_grad_(True), ln.bias.detach().clone().requires_grad_(True)
    yr = F.layer_norm(xr, (1280,), w, b, 1e-6)
    yr.backward(gy.float())
    close(y, yr.detach(), what="LayerNorm(1280) forward")
    close(xg.grad, xr.grad, rtol=3e-2, atol=1e-2 * float(xr.grad.abs().max()), what="LayerNorm(1280) dx")
    assert rel_l2(ln.weight.grad, w.grad) <= 1e-3 and rel_l2(ln.bias.grad, b.grad) <= 1e-3


# ------------------------------------------------------------------------------------------------ ViT-H against the reference
@pytest.mark.parametrize("crop", ["128x128", "320x320"])
def test_vit_huge_against_reference(m, golden_dir, crop):
    """ViT-H/16 (32 layers, 4 checkpointed segments as the reference ran) at the sampler's smallest and largest crops against the REAL
    reference (tests/golden/make_golden_vit_huge.py): logits and loss with the bounds of test_vit_multiscale_gpu.py, gradients as below."""
    fx = torch.load(os.path.join(golden_dir, "vit_huge_fp32.pt"), weights_only=False)
    c = fx["crops"][crop]
    h, w = c["size"]
    model = m.VisionTransformer(m.default_vit_opts("huge", **{CKPT: True}))
    model.load_state_dict(O.seeded_fill_(vit_huge_shapes(), fx["seed"]), strict=True)
    model = model.cuda().train()
    x = O.seeded_input((2, 3, h, w), c["x_seed"]).cuda()
    logits = model(x)
    loss = F.cross_entropy(logits.float(), c["labels"].cuda(), label_smoothing=0.1)
    loss.backward()
    named = {k: p.grad.detach().cpu() for k, p in model.named_parameters()}
    del model
    Pa = O.clone_params(O.seeded_fill_(vit_huge_shapes(), fx["seed"]), device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        la = vit_huge_forward(Pa, x)
        F.cross_entropy(la, c["labels"].cuda(), label_smoothing=0.1).backward()
    e, ea = rel_l2(logits, c["logits"]), rel_l2(la, c["logits"])
    print(f"[vit huge {crop}] logits rel-L2 vs the reference: ours {e:.4g}, torch-autocast {ea:.4g}; loss {float(loss):.5f} vs {float(c['loss']):.5f}")
    assert e <= max(2e-2, 1.5 * ea)
    assert abs(float(loss) - float(c["loss"])) <= 5e-3 * abs(float(c["loss"]))
    # Every activation here is stored in bf16, the residual stream included, where autocast keeps an fp32 residual stream; over 32 layers the
    # ratio of the two errors grows from ~1.7 at the first layer to ~3 at the last (ViT-H, H100).  The whole sampled gradient keeps the
    # 12-layer bound; single parameters may exceed it in at most 2 % of the cases, and none goes past max(0.3, 3x autocast).
    total = sum(n * n for n in c["grad_norms"].values()) ** 0.5
    errs, cat = [], ([], [], [])
    for k, g in c["grads"].items():
        if c["grad_norms"][k] < 1e-3 * total:
            continue
        ours, ref = at_sample(named[k], g)
        auto, _ = at_sample(Pa[k].grad, g)
        errs.append((rel_l2(ours, ref), rel_l2(auto, ref), k))
        for lst, t in zip(cat, (ours, ref, auto)):
            lst.append(t.detach().float().cpu().flatten())
    errs.sort(reverse=True)
    bad = [e for e in errs if e[0] > max(6e-2, 2.0 * e[1])]
    ew, aw = rel_l2(torch.cat(cat[0]), torch.cat(cat[1])), rel_l2(torch.cat(cat[2]), torch.cat(cat[1]))
    print(f"[vit huge {crop}] all sampled gradients rel-L2 {ew:.4g} (autocast {aw:.4g}); {len(bad)} of {len(errs)} parameters over the 12-layer "
          f"bound; worst (ours, autocast, name): {errs[:6]}")
    assert ew <= max(6e-2, 2.0 * aw)
    assert len(bad) <= 0.02 * len(errs), bad
    assert all(e[0] <= max(0.3, 3.0 * e[1]) for e in errs), errs[:6]


# ------------------------------------------------------------------------------------------------ checkpointing equivalence
def _nondeterministic(name):
    """Gradients compared with a tolerance: LayerNorm gains / biases and the out_proj bias (the column sums of cvb_ln_bwd's dx), and the
    token-embedding table (cvb_embedding_bwd, fp32 atomics: test_reproducible_gpu.NONDETERMINISTIC)."""
    return (".pre_norm_mha.0." in name or ".pre_norm_ffn.0." in name or name.startswith("post_transformer_norm.")
            or "final_layer_norm." in name or name.endswith("out_proj.bias") or name == "embedding_layer.weight")


def _run(m, model, fn, ckpt, seed=77):
    for p in model.parameters():
        p.grad = None
    model.gradient_checkpointing = ckpt
    m.ops.rng_seed(seed, device="cuda")
    out = fn()
    torch.cuda.synchronize()
    return out.detach().clone(), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}


def _compare(plain, ckpt, what):
    assert torch.equal(plain[0], ckpt[0]), f"{what}: forward output differs with checkpointing"
    assert plain[1].keys() == ckpt[1].keys()
    for k, g in plain[1].items():
        if _nondeterministic(k):
            r = rel_l2(ckpt[1][k], g)
            assert r <= 1e-5, (what, k, r)
        else:
            assert torch.equal(ckpt[1][k], g), (what, k, float((ckpt[1][k] - g).abs().max()))


@pytest.mark.parametrize("sd", [0.0, 0.1])
def test_vit_b16_checkpointing_is_bitwise_equivalent(m, sd):
    """ViT-B/16, 12 layers in 4 segments, at 288 x 288 (S = 325: the streaming attention, whose backward is deterministic): the same logits
    and, but for the fp32-atomic reductions, the same gradients bit for bit; with stochastic depth the replayed keys give the same masks."""
    torch.manual_seed(0)
    model = m.VisionTransformer(m.default_vit_opts("base", n_classes=100, **{"model.classification.vit.stochastic_dropout": sd})).cuda().train()
    x = _image(2, 288, 288, 5)
    y = torch.tensor([3, 71], device="cuda")

    def fn():
        logits = model(x)
        F.cross_entropy(logits.float(), y, label_smoothing=0.1).backward()
        return logits

    plain = _run(m, model, fn, False)
    ck = _run(m, model, fn, True)
    _compare(plain, ck, f"vit-b/16 sd={sd}")


@pytest.mark.parametrize("mask", ["causal", "padding"])
def test_text_tower_checkpointing_is_bitwise_equivalent(m, lib, mask):
    """The CLIP text tower (512 wide, 8 heads of 64), every layer checkpointed, with the causal mask or a key-padding mask.  The streaming
    attention kernels are forced (test mode 2) so that the attention backward is deterministic at S = 77."""
    torch.manual_seed(0)
    opts = m.default_clip_opts("tiny", text_layers=4, **{"model.text.transformer.causal_masking": mask == "causal"})
    tower = m.CLIP(opts).text_encoder.cuda().train()
    g = torch.Generator().manual_seed(9)
    tok = torch.randint(1, 49000, (4, 77), generator=g)
    tok[:, 40] = 49407
    tok = tok.cuda()
    kpm = None
    if mask == "padding":
        kpm = torch.zeros(4, 77, dtype=torch.bool, device="cuda")
        kpm[:, 60:] = True
    gy = bf(rnd(4, 512, seed=1710))

    def fn():
        feats = tower(tok, key_padding_mask=kpm)
        feats.backward(gy.to(feats.dtype))
        return feats

    old = lib.cvb_set_mha_impl(STREAMING)
    try:
        tower.gradient_checkpoint = False
        plain = _run_text(m, tower, fn)
        tower.gradient_checkpoint = True
        ck = _run_text(m, tower, fn)
    finally:
        lib.cvb_set_mha_impl(old)
    _compare(plain, ck, f"text tower {mask}")


def _run_text(m, tower, fn):
    for p in tower.parameters():
        p.grad = None
    m.ops.rng_seed(78, device="cuda")
    out = fn()
    torch.cuda.synchronize()
    return out.detach().clone(), {k: p.grad.detach().clone() for k, p in tower.named_parameters() if p.grad is not None}


@pytest.fixture(scope="module")
def lib(m):
    from ml_cvnets_b200 import _lib as L
    return L.load()


def test_checkpointing_is_ignored_in_eval(m):
    model = m.VisionTransformer(m.default_vit_opts("tiny", n_classes=10, **{CKPT: True})).cuda().eval()
    x = _image(2, 64, 64, 6)
    a = model(x)
    model.gradient_checkpointing = False
    assert torch.equal(a, model(x))


# ------------------------------------------------------------------------------------------------ TrainStep: memory and workspace reporting
def _step_growth(step, x, y):
    """Allocated-memory growth during one eager step (after two warm-up steps of the same configuration)."""
    for _ in range(2):
        step(x, y)
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    step(x, y)
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_vit_b16_checkpointing_saves_memory(m):
    torch.manual_seed(0)
    model = m.VisionTransformer(m.default_vit_opts("base", n_classes=1000)).cuda().train()
    step = m.TrainStep(model, lr=1e-4, weight_decay=0.05, max_norm=1.0, label_smoothing=0.1)
    x = _image(64, 224, 224, 7)
    y = torch.arange(64, device="cuda")
    plain = _step_growth(step, x, y)
    model.gradient_checkpointing = True
    ck = _step_growth(step, x, y)
    print(f"ViT-B/16 B=64 224: step memory growth {plain / 2**30:.2f} GiB plain, {ck / 2**30:.2f} GiB with 4 checkpointed segments "
          f"(ratio {ck / plain:.3f})")
    assert ck <= 0.6 * plain


def test_workspace_reports_every_parameter_once(m):
    """With checkpointing each layer of a recomputed run reports its flat range as its backward finishes, so the all-reduce buckets still tile
    the gradient buffer: every parameter once per step, as without checkpointing."""
    torch.manual_seed(0)
    model = m.VisionTransformer(m.default_vit_opts("tiny", n_classes=10, **{CKPT: True})).cuda().train()
    step = m.TrainStep(model, lr=1e-4)
    seen = []
    real = step.ws.unit_done
    step.ws.unit_done = lambda params: (seen.extend(id(p) for p in params), real(params))
    x, y = _image(4, 96, 96, 8), torch.arange(4, device="cuda")
    counts = {}
    for ck in (False, True):
        model.gradient_checkpointing = ck
        seen.clear()
        step(x, y)
        counts[ck] = Counter(seen)
    torch.cuda.synchronize()
    ids = {id(p) for p in model.parameters()}
    enc = {id(p) for p in model.transformer.parameters()}
    assert counts[True] == counts[False]
    assert enc <= set(counts[True]) and set(counts[True]) <= ids
    assert all(n == 1 for n in counts[True].values())


# ------------------------------------------------------------------------------------------------ captured CLIP ViT-H + RangeAugment step
def _clip_huge_step(m, captured):
    torch.manual_seed(0)
    opts = m.default_clip_opts("huge", projection_dim=512, text_dim=768, text_layers=12, text_heads=12, **AUG,
                               **{CKPT: True, "model.text.transformer.gradient_checkpoint": True})
    model = m.CLIP(opts).cuda().train()
    na = m.NeuralAugmentationLoss(target_value=(40, 20), curriculum_method="cosine", period=10)

    def fl(mod, im, tok, cfg):
        img, txt, scale, x_aug = mod(im, tok)
        return m.clip_contrastive_loss(img, txt, scale, _cfg=cfg), x_aug

    step = m.TrainStep(model, lr=1e-5, betas=(0.9, 0.98), eps=1e-6, weight_decay=0.2, max_norm=None, ema_momentum=0.0005, aug_loss=na,
                       forward_loss=fl)
    step.set_epoch(2)
    g = torch.Generator().manual_seed(11)
    tok = torch.randint(1, 49000, (8, 77), generator=g)
    tok[torch.arange(8), torch.randint(5, 77, (8,), generator=g)] = 49407
    x, tok = _image(8, 224, 224, 12), tok.cuda()
    m.ops.rng_seed(31, device="cuda")
    before = model.image_encoder.transformer[0].pre_norm_ffn[1].weight.detach().clone()
    losses = []
    if captured:
        step.capture(x, tok)  # three eager warm-up steps
    for _ in range(6 if not captured else 3):
        losses.append(float(step(x, tok)))
    torch.cuda.synchronize()
    changed = not torch.equal(before, model.image_encoder.transformer[0].pre_norm_ffn[1].weight)
    return losses, changed


def test_captured_clip_vit_huge_range_augment_step(m):
    cap, changed = _clip_huge_step(m, captured=True)
    torch.cuda.empty_cache()
    eager, _ = _clip_huge_step(m, captured=False)
    print("captured replays", cap, "eager steps 4-6", eager[3:])
    assert all(math.isfinite(v) for v in cap + eager)
    assert changed
    for a, b in zip(cap, eager[3:]):
        assert abs(a - b) <= 1e-3 * abs(b), (cap, eager)

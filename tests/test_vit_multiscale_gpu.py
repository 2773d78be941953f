"""ViT / CLIP image tower at the multi-scale recipes' crops (-m gpu): the streaming head_dim-64 attention kernels (S > 256), the
interpolating token assembly, and VisionTransformer / TrainStep at resolutions other than 224 x 224."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_sample import at_sample  # noqa: E402
from vit_multiscale_ref import vit_forward_any_size  # noqa: E402
from test_kernels_gpu import _mha_ref, bf, close, rnd  # noqa: E402
from test_modules_gpu import rel_l2  # noqa: E402

pytestmark = pytest.mark.gpu

STREAMING = 2  # cvb_set_mha_impl mode: the streaming kernels for every head_dim-64 shape


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ml_cvnets_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def lib(ops):
    from ml_cvnets_b200 import _lib as L
    return L.load()


def _masks(B, S, mask):
    amask = kpm = None
    if mask == "causal":
        amask = torch.full((S, S), float("-inf"), device="cuda").triu(1)[None].repeat(B, 1, 1).contiguous()
    if mask == "padding":
        kpm = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
        kpm[:, S - max(1, S // 5):] = 1
    return amask, kpm


@pytest.mark.parametrize("B,S,H", [(2, 257, 3), (1, 401, 12), (2, 577, 2), (1, 1025, 2)])
@pytest.mark.parametrize("mask", ["none", "causal", "padding"])
def test_streaming_mha_against_fp32(ops, B, S, H, mask):
    C = H * 64
    qkv = bf(rnd(B * S, 3 * C, seed=81))
    dO = bf(rnd(B * S, C, seed=82))
    amask, kpm = _masks(B, S, mask)
    O_, LSE = ops.mha_fwd(qkv, B, S, H, 64, 0.125, attn_mask=amask, key_padding_mask=kpm)
    x = qkv.float().requires_grad_(True)
    ref = _mha_ref(x, B, S, H, 64, 0.125, amask, kpm)
    close(O_, ref.detach(), what="streaming mha fwd")
    ref.backward(dO.float())
    DQKV = ops.mha_bwd(qkv, O_, dO, LSE, B, S, H, 64, 0.125, attn_mask=amask, key_padding_mask=kpm)
    close(DQKV, x.grad, rtol=3e-2, atol=2e-2 * float(x.grad.abs().max()) + 1e-6, what="streaming mha bwd")


@pytest.mark.parametrize("B,S,H", [(2, 77, 2), (2, 197, 3), (1, 250, 2)])
@pytest.mark.parametrize("mask", ["none", "causal", "padding"])
def test_streaming_matches_register_resident(ops, lib, B, S, H, mask):
    """Forced streaming kernels (test mode 2) against the default kernels: the register-resident wgmma kernels of mha_tc.cu for `none` and
    `padding`, the mma.sync kernels of mha.cu for `causal` (an additive mask).  O, LSE (same convention) and dQKV."""
    C = H * 64
    qkv = bf(rnd(B * S, 3 * C, seed=83))
    dO = bf(rnd(B * S, C, seed=84))
    amask, kpm = _masks(B, S, mask)
    res = {}
    old = lib.cvb_set_mha_impl(0)
    try:
        for name, m in (("default", 0), ("long", STREAMING)):
            lib.cvb_set_mha_impl(m)
            O_, LSE = ops.mha_fwd(qkv, B, S, H, 64, 0.125, attn_mask=amask, key_padding_mask=kpm)
            D = ops.mha_bwd(qkv, O_, dO, LSE, B, S, H, 64, 0.125, attn_mask=amask, key_padding_mask=kpm)
            res[name] = (O_.float(), LSE.clone(), D.float())
    finally:
        lib.cvb_set_mha_impl(old)
    for i, what in enumerate(("O", "LSE", "dQKV")):
        a, b = res["long"][i].double(), res["default"][i].double()
        fin = torch.isfinite(b)
        assert torch.equal(fin, torch.isfinite(a)), what
        r = float((a[fin] - b[fin]).norm() / (b[fin].norm() + 1e-30))
        assert r <= 4e-3, f"{what}: streaming vs default rel-L2 {r:.3g}"


def test_streaming_mha_and_token_backward_are_deterministic(ops):
    B, S, H = 2, 401, 4
    C = H * 64
    qkv = bf(rnd(B * S, 3 * C, seed=85))
    dO = bf(rnd(B * S, C, seed=86))
    _, kpm = _masks(B, S, "padding")
    outs = []
    for _ in range(2):
        O_, LSE = ops.mha_fwd(qkv, B, S, H, 64, 0.125, key_padding_mask=kpm)
        D = ops.mha_bwd(qkv, O_, dO, LSE, B, S, H, 64, 0.125, key_padding_mask=kpm)
        outs.append((O_.clone(), LSE.clone(), D.clone()))
    for a, b in zip(*outs):
        assert torch.equal(a, b)
    Bt, N, Ct = 3, 400, 192
    dout = bf(rnd(Bt, N + 1, Ct, seed=87))
    res = []
    for _ in range(2):
        dpos = torch.zeros(196, Ct, device="cuda")
        dcls = torch.zeros(Ct, device="cuda")
        dpatch = ops.vit_tokens_interp_bwd(dout, dpos, dcls, Bt, N, Ct)
        res.append((dpos, dcls, dpatch))
    for a, b in zip(*res):
        assert torch.equal(a, b)


@pytest.mark.parametrize("N", [64, 196, 320, 400, 576])
def test_interpolating_token_kernel(ops, N):
    """196-entry table resampled to N rows as F.interpolate(bilinear, align_corners=False) does, fused into cat(cls, patch + pos); N = 196 is
    the 224-px identity resample."""
    B, C = 3, 192
    pos = rnd(1, 1, 196, C, seed=88)
    cls = rnd(1, 1, C, seed=89)
    patch = bf(rnd(B * N, C, seed=90))
    table = F.interpolate(pos, size=(N, C), mode="bilinear").reshape(N, C)
    # the table alone (zero patch): within 1e-4 of F.interpolate, plus the bf16 rounding of the output
    t_out = ops.vit_tokens_interp_fwd(torch.zeros_like(patch), pos, cls, B, N, C).float()
    assert float((t_out[:, 1:] - table).abs().sub(table.abs() * 2.0 ** -8).max()) <= 1e-4
    out = ops.vit_tokens_interp_fwd(patch, pos, cls, B, N, C).float()
    ref = patch.float().view(B, N, C) + table
    assert float((out[:, 1:] - ref).abs().sub(ref.abs() * 2.0 ** -8).max()) <= 1e-4
    assert torch.equal(out[:, 0], cls.view(1, C).to(torch.bfloat16).float().expand(B, C))
    # backward against autograd
    dout = bf(rnd(B, N + 1, C, seed=91))
    p_ = pos.clone().requires_grad_(True)
    c_ = cls.clone().requires_grad_(True)
    x_ = patch.float().view(B, N, C).requires_grad_(True)
    y = torch.cat((c_.expand(B, -1, -1), x_ + F.interpolate(p_, size=(N, C), mode="bilinear").reshape(1, N, C)), dim=1)
    y.backward(dout.float())
    dpos = torch.zeros(196, C, device="cuda")
    dcls = torch.zeros(C, device="cuda")
    dpatch = ops.vit_tokens_interp_bwd(dout, dpos, dcls, B, N, C)
    assert torch.equal(dpatch.float().view(B, N, C), x_.grad)
    close(dpos, p_.grad.view(196, C), rtol=1e-4, atol=1e-4 * float(p_.grad.abs().max()) + 1e-6, what="dpos", rel_l2=1e-5)
    close(dcls, c_.grad.view(C), rtol=1e-5, atol=1e-6, what="dcls", rel_l2=1e-6)


@pytest.mark.parametrize("crop", ["320x320", "128x128", "256x320"])
def test_vision_transformer_multiscale_against_reference(golden_dir, crop):
    """VisionTransformer ('small': 12 layers, head_dim 64, like base) at the sampler's crops against the REAL reference
    (tests/golden/make_golden_vit_multiscale.py), with the bounds of the 224-px fixture test."""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as pkg
    fx = torch.load(os.path.join(golden_dir, "vit_multiscale_fp32.pt"), weights_only=False)
    c = fx["crops"][crop]
    h, w = c["size"]
    model = pkg.VisionTransformer(pkg.default_vit_opts(fx["mode"]))
    model.load_state_dict(O.seeded_fill_(O.vit_shapes(fx["mode"]), fx["seed"]), strict=True)
    model = model.cuda().train()
    x = O.seeded_input((2, 3, h, w), c["x_seed"]).cuda()
    logits = model(x)
    loss = F.cross_entropy(logits.float(), c["labels"].cuda(), label_smoothing=0.1)
    loss.backward()
    Pa = O.clone_params(O.seeded_fill_(O.vit_shapes(fx["mode"]), fx["seed"]), device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        la = vit_forward_any_size(Pa, x, mode=fx["mode"])
        F.cross_entropy(la, c["labels"].cuda(), label_smoothing=0.1).backward()
    e, ea = rel_l2(logits, c["logits"]), rel_l2(la, c["logits"])
    print(f"[vit small {crop}] logits rel-L2 vs the reference: ours {e:.4g}, torch-autocast {ea:.4g}; loss {float(loss):.5f} vs {float(c['loss']):.5f}")
    assert e <= max(2e-2, 1.5 * ea)
    assert abs(float(loss) - float(c["loss"])) <= 5e-3 * abs(float(c["loss"]))
    named = dict(model.named_parameters())
    total = sum(n * n for n in c["grad_norms"].values()) ** 0.5
    worst = 0.0
    for k, g in c["grads"].items():
        if c["grad_norms"][k] < 1e-3 * total:
            continue
        ours, ref = at_sample(named[k].grad, g)
        auto, _ = at_sample(Pa[k].grad, g)
        eo, eau = rel_l2(ours, ref), rel_l2(auto, ref)
        worst = max(worst, eo)
        assert eo <= max(6e-2, 2.0 * eau), (k, eo, eau)
    print(f"[vit small {crop}] worst parameter-gradient rel-L2 {worst:.4g}")


def test_train_step_over_changing_crops(lib):
    """Eager TrainStep on ViT-tiny over 224 -> 320 -> 128 -> 288 -> 224 with the batch size changing too, twice from the same seed.
    Test mode 2 routes every head_dim-64 attention through the streaming kernels, whose backward is bitwise reproducible (the register-resident
    S <= 256 backward sums dQ with shared-memory atomics).  The encoder's LayerNorm-gain and bias-gradient reductions still depend on
    arrival order in their last bits (at 224 px as well), so the two runs must agree exactly on the first loss and then stay within
    AdamW's noise bound: an update moves a parameter by at most ~lr per step whatever the gradient's noise."""
    import ml_cvnets_b200 as pkg
    from ml_cvnets_b200 import ops
    plan = ((224, 4), (320, 2), (128, 8), (288, 3), (224, 4))
    lr = 1e-3
    old = lib.cvb_set_mha_impl(STREAMING)
    try:
        runs = []
        for _ in range(2):
            torch.manual_seed(0)
            model = pkg.VisionTransformer(pkg.default_vit_opts("tiny", n_classes=100)).cuda().train()
            ts = pkg.TrainStep(model, lr=lr, weight_decay=0.05, max_norm=10.0, label_smoothing=0.1)
            ops.rng_seed(1234)
            g = torch.Generator(device="cuda").manual_seed(5)
            losses = []
            for crop, B in plan:
                x = torch.randn(B, 3, crop, crop, device="cuda", generator=g)
                y = torch.randint(0, 100, (B,), device="cuda", generator=g)
                losses.append(float(ts.step(x, y)))
            torch.cuda.synchronize()
            runs.append((losses, {k: v.detach().clone() for k, v in model.named_parameters()}))
    finally:
        lib.cvb_set_mha_impl(old)
    print("losses", runs[0][0], runs[1][0])
    assert all(torch.isfinite(torch.tensor(l)) for l in runs[0][0] + runs[1][0])
    assert runs[0][0][0] == runs[1][0][0]
    assert max(abs(a - b) for a, b in zip(runs[0][0], runs[1][0])) <= 1e-2
    for k, v in runs[0][1].items():
        assert float((v - runs[1][1][k]).abs().max()) <= 2.5 * lr * len(plan), k


def test_long_sequences_need_head_dim_64():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as pkg
    mha = pkg.MultiHeadAttention(128, 4).cuda()  # head_dim 32
    with pytest.raises(NotImplementedError, match="head_dim"):
        mha(torch.randn(1, 300, 128, device="cuda"))

"""Module- and model-level parity (-m gpu): the drop-in nn.Modules (hand-written CUDA path, bf16 activations) against
(1) the golden fixtures produced by the REAL reference modules in fp32 and (2) the oracle restatement, on identical
seeded parameters and inputs.

Tolerances (stated per SURVEY.md App. C): activations are stored in bf16 (8 mantissa bits, eps = 2^-8 = 3.9e-3) at every
layer boundary, exactly like the reference under ``autocast(bfloat16)``; against the fp32 reference we therefore accept
rel-L2 <= 2e-2 on block outputs, <= 4e-2 on input gradients, <= 5e-2 (and cosine >= 0.998) on parameter gradients, and we
additionally require our error to stay within 2.5x the error of the oracle itself run under bf16 autocast on the same GPU.
"""
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O
from golden_sample import at_sample, ref_norm

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as m
    return m


@pytest.fixture(scope="module")
def mods(golden_dir):
    return torch.load(os.path.join(golden_dir, "modules_fp32.pt"), weights_only=False)


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))


def cosine(a, b):
    a, b = a.detach().float().cpu().flatten(), b.detach().float().cpu().flatten()
    return float(torch.dot(a, b) / (a.norm() * b.norm() + 1e-20))


def load_seeded(module, shapes, seed, prefix="m."):
    P = O.seeded_fill_(shapes, seed)
    sd = {k[len(prefix):]: v for k, v in P.items()}
    module.load_state_dict(sd, strict=True)
    return module.cuda().train()


def autocast_errors(oracle_fn, shapes, seed, fx):
    """Same-precision comparator: the oracle under torch bf16 autocast on this GPU, errors measured against the fp32 reference."""
    P = O.clone_params(O.seeded_fill_(dict(shapes), seed), device="cuda")
    x = fx["x"].cuda().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = oracle_fn(P, x)
    y.backward(fx["gy"].cuda().to(y.dtype))
    return {k: rel_l2(*at_sample(P["m." + k].grad, g)) for k, g in fx["grads"].items()}


def run_and_check(module, fx, out_tol=2e-2, gx_tol=4e-2, gp_tol=5e-2, check_gx=True, auto=None):
    x = fx["x"].cuda().requires_grad_(check_gx)
    y = module(x)
    assert y.shape == fx["y"].shape, (y.shape, fx["y"].shape)
    y.backward(fx["gy"].cuda().to(y.dtype))
    torch.cuda.synchronize()
    errs = {"y": rel_l2(y, fx["y"])}
    assert errs["y"] <= out_tol, f"output rel-L2 {errs['y']:.4g}"
    if check_gx:
        errs["gx"] = rel_l2(x.grad, fx["gx"])
        assert errs["gx"] <= gx_tol, f"input-grad rel-L2 {errs['gx']:.4g}"
    named = dict(module.named_parameters())
    for k, g in fx["grads"].items():
        assert named[k].grad is not None, k
        ours, gs = at_sample(named[k].grad, g)
        e, c = rel_l2(ours, gs), cosine(ours, gs)
        errs[k] = e
        # bias-like gradients are sums over pixels of bf16 gradient tensors: their noise floor is set by bf16 rounding,
        # so the bound is the larger of the fixed tolerance and 3x the torch-autocast error on the same quantity
        tol = max(gp_tol, 3.0 * auto[k]) if auto is not None else gp_tol
        small = ref_norm(g) < 1e-3 * float(fx["gy"].norm())  # e.g. d(query bias): softmax grads sum to ~0
        assert (e <= tol and c >= 1 - tol) or small, f"{k}: rel-L2 {e:.4g} (tol {tol:.3g}) cos {c:.5f} |g|={ref_norm(g):.3g}"
    bufs = dict(module.named_buffers())
    for k, b in fx.get("buffers", {}).items():
        if k.endswith("num_batches_tracked"):
            assert int(bufs[k]) == int(b), k
        else:
            assert rel_l2(bufs[k], b) <= 1e-2, f"{k}: {rel_l2(bufs[k], b):.4g}"
    return errs


def test_stem(pkg, mods):
    fx = mods["stem"]
    shapes = {}
    O._conv_bn(shapes, "m", 3, 16, 3)
    m = load_seeded(pkg.ConvLayer2d(pkg.default_opts(), 3, 16, 3, stride=2, use_norm=True, use_act=True), shapes, fx["seed"])
    run_and_check(m, fx, check_gx=False)


@pytest.mark.parametrize("name", ["ir_s1_res", "ir_s2"])
def test_inverted_residual(pkg, mods, name):
    fx = mods[name]
    c = fx["cfg"]
    shapes = {}
    O.inverted_residual_shapes(shapes, "m", c["cin"], c["cout"], c["expand_ratio"])
    auto = autocast_errors(lambda P, x: O.inverted_residual(P, "m", x, stride=c["stride"]), shapes, fx["seed"], fx)
    m = load_seeded(pkg.InvertedResidual(pkg.default_opts(), c["cin"], c["cout"], c["stride"], c["expand_ratio"]), shapes, fx["seed"])
    run_and_check(m, fx, auto=auto)


def test_mobilevit_block_v2(pkg, mods):
    fx = mods["mvit_v2"]
    c = fx["cfg"]
    shapes = {}
    O.mobilevit_block_v2_shapes(shapes, "m", c["c"], c["d"], c["n_attn_blocks"])
    auto = autocast_errors(lambda P, x: O.mobilevit_block_v2(P, "m", x, n_attn_blocks=c["n_attn_blocks"]), shapes, fx["seed"], fx)
    m = load_seeded(pkg.MobileViTBlockv2(pkg.default_opts(), c["c"], c["d"], 2.0, c["n_attn_blocks"], patch_h=2, patch_w=2), shapes, fx["seed"])
    run_and_check(m, fx, auto=auto)


def test_eval_mode_uses_running_stats(pkg, mods):
    """val_epoch path (engine/training_engine.py:416): model.eval() -> BN normalises with running statistics."""
    fx = mods["ir_s2"]
    c = fx["cfg"]
    shapes = {}
    O.inverted_residual_shapes(shapes, "m", c["cin"], c["cout"], c["expand_ratio"])
    m = load_seeded(pkg.InvertedResidual(pkg.default_opts(), c["cin"], c["cout"], c["stride"], c["expand_ratio"]), shapes, fx["seed"]).eval()
    P = O.clone_params(O.seeded_fill_(shapes, fx["seed"]), requires_grad=False)
    ref = O.inverted_residual(P, "m", fx["x"], stride=c["stride"], training=False)
    before = {k: v.clone() for k, v in m.named_buffers()}
    with torch.no_grad():
        y = m(fx["x"].cuda())
    assert rel_l2(y, ref) <= 2e-2
    for k, v in m.named_buffers():
        assert torch.equal(v, before[k]), k


def _model_and_oracle(pkg, width, seed):
    model = pkg.MobileViTv2(pkg.default_opts(width_multiplier=width))
    P = O.seeded_fill_(O.mobilevit_v2_shapes(width), seed)
    model.load_state_dict(P, strict=True)
    return model.cuda().train(), P


@pytest.mark.parametrize("width", ["1.0", "0.5"])
def test_model_against_reference_golden(pkg, golden_dir, width):
    check_model_against_fixture(pkg, torch.load(os.path.join(golden_dir, "mobilevit_v2_fp32.pt"), weights_only=False)[width])


def check_model_against_fixture(pkg, fx):
    """A train-mode forward / backward of MobileViTv2 at the fixture's width against the real reference's fp32 record, bounded by the oracle
    run under torch bf16 autocast on this GPU."""
    width = str(fx["width"])
    model, P = _model_and_oracle(pkg, fx["width"], fx["seed"])
    x = O.seeded_input((2, 3, fx["res"], fx["res"]), fx["x_seed"]).cuda()
    logits = model(x)
    loss = F.cross_entropy(logits.float(), fx["labels"].cuda(), label_smoothing=0.1)
    loss.backward()
    torch.cuda.synchronize()
    # same-precision comparator: the oracle under bf16 autocast on this GPU
    Pg = O.clone_params(P, device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ref_logits = O.mobilevit_v2_forward(Pg, x, width_multiplier=fx["width"])
        ref_loss = F.cross_entropy(ref_logits, fx["labels"].cuda(), label_smoothing=0.1)
    ref_loss.backward()
    e_ours, e_auto = rel_l2(logits, fx["logits"]), rel_l2(ref_logits, fx["logits"])
    print(f"[width {width}] logits rel-L2 vs fp32 reference: ours {e_ours:.4g}, torch-autocast {e_auto:.4g}; loss ours {float(loss):.5f} ref {float(fx['loss']):.5f}")
    assert e_ours <= max(2.5 * e_auto, 1e-2) + 5e-3, (e_ours, e_auto)
    assert abs(float(loss) - float(fx["loss"])) <= 2e-2 * abs(float(fx["loss"]))
    # Gradients.  Through ~60 bf16 layers with batch-2 BatchNorm the parameter gradients of ANY bf16 implementation sit
    # 10-30% (rel-L2) away from fp32 (tools/diag_grads.py: torch-autocast 0.2-0.25 on the first layers, >1 on tiny
    # gradients), so the bound is relative to the same-precision comparator, per parameter and in aggregate; the truth is the
    # fp32 oracle on this GPU (itself pinned to the reference's gradients by tests/test_oracle_golden.py).
    P32 = O.clone_params(P, device="cuda")
    l32 = O.mobilevit_v2_forward(P32, x, width_multiplier=fx["width"])
    F.cross_entropy(l32, fx["labels"].cuda(), label_smoothing=0.1).backward()
    named = dict(model.named_parameters())
    ours, auto, bad = [], [], []
    for k in fx["grad_norms"]:
        g = named[k].grad
        assert g is not None and torch.isfinite(g).all(), k
        eo, ea = rel_l2(g, P32[k].grad), rel_l2(Pg[k].grad, P32[k].grad)
        ours.append(eo)
        auto.append(ea)
        if eo > 2.0 * ea + 0.05:
            bad.append((k, eo, ea))
    ours_t, auto_t = torch.tensor(ours), torch.tensor(auto)
    print(f"[width {width}] grad rel-L2 vs fp32: median ours {float(ours_t.median()):.4f} autocast {float(auto_t.median()):.4f}; "
          f"mean log-ratio {float((ours_t / auto_t).log().mean()):.3f}; outliers {len(bad)}/{len(ours)}")
    assert float(ours_t.median()) <= 1.25 * float(auto_t.median()) + 0.02
    assert float((ours_t / auto_t).log().mean()) <= 0.2, "on average our gradients must be as close to fp32 as torch-autocast's"
    assert len(bad) <= 0.05 * len(ours), bad[:10]
    bufs = dict(model.named_buffers())
    for k, b in fx["buffers_after"].items():
        if k.endswith("num_batches_tracked"):
            assert int(bufs[k]) == int(b)
        else:  # BatchNorm over very few samples (2x2 maps at batch 2) amplifies bf16 noise: bound by the same-precision comparator
            assert rel_l2(bufs[k], b) <= max(2e-2, 3.0 * rel_l2(Pg[k], b)), (k, rel_l2(bufs[k], b), rel_l2(Pg[k], b))


def test_model_full_resolution_against_oracle(pkg):
    """BASELINE config resolution (256x256), batch 8: logits against the fp32 oracle run on the GPU box's CPU-free path
    (fp32 torch on the same device) + run-to-run stability of two identical forwards."""
    model, P = _model_and_oracle(pkg, 1.0, 5)
    x = O.seeded_input((8, 3, 256, 256), 77).cuda()
    with torch.no_grad():
        model.eval()
        a = model(x)
        b = model(x)
        # GroupNorm statistics are accumulated with atomics (order-dependent fp32 partials): run-to-run noise must stay far
        # below the bf16 resolution of the outputs
        assert rel_l2(a, b) <= 1e-3
        Pg = O.clone_params(P, requires_grad=False, device="cuda")
        ref = O.mobilevit_v2_forward(Pg, x, training=False)
    e = rel_l2(a, ref)
    print(f"eval logits rel-L2 vs fp32 oracle @256: {e:.4g}")
    assert e <= 3e-2
    assert (a.float().argmax(1) == ref.argmax(1)).float().mean() >= 0.75


def test_state_dict_roundtrip_and_deepcopy(pkg):
    """EMA does deepcopy(model) (cvnets/misc/averaging_utils.py:33); checkpoints load strict by key."""
    import copy
    model, _ = _model_and_oracle(pkg, 0.5, 3)
    x = O.seeded_input((2, 3, 64, 64), 9).cuda()
    model.eval()
    with torch.no_grad():
        y0 = model(x)
        clone = copy.deepcopy(model)
        y1 = clone(x)
        fresh = pkg.MobileViTv2(pkg.default_opts(width_multiplier=0.5)).cuda().eval()
        fresh.load_state_dict(model.state_dict(), strict=True)
        y2 = fresh(x)
    assert rel_l2(y1, y0) <= 1e-3 and rel_l2(y2, y0) <= 1e-3


# ------------------------------------------------------------------------------------------- transformer rows (a10-a12)
@pytest.fixture(scope="module")
def tfx(golden_dir):
    return torch.load(os.path.join(golden_dir, "transformer_fp32.pt"), weights_only=False)


@pytest.mark.parametrize("name", ["mha", "mha_hd32", "mha_causal", "mha_padding"])
def test_multi_head_attention(pkg, tfx, name):
    fx = tfx[name]
    c = fx["cfg"]
    shapes = {}
    O.multi_head_attention_shapes(shapes, "m", c["c"])
    kw = {}
    if "attn_mask" in fx:
        kw["attn_mask"] = fx["attn_mask"].cuda()
    if "key_padding_mask" in fx:
        kw["key_padding_mask"] = fx["key_padding_mask"].cuda()
    auto = autocast_errors(lambda P, x: O.multi_head_attention(P, "m", x, c["heads"], key_padding_mask=kw.get("key_padding_mask"),
                                                               attn_mask=kw.get("attn_mask")), shapes, fx["seed"], fx)
    m = load_seeded(pkg.MultiHeadAttention(c["c"], c["heads"]), shapes, fx["seed"])
    mod = lambda x: m(x, **kw)  # noqa: E731
    mod.named_parameters, mod.named_buffers = m.named_parameters, m.named_buffers
    run_and_check(mod, fx, auto=auto)


@pytest.mark.parametrize("name", ["enc_swish", "enc_gelu"])
def test_transformer_encoder(pkg, tfx, name):
    fx = tfx[name]
    c = fx["cfg"]
    shapes = {}
    O.transformer_encoder_shapes(shapes, "m", c["c"], c["ffn"])
    auto = autocast_errors(lambda P, x: O.transformer_encoder(P, "m", x, c["heads"], act=c["act"], eps=c["eps"]), shapes, fx["seed"], fx)
    opts = pkg.default_opts(**{"model.activation.name": c["act"]})
    m = load_seeded(pkg.TransformerEncoder(opts, c["c"], c["ffn"], num_heads=c["heads"]), shapes, fx["seed"])
    assert abs(float(m.pre_norm_mha[0].eps) - c["eps"]) < 1e-12
    run_and_check(m, fx, auto=auto)


@pytest.mark.parametrize("p,p_ffn,p_row", [(0.1, 0.0, 0.0), (0.1, 0.2, 0.0), (0.0, 0.0, 0.25)])
def test_transformer_encoder_dropout_training(pkg, p, p_ffn, p_row):
    """Training-mode dropout / FFN-hidden dropout / stochastic depth (cvnets/modules/transformer.py:77-100, 139-156; the MobileViT-v1 recipe trains
    with dropout 0.1).  The module's hashed masks are reproduced from the same generator state (same seed -> same key sequence) and handed to the
    fp32 oracle as inputs, so outputs, the input gradient and every parameter gradient are compared under IDENTICAL masks."""
    from ml_cvnets_b200 import ops
    C, F_, H, N, S = 64, 128, 4, 16, 40
    shapes = {}
    O.transformer_encoder_shapes(shapes, "m", C, F_)
    opts = pkg.default_opts(**{"model.activation.name": "swish"})
    m = load_seeded(pkg.TransformerEncoder(opts, C, F_, num_heads=H, dropout=p, ffn_dropout=p_ffn, stochastic_dropout=p_row), shapes, 78)
    P = O.clone_params(O.seeded_fill_(dict(shapes), 78), device="cuda")
    g = torch.Generator(device="cuda").manual_seed(3)
    x = torch.randn(N, S, C, device="cuda", generator=g).bfloat16().float()
    gy = torch.randn(N, S, C, device="cuda", generator=g).bfloat16().float()
    ops.rng_seed(99)
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    y.backward(gy.to(y.dtype))
    # the same key sequence: attention branch, ffn branch, then the ffn-hidden key (functional.TransformerEncoderFn.forward)
    ops.rng_seed(99)
    k1, k2 = ops.rng_next("cuda"), ops.rng_next("cuda")
    ones = lambda c: torch.ones(N * S, c, device="cuda", dtype=torch.bfloat16)  # noqa: E731
    m_attn = ops.dropout_fwd(ones(C), None, p, k1, p_row=p_row, rows_per_sample=S).float().view(N, S, C)
    m_ffn = ops.dropout_fwd(ones(C), None, p, k2, p_row=p_row, rows_per_sample=S).float().view(N, S, C)
    m_hid = ops.dropout_fwd(ones(F_), None, p_ffn, ops.rng_next("cuda")).float().view(N, S, F_) if p_ffn > 0 else None
    # masks carry bf16(1/keep); the oracle must scale by the exact factor
    fix = lambda mk, keep: (mk != 0).float() / keep  # noqa: E731
    masks = (fix(m_attn, (1 - p) * (1 - p_row)), None if m_hid is None else fix(m_hid, 1 - p_ffn), fix(m_ffn, (1 - p) * (1 - p_row)))
    assert 0 < float((masks[0] == 0).float().mean()) < 0.6
    xo = x.clone().requires_grad_(True)
    yo = O.transformer_encoder(P, "m", xo, H, act="swish", drop_masks=masks)
    yo.backward(gy)
    assert rel_l2(y, yo) <= 2e-2, rel_l2(y, yo)
    assert rel_l2(xg.grad, xo.grad) <= 5e-2, rel_l2(xg.grad, xo.grad)
    for k, prm in m.named_parameters():
        e = rel_l2(prm.grad, P["m." + k].grad)
        assert e <= 6e-2, f"{k}: {e:.4g}"
    # eval mode: identity
    m.eval()
    ye = m(x.clone())
    yoe = O.transformer_encoder(P, "m", x.clone(), H, act="swish")
    assert rel_l2(ye, yoe) <= 2e-2


def test_dropout_layer_and_classifier_dropout(pkg):
    """Stand-alone Dropout module (cvnets/layers/dropout.py): identity in eval, hashed mask + exact gradient in training; the MobileViT-v1
    classifier head with classifier_dropout = 0.1 (mobilevit.py:110-113) trains."""
    from ml_cvnets_b200 import ops
    d = pkg.Dropout(p=0.25).cuda()
    x = torch.randn(64, 320, device="cuda").bfloat16().requires_grad_(True)
    d.eval()
    assert d(x) is x
    d.train()
    ops.rng_seed(5)
    y = d(x)
    keep = (y != 0).float()
    assert 0.65 < float(keep.mean()) < 0.85
    assert rel_l2(y, x.detach().float() * keep / 0.75) <= 4e-3
    y.float().sum().backward()
    assert rel_l2(x.grad, keep / 0.75) <= 4e-3
    x4 = torch.randn(2, 16, 5, 7, device="cuda")
    y4 = d(x4)
    assert y4.shape == x4.shape and 0.6 < float((y4 != 0).float().mean()) < 0.9


def test_transformer_encoder_vit_base_shape(pkg):
    """ViT-B/16 geometry (SURVEY.md 8a a10: [N,197,768], 12 heads, f=3072, GELU) against the fp32 oracle on this GPU."""
    torch.manual_seed(0)
    C, F_, H, N, S = 768, 3072, 12, 4, 197
    shapes = {}
    O.transformer_encoder_shapes(shapes, "m", C, F_)
    opts = pkg.default_opts(**{"model.activation.name": "gelu"})
    m = load_seeded(pkg.TransformerEncoder(opts, C, F_, num_heads=H), shapes, 77)
    P = O.clone_params(O.seeded_fill_(dict(shapes), 77), device="cuda")
    x = torch.randn(N, S, C, device="cuda").bfloat16().float()
    gy = torch.randn(N, S, C, device="cuda").bfloat16().float()
    xo = x.clone().requires_grad_(True)
    yo = O.transformer_encoder(P, "m", xo, H, act="gelu")
    yo.backward(gy)
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    y.backward(gy.to(y.dtype))
    assert rel_l2(y, yo) <= 2e-2
    assert rel_l2(xg.grad, xo.grad) <= 5e-2
    named = dict(m.named_parameters())
    for k, p in named.items():
        e = rel_l2(p.grad, P["m." + k].grad)
        assert e <= 6e-2, f"{k}: {e:.4g}"

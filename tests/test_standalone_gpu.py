"""Stand-alone drop-in layers (-m gpu): the layers north_star names as drop-in nn.Modules (LinearSelfAttention incl. cross-attention,
LinearAttnFFN, ConvLayer2d 1x1 / depthwise, LayerNorm2D_NCHW, LayerNorm / LayerNormFP32, LinearLayer, GlobalPool) used OUTSIDE the fused
blocks, against fixtures generated from the real reference (tests/golden/make_golden.py, make_golden_r2.py).  Tolerances as in
test_modules_gpu.py: bf16 activations (rel-L2 <= 2e-2 outputs, 4e-2 input gradients, 5e-2 parameter gradients or 3x torch-autocast)."""
import os
import sys

import pytest
import torch

from oracle import cvnets_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_modules_gpu import autocast_errors, load_seeded, rel_l2, run_and_check  # noqa: F401,E402
from golden_sample import at_sample, ref_shape  # noqa: E402

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as m
    return m


@pytest.fixture(scope="module")
def mods(golden_dir):
    d = torch.load(os.path.join(golden_dir, "modules_fp32.pt"), weights_only=False)
    d.update(torch.load(os.path.join(golden_dir, "standalone_fp32.pt"), weights_only=False))
    return d


def _lsa_shapes(d=16):
    shapes = {}
    O._conv_bn(shapes, "m.qkv_proj", d, 2 * d + 1, 1, norm=False, bias=True)
    O._conv_bn(shapes, "m.out_proj", d, d, 1, norm=False, bias=True)
    return shapes


def test_linear_self_attention_standalone(pkg, mods):
    fx = mods["lsa"]
    shapes = _lsa_shapes()
    auto = autocast_errors(lambda P, x: O.linear_self_attention(P, "m", x), shapes, fx["seed"], fx)
    m = load_seeded(pkg.LinearSelfAttention(pkg.default_opts(), embed_dim=16), shapes, fx["seed"])
    run_and_check(m, fx, auto=auto)


def test_linear_attn_ffn_standalone(pkg, mods):
    fx = mods["laffn"]
    shapes = {}
    O.linear_attn_ffn_shapes(shapes, "m", 16, 32)
    auto = autocast_errors(lambda P, x: O.linear_attn_ffn(P, "m", x), shapes, fx["seed"], fx)
    m = load_seeded(pkg.LinearAttnFFN(pkg.default_opts(), embed_dim=16, ffn_latent_dim=32, dropout=0.0), shapes, fx["seed"])
    run_and_check(m, fx, auto=auto)


@pytest.mark.parametrize("name", ["lsa_cross", "laffn_cross"])
def test_cross_attention(pkg, mods, name):
    fx = mods[name]
    if name == "lsa_cross":
        shapes = _lsa_shapes()
        m = load_seeded(pkg.LinearSelfAttention(pkg.default_opts(), embed_dim=16), shapes, fx["seed"])
    else:
        shapes = {}
        O.linear_attn_ffn_shapes(shapes, "m", 16, 32)
        m = load_seeded(pkg.LinearAttnFFN(pkg.default_opts(), embed_dim=16, ffn_latent_dim=32, dropout=0.0), shapes, fx["seed"])
    x, xp = fx["x"].cuda().requires_grad_(True), fx["x_prev"].cuda().requires_grad_(True)
    y = m(x, xp)
    y.backward(fx["gy"].cuda().to(y.dtype))
    assert rel_l2(y, fx["y"]) <= 2e-2
    assert rel_l2(x.grad, fx["gx"]) <= 4e-2 and rel_l2(xp.grad, fx["gx_prev"]) <= 4e-2
    named = dict(m.named_parameters())
    for k, g in fx["grads"].items():
        small = float(g.norm()) < 1e-3 * float(fx["gy"].norm())
        assert rel_l2(named[k].grad, g) <= 6e-2 or small, (k, rel_l2(named[k].grad, g))


@pytest.mark.parametrize("name", ["pw_bn_act", "pw_bias", "dw_bn_act"])
def test_conv_layer_standalone(pkg, mods, name):
    fx = mods[name]
    c = fx["cfg"]
    shapes = {}
    if name == "dw_bn_act":
        O._conv_bn(shapes, "m", c["c"], c["c"], 3, groups=c["c"])
        m = pkg.ConvLayer2d(pkg.default_opts(), c["c"], c["c"], 3, stride=c["stride"], groups=c["c"], use_norm=True, use_act=True)
    elif name == "pw_bn_act":
        O._conv_bn(shapes, "m", c["cin"], c["cout"], 1)
        m = pkg.ConvLayer2d(pkg.default_opts(), c["cin"], c["cout"], 1, use_norm=True, use_act=True)
    else:
        O._conv_bn(shapes, "m", c["cin"], c["cout"], 1, norm=False, bias=True)
        m = pkg.ConvLayer2d(pkg.default_opts(), c["cin"], c["cout"], 1, use_norm=False, use_act=False, bias=True)
    run_and_check(load_seeded(m, shapes, fx["seed"]), fx)


@pytest.mark.parametrize("name", ["ir_se_hs_res", "ir_se_relu_s2", "ir_nose_relu"])
def test_inverted_residual_se(pkg, golden_dir, name):
    """InvertedResidualSE + SqueezeExcitation (SURVEY.md 8f row 4; cvnets/modules/mobilenetv2.py:16-138) vs the real reference's outputs, input
    gradient, every parameter gradient and the BatchNorm running statistics."""
    import copy
    fx = torch.load(os.path.join(golden_dir, "inverted_residual_se_fp32.pt"), weights_only=False)[name]
    c = fx["cfg"]
    shapes = {}
    O.inverted_residual_se_shapes(shapes, "m", c["cin"], c["cout"], c["expand_ratio"], use_se=c["use_se"])
    fn = lambda P, x: O.inverted_residual_se(P, "m", x, stride=c["stride"], act=c["act_fn_name"])  # noqa: E731
    auto = autocast_errors(fn, shapes, fx["seed"], fx)
    # same-precision comparator for the INPUT gradient: batch-4 train-mode BatchNorm followed by ReLU gates (discontinuous derivative) amplifies
    # bf16 rounding for torch autocast as well; ours must stay within 1.5x of it (or the fixed 4e-2)
    Pa = O.clone_params(O.seeded_fill_(dict(shapes), fx["seed"]), device="cuda")
    xa = fx["x"].cuda().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ya = fn(Pa, xa)
    ya.backward(fx["gy"].cuda().to(ya.dtype))
    auto_gx, auto_y = rel_l2(xa.grad, fx["gx"]), rel_l2(ya, fx["y"])
    opts = copy.deepcopy(pkg.default_opts())
    setattr(opts, "model.activation.name", "relu")  # the reference default: fc1 of the SE unit takes the model-wide activation
    m = pkg.InvertedResidualSE(opts, c["cin"], c["cout"], c["expand_ratio"], stride=c["stride"], use_se=c["use_se"], act_fn_name=c["act_fn_name"])
    errs = run_and_check(load_seeded(m, shapes, fx["seed"]), fx, auto=auto, out_tol=max(2e-2, 1.5 * auto_y), gx_tol=max(4e-2, 1.5 * auto_gx))
    print(f"{name}: y {errs['y']:.4f} (autocast {auto_y:.4f})  gx {errs['gx']:.4f} (autocast {auto_gx:.4f})")


@pytest.mark.parametrize("B,HW,C", [(3, 50, 64), (2, 4096, 96), (5, 1, 8)])
def test_se_scale_kernels(pkg, B, HW, C):
    from ml_cvnets_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    X = torch.randn(B * HW, C, device="cuda", generator=g).to(torch.bfloat16)
    S = torch.rand(B, C, device="cuda", generator=g).to(torch.bfloat16)
    DY = torch.randn(B * HW, C, device="cuda", generator=g).to(torch.bfloat16)
    Y = ops.se_scale_fwd(X, S, B, HW)
    ref = (X.float().view(B, HW, C) * S.float()[:, None]).view(B * HW, C)
    assert rel_l2(Y, ref) <= 4e-3
    DX, DS = ops.se_scale_bwd(DY, X, S, B, HW)
    assert rel_l2(DX, (DY.float().view(B, HW, C) * S.float()[:, None]).view(B * HW, C)) <= 4e-3
    assert rel_l2(DS, (DY.float() * X.float()).view(B, HW, C).sum(1)) <= 1e-4


@pytest.mark.parametrize("name", ["ln2d", "ln", "ln_fp32"])
def test_norm_layers_standalone(pkg, mods, name):
    fx = mods[name]
    shapes = {}
    O._gn(shapes, "m", fx["cfg"]["c"])
    cls = {"ln2d": pkg.LayerNorm2D_NCHW, "ln": pkg.LayerNorm, "ln_fp32": pkg.LayerNormFP32}[name]
    run_and_check(load_seeded(cls(fx["cfg"]["c"]), shapes, fx["seed"]), fx)


def test_linear_and_pool_standalone(pkg, mods):
    fx = mods["linear"]
    shapes = {}
    O._linear(shapes, "m", fx["cfg"]["cin"], fx["cfg"]["cout"])
    run_and_check(load_seeded(pkg.LinearLayer(fx["cfg"]["cin"], fx["cfg"]["cout"]), shapes, fx["seed"]), fx)
    fx = mods["pool"]
    run_and_check(pkg.GlobalPool(pool_type="mean").cuda(), fx)


def test_model_batch16_reference_fixture(pkg, golden_dir):
    """Well-conditioned end-to-end fixture from the REAL reference (batch 16, 128x128, train): fixed bounds, no comparator needed."""
    import torch.nn.functional as F
    fx = torch.load(os.path.join(golden_dir, "mobilevit_v2_b16_fp32.pt"), weights_only=False)
    model = pkg.MobileViTv2(pkg.default_opts(width_multiplier=fx["width"]))
    model.load_state_dict(O.seeded_fill_(O.mobilevit_v2_shapes(fx["width"]), fx["seed"]), strict=True)
    model = model.cuda().train()
    x = O.seeded_input((fx["batch"], 3, fx["res"], fx["res"]), fx["x_seed"]).cuda()
    logits = model(x)
    loss = F.cross_entropy(logits.float(), fx["labels"].cuda(), label_smoothing=0.1)
    loss.backward()
    e = rel_l2(logits, fx["logits"])
    Pa = O.clone_params(O.seeded_fill_(O.mobilevit_v2_shapes(fx["width"]), fx["seed"]), device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        la = O.mobilevit_v2_forward(Pa, x, width_multiplier=fx["width"], training=True)
    ea = rel_l2(la, fx["logits"])
    print(f"[b16 fixture] logits rel-L2 vs the reference: ours {e:.4g}, torch-autocast {ea:.4g}; loss {float(loss):.5f} vs {float(fx['loss']):.5f}")
    assert e <= 0.12 and e <= 1.25 * ea + 5e-3  # end-to-end train-mode bf16 (see tests/test_parity_gpu.py for the stage-wise bound)
    assert abs(float(loss) - float(fx["loss"])) <= 5e-3 * abs(float(fx["loss"]))
    named = dict(model.named_parameters())
    total = sum(n * n for n in fx["grad_norms"].values()) ** 0.5
    errs = []
    for k, g in fx["grads"].items():
        if fx["grad_norms"][k] < 1e-3 * total:
            continue
        errs.append((rel_l2(*at_sample(named[k].grad, g)), k))
    errs.sort()
    med, worst = errs[len(errs) // 2], errs[-1]
    print(f"[b16 fixture] parameter-gradient rel-L2 vs the reference: median {med[0]:.4g}, worst {worst[0]:.4g} ({worst[1]}), n={len(errs)}")
    assert med[0] <= 0.25 and worst[0] <= 0.6  # train-mode bf16 gradients at batch 16 (torch-autocast sits at the same level)


def test_dilated_backbone_against_reference_fixture(pkg, golden_dir):
    """SURVEY.md 8f row 4: MobileViTv2 built with output_stride 8 / 16 (segmentation backbones: dilated depthwise convs in layer_4 / layer_5),
    ``extract_end_points_all`` forward + backward against the REAL reference (tests/golden/make_golden_dilated.py)."""
    fx = torch.load(os.path.join(golden_dir, "mobilevit_v2_dilated_fp32.pt"), weights_only=False)
    for os_ in (8, 16):
        rec = fx[f"os{os_}"]
        model = pkg.MobileViTv2(pkg.default_opts(width_multiplier=fx["width"]), output_stride=os_)
        model.load_state_dict(O.seeded_fill_(O.mobilevit_v2_shapes(fx["width"]), fx["seed"]), strict=True)
        model = model.cuda().train()
        dil = {n: list(m.dilation) for n, m in model.named_modules() if isinstance(m, torch.nn.Conv2d) and tuple(m.dilation) != (1, 1)}
        assert dil == rec["dilations"], (dil, rec["dilations"])
        x = O.seeded_input((fx["batch"], 3, fx["res"], fx["res"]), fx["x_seed"]).cuda()
        ends = model.extract_end_points_all(x)
        assert set(ends) == {"out_l1", "out_l2", "out_l3", "out_l4", "out_l5"}
        Pa = O.clone_params(O.seeded_fill_(O.mobilevit_v2_shapes(fx["width"]), fx["seed"]), device="cuda")
        with torch.autocast("cuda", dtype=torch.bfloat16):
            _, st = O.mobilevit_v2_forward(Pa, x, width_multiplier=fx["width"], training=True, return_stages=True, output_stride=os_)
        auto = {"out_l3": st["layer_3.1"], "out_l4": st["layer_4.1"], "out_l5": st["layer_5.1"]}
        for k, v in rec["ends"].items():
            assert tuple(ends[k].shape) == ref_shape(v), (os_, k)
            e, ea = rel_l2(*at_sample(ends[k], v)), rel_l2(*at_sample(auto[k], v))
            print(f"[dilated backbone os={os_}] {k} rel-L2 vs the reference: ours {e:.4g}, torch-autocast {ea:.4g}")
            assert e <= max(3e-2, 1.5 * ea), (os_, k, e, ea)
        if "grads" in rec:
            gy4, gy5 = (O.seeded_input(tuple(ends[k].shape), sd).cuda() for k, sd in zip(("out_l4", "out_l5"), rec["gy_seeds"]))
            ((ends["out_l4"].float() * gy4).sum() + (ends["out_l5"].float() * gy5).sum()).backward()
            ((auto["out_l4"].float() * gy4).sum() + (auto["out_l5"].float() * gy5).sum()).backward()
            named = dict(model.named_parameters())
            total = sum(n * n for n in rec["grad_norms"].values()) ** 0.5
            errs = []
            for k, g in rec["grads"].items():
                if rec["grad_norms"][k] < 1e-3 * total:
                    continue
                errs.append((rel_l2(*at_sample(named[k].grad, g)), rel_l2(*at_sample(Pa[k].grad, g)), k))
            errs.sort()
            med, worst = errs[len(errs) // 2], errs[-1]
            print(f"[dilated backbone os={os_}] parameter-gradient rel-L2: median ours {med[0]:.4g} (autocast {med[1]:.4g}), worst {worst[0]:.4g} "
                  f"(autocast {worst[1]:.4g}, {worst[2]}), n={len(errs)}")
            med_auto = sorted(e[1] for e in errs)[len(errs) // 2]
            assert med[0] <= max(5e-2, 1.5 * med_auto) and worst[0] <= max(0.3, 2.0 * max(e[1] for e in errs))


def test_vision_transformer_against_reference_fixture(pkg, golden_dir):
    """VisionTransformer (BASELINE.json configs[2] family; 'small' geometry = the same code path as ViT-B/16: 12 layers, head_dim 64,
    S = 197, layer_norm_fp32, GELU) against logits / loss / gradients of the REAL reference (tests/golden/make_golden_r2.py)."""
    import torch.nn.functional as F
    fx = torch.load(os.path.join(golden_dir, "vit_small_fp32.pt"), weights_only=False)
    model = pkg.VisionTransformer(pkg.default_vit_opts(fx["mode"]))
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == {k: s for k, s in fx["keys"]}  # state_dict contract
    model.load_state_dict(O.seeded_fill_(O.vit_shapes(fx["mode"]), fx["seed"]), strict=True)
    model = model.cuda().train()
    x = O.seeded_input((2, 3, 224, 224), fx["x_seed"]).cuda()
    logits = model(x)
    loss = F.cross_entropy(logits.float(), fx["labels"].cuda(), label_smoothing=0.1)
    loss.backward()
    # same-precision comparator
    Pa = O.clone_params(O.seeded_fill_(O.vit_shapes(fx["mode"]), fx["seed"]), device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        la = O.vit_forward(Pa, x, mode=fx["mode"])
        F.cross_entropy(la, fx["labels"].cuda(), label_smoothing=0.1).backward()
    e, ea = rel_l2(logits, fx["logits"]), rel_l2(la, fx["logits"])
    print(f"[vit small] logits rel-L2 vs the reference: ours {e:.4g}, torch-autocast {ea:.4g}; loss {float(loss):.5f} vs {float(fx['loss']):.5f}")
    assert e <= max(2e-2, 1.5 * ea)
    assert abs(float(loss) - float(fx["loss"])) <= 5e-3 * abs(float(fx["loss"]))
    named = dict(model.named_parameters())
    total = sum(n * n for n in fx["grad_norms"].values()) ** 0.5
    worst = 0.0
    for k, g in fx["grads"].items():
        if fx["grad_norms"][k] < 1e-3 * total:
            continue
        eo, eau = rel_l2(named[k].grad, g), rel_l2(Pa[k].grad, g)
        worst = max(worst, eo)
        assert eo <= max(6e-2, 2.0 * eau), (k, eo, eau)
    print(f"[vit small] worst parameter-gradient rel-L2 {worst:.4g}")


def test_mobilevit_v1_xxs_against_reference_fixture(pkg, golden_dir):
    """SURVEY.md 8a row a9 / BASELINE.json configs[0]: MobileViT-v1 XXS -- state_dict contract, eval forward at 1x3x256x256 and a train-mode
    forward/backward (dropouts 0) against the REAL reference (dense 3x3 convs via im2col + GEMM, unfold / fold permutations, head dims
    16 / 20 / 24 in the attention core)."""
    check_mobilevit_v1_against_fixture(pkg, torch.load(os.path.join(golden_dir, "mobilevit_v1_xxs_fp32.pt"), weights_only=False), (4, 3, 192, 192))


def check_mobilevit_v1_against_fixture(pkg, fx, train_shape):
    """One MobileViT-v1 mode against the real reference's fp32 record: the state_dict keys, the eval logits at 1x3x256x256 and a train-mode
    forward / backward (dropouts 0) on a ``train_shape`` batch, each bounded by the oracle under torch bf16 autocast on this GPU.  Gradients
    the fixture stores as a sample (tests/golden_sample.py) are compared at the sampled positions."""
    import torch.nn.functional as F
    mode = fx["mode"]
    opts = pkg.default_mit_opts(fx["mode"], **{"model.classification.mit.dropout": 0.0, "model.classification.classifier_dropout": 0.0})
    model = pkg.MobileViT(opts)
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == {k: s for k, s in fx["keys"]}
    model.load_state_dict(O.seeded_fill_(O.mobilevit_v1_shapes(fx["mode"]), fx["seed"]), strict=True)
    model = model.cuda().eval()
    x1 = O.seeded_input((1, 3, 256, 256), fx["eval_x_seed"]).cuda()
    with torch.no_grad():
        ev = model(x1)
        Pa = O.clone_params(O.seeded_fill_(O.mobilevit_v1_shapes(fx["mode"]), fx["seed"]), requires_grad=False, device="cuda")
        with torch.autocast("cuda", dtype=torch.bfloat16):
            eva = O.mobilevit_v1_forward(Pa, x1, mode=fx["mode"], training=False)
    e, ea = rel_l2(ev, fx["eval_logits"]), rel_l2(eva, fx["eval_logits"])
    print(f"[mobilevit v1 {mode}] eval logits rel-L2 vs the reference: ours {e:.4g}, torch-autocast {ea:.4g}")
    assert e <= max(3e-2, 1.5 * ea)
    assert int(ev.argmax()) == int(fx["eval_logits"].argmax()) or e <= 1e-2
    model.train()
    x = O.seeded_input(train_shape, fx["x_seed"]).cuda()
    logits = model(x)
    loss = F.cross_entropy(logits.float(), fx["labels"].cuda(), label_smoothing=0.1)
    loss.backward()
    Pt = O.clone_params(O.seeded_fill_(O.mobilevit_v1_shapes(fx["mode"]), fx["seed"]), device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        lt = O.mobilevit_v1_forward(Pt, x, mode=fx["mode"], training=True)
        F.cross_entropy(lt, fx["labels"].cuda(), label_smoothing=0.1).backward()
    et, eta = rel_l2(logits, fx["logits"]), rel_l2(lt, fx["logits"])
    print(f"[mobilevit v1 {mode}] train logits rel-L2 vs the reference: ours {et:.4g}, torch-autocast {eta:.4g}; loss {float(loss):.5f} vs {float(fx['loss']):.5f}")
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
    return e, et


def test_mobilevit_v1_trains_with_recipe_dropouts(pkg):
    """config/classification/imagenet/mobilevit.yaml trains with mit.dropout 0.1 and classifier_dropout 0.1: the training step must run (hashed-mask
    dropout inside every TransformerEncoder and in the classifier head), be reproducible from the generator seed, differ between steps, and eval
    mode must be dropout-free and deterministic."""
    import torch.nn.functional as F
    from ml_cvnets_b200 import ops
    torch.manual_seed(0)
    model = pkg.MobileViT(pkg.default_mit_opts("xx_small")).cuda().train()
    assert model.classifier.dropout.p == 0.1 and model.layer_3[1].global_rep[0].std_dropout == 0.1
    x = torch.randn(8, 3, 192, 192, device="cuda")  # (192: no layer sees S == d, every map is a multiple of the 2x2 patch)
    y = torch.randint(0, 1000, (8,), device="cuda")

    def step(seed):
        ops.rng_seed(seed)
        model.zero_grad(set_to_none=True)
        for m in model.modules():  # identical BatchNorm state for every run
            if isinstance(m, torch.nn.BatchNorm2d):
                m.reset_running_stats()
        lg = model(x)
        F.cross_entropy(lg.float(), y).backward()
        return lg.detach().float().clone(), model.classifier.fc.weight.grad.detach().clone()

    l1, g1 = step(11)
    l2, g2 = step(11)
    l3, _ = step(12)
    assert torch.isfinite(l1).all() and torch.isfinite(g1).all()
    assert rel_l2(l2, l1) <= 2e-2 and rel_l2(g2, g1) <= 5e-2           # same seed -> same masks (up to atomics-order noise)
    assert rel_l2(l3, l1) > 5 * max(rel_l2(l2, l1), 1e-3)              # another seed -> other masks
    model.eval()
    with torch.no_grad():
        e1, e2 = model(x).float(), model(x).float()
    assert rel_l2(e2, e1) <= 1e-3


def test_clip_against_reference_fixture(pkg, golden_dir):
    """BASELINE.json configs[4] at a reduced geometry (ViT-small image tower, 4-layer causal text transformer): state_dict contract, image /
    text features, contrastive loss and gradients against the REAL reference (tests/golden/make_golden_r2.py)."""
    from ml_cvnets_b200.models_clip import CLIP, clip_contrastive_loss, default_clip_opts
    fx = torch.load(os.path.join(golden_dir, "clip_small_fp32.pt"), weights_only=False)
    model = CLIP(default_clip_opts("small", projection_dim=128, text_dim=256, text_layers=4, text_heads=4, vocab_size=1000, context_length=16))
    assert {k: list(v.shape) for k, v in model.state_dict().items()} == {k: s for k, s in fx["keys"]}
    shapes = O.clip_shapes("small", proj=128, text_dim=256, text_layers=4, vocab=1000, ctx=16)
    model.load_state_dict(O.seeded_fill_(shapes, fx["seed"]), strict=True)
    model = model.cuda().train()
    images, tokens = O.seeded_input((8, 3, 224, 224), fx["x_seed"]).cuda(), fx["tokens"].cuda()
    img, txt, ls = model(images, tokens)
    loss = clip_contrastive_loss(img, txt, ls)
    loss.backward()
    Pa = O.clone_params(O.seeded_fill_(dict(shapes), fx["seed"]), device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ia, ta = O.clip_forward(Pa, images, tokens, vit_mode="small", text_layers=4, text_heads=4)
        la = O.clip_loss(ia, ta, Pa["logit_scale"])
    la.backward()
    ei, et = rel_l2(img, fx["image_features"]), rel_l2(txt, fx["text_features"])
    print(f"[clip] feature rel-L2 vs the reference: image {ei:.4g} (autocast {rel_l2(ia, fx['image_features']):.4g}), text {et:.4g} "
          f"(autocast {rel_l2(ta, fx['text_features']):.4g}); loss {float(loss):.5f} vs {float(fx['loss']):.5f} (autocast {float(la):.5f})")
    assert ei <= 2e-2 and et <= 2e-2
    assert abs(float(loss) - float(fx["loss"])) <= max(2e-2 * abs(float(fx["loss"])), 2.0 * abs(float(la) - float(fx["loss"])))
    named = dict(model.named_parameters())
    total = sum(n * n for n in fx["grad_norms"].values()) ** 0.5
    bad = []
    for k, g in fx["grads"].items():
        if fx["grad_norms"][k] < 1e-3 * total:
            continue
        eo, eau = rel_l2(named[k].grad, g), rel_l2(Pa[k].grad, g)
        if eo > max(0.1, 2.0 * eau):
            bad.append((k, eo, eau))
    assert not bad, bad[:8]
    g_ls, g_ref = float(named["logit_scale"].grad), float(fx["grads"]["logit_scale"])
    assert abs(g_ls - g_ref) <= max(0.1 * abs(g_ref), 3.0 * abs(float(Pa["logit_scale"].grad) - g_ref)), (g_ls, g_ref)

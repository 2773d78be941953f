"""Pin the oracle (oracle/cvnets_oracle.py) to the fixtures generated from the REAL reference
(tests/golden/make_golden.py).  CPU only, fp32, tight tolerances."""
import json
import math
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O
from golden_sample import at_sample, ref_shape

TOL = dict(atol=2e-5, rtol=2e-4)


@pytest.fixture(scope="module")
def mods(golden_dir):
    return torch.load(os.path.join(golden_dir, "modules_fp32.pt"), weights_only=False)


def _run(fn, P, fx):
    x = fx["x"].clone().requires_grad_(True)
    y = fn(P, x)
    y.backward(fx["gy"])
    return x, y


def _check(P, fx, x, y, prefix="m."):
    torch.testing.assert_close(y, fx["y"], **TOL)
    torch.testing.assert_close(x.grad, fx["gx"], **TOL)
    for k, g in fx["grads"].items():
        torch.testing.assert_close(*at_sample(P[prefix + k].grad, g), atol=5e-5, rtol=5e-4, msg=lambda m, k=k: f"{k}: {m}")
    for k, b in fx["buffers"].items():
        torch.testing.assert_close(P[prefix + k].detach(), b, **TOL, msg=lambda m, k=k: f"{k}: {m}")


def test_stem(mods):
    fx = mods["stem"]
    P = {}
    O._conv_bn(P, "m", 3, 16, 3)
    P = O.clone_params(O.seeded_fill_(P, fx["seed"]))
    x, y = _run(lambda P, x: O.conv_layer_2d(P, "m", x, stride=2), P, fx)
    _check(P, fx, x, y)


@pytest.mark.parametrize("name", ["ir_s1_res", "ir_s2"])
def test_inverted_residual(mods, name):
    fx = mods[name]
    c = fx["cfg"]
    P = {}
    O.inverted_residual_shapes(P, "m", c["cin"], c["cout"], c["expand_ratio"])
    P = O.clone_params(O.seeded_fill_(P, fx["seed"]))
    x, y = _run(lambda P, x: O.inverted_residual(P, "m", x, stride=c["stride"]), P, fx)
    _check(P, fx, x, y)


@pytest.mark.parametrize("name", ["ir_se_hs_res", "ir_se_relu_s2", "ir_nose_relu"])
def test_inverted_residual_se(golden_dir, name):
    """InvertedResidualSE / SqueezeExcitation (cvnets/modules/mobilenetv2.py:16-138, squeeze_excitation.py) against the real reference."""
    fx = torch.load(os.path.join(golden_dir, "inverted_residual_se_fp32.pt"), weights_only=False)[name]
    c = fx["cfg"]
    P = {}
    O.inverted_residual_se_shapes(P, "m", c["cin"], c["cout"], c["expand_ratio"], use_se=c["use_se"])
    P = O.clone_params(O.seeded_fill_(P, fx["seed"]))
    x, y = _run(lambda P, x: O.inverted_residual_se(P, "m", x, stride=c["stride"], act=c["act_fn_name"]), P, fx)
    _check(P, fx, x, y)


def test_linear_self_attention(mods):
    fx = mods["lsa"]
    P = {}
    O._conv_bn(P, "m.qkv_proj", 16, 33, 1, norm=False, bias=True)
    O._conv_bn(P, "m.out_proj", 16, 16, 1, norm=False, bias=True)
    P = O.clone_params(O.seeded_fill_(P, fx["seed"]))
    x, y = _run(lambda P, x: O.linear_self_attention(P, "m", x), P, fx)
    _check(P, fx, x, y)


def test_linear_attn_ffn(mods):
    fx = mods["laffn"]
    P = {}
    O.linear_attn_ffn_shapes(P, "m", 16, 32)
    P = O.clone_params(O.seeded_fill_(P, fx["seed"]))
    x, y = _run(lambda P, x: O.linear_attn_ffn(P, "m", x), P, fx)
    _check(P, fx, x, y)


def test_mobilevit_block_v2(mods):
    fx = mods["mvit_v2"]
    c = fx["cfg"]
    P = {}
    O.mobilevit_block_v2_shapes(P, "m", c["c"], c["d"], c["n_attn_blocks"])
    P = O.clone_params(O.seeded_fill_(P, fx["seed"]))
    x, y = _run(lambda P, x: O.mobilevit_block_v2(P, "m", x, n_attn_blocks=c["n_attn_blocks"]), P, fx)
    _check(P, fx, x, y)


def test_unfold_index_map(mods):
    """SURVEY 8a a5: patches[b,c,p,n] = x[b,c,(n//n_w)*2 + p//2, (n%n_w)*2 + p%2]; fold is the inverse."""
    fx = mods["unfold_probe"]
    x = fx["x"]
    patches, size = O.unfolding(x)
    assert torch.equal(patches, fx["patches"])
    B, C, H, W = x.shape
    nw = W // 2
    for p in range(4):
        for n in range(patches.shape[-1]):
            assert torch.equal(patches[:, :, p, n], x[:, :, (n // nw) * 2 + p // 2, (n % nw) * 2 + p % 2])
    assert torch.equal(O.folding(patches, size), x)


def test_state_dict_contract(golden_dir):
    with open(os.path.join(golden_dir, "state_dict_contract.json")) as f:
        contract = json.load(f)
    for width, entries in contract.items():
        P = O.mobilevit_v2_shapes(float(width))
        assert list(P.keys()) == [e[0] for e in entries] or set(P.keys()) == {e[0] for e in entries}
        for k, shape, dtype in entries:
            assert list(P[k].shape) == shape, k
    assert sum(v.numel() for k, v in O.mobilevit_v2_shapes(1.0).items()
               if not k.endswith(("running_mean", "running_var", "num_batches_tracked"))) == 4901841


def _noise_floor(norms):
    """Gradients below this norm are analytically zero (e.g. the bias of a BatchNorm whose output only feeds another normalisation): what the
    fixture stores for them is the floating-point rounding of the CPU it was generated on, so only their smallness is checked."""
    return 1e-6 * math.sqrt(sum(float(n) ** 2 for n in norms))


@pytest.mark.parametrize("width", ["1.0", "0.5"])
def test_mobilevit_v2_model(golden_dir, width):
    fx = torch.load(os.path.join(golden_dir, "mobilevit_v2_fp32.pt"), weights_only=False)[width]
    P = O.clone_params(O.seeded_fill_(O.mobilevit_v2_shapes(fx["width"]), fx["seed"]))
    x = O.seeded_input((2, 3, fx["res"], fx["res"]), fx["x_seed"])
    logits, stages = O.mobilevit_v2_forward(P, x, width_multiplier=fx["width"], return_stages=True)
    loss = F.cross_entropy(logits, fx["labels"], label_smoothing=0.1)
    loss.backward()
    torch.testing.assert_close(logits, fx["logits"], atol=1e-4, rtol=1e-4)
    torch.testing.assert_close(loss.detach(), fx["loss"], atol=1e-5, rtol=1e-5)
    last = {"conv_1": "conv_1", "layer_1": "layer_1.0", "layer_2": "layer_2.1", "layer_3": "layer_3.1",
            "layer_4": "layer_4.1", "layer_5": "layer_5.1"}
    for name, pre in last.items():
        v = stages[pre].detach()
        assert abs(float(v.norm()) - fx["stage_norms"][name]) <= 1e-4 * fx["stage_norms"][name]
        torch.testing.assert_close(v.flatten()[:: max(1, v.numel() // 512)][:512], fx["stage_sample"][name], atol=1e-4, rtol=1e-3)
    for k, n in fx["grad_norms"].items():
        assert abs(float(P[k].grad.norm()) - n) <= 2e-3 * n + 1e-6, (k, float(P[k].grad.norm()), n)
    floor = _noise_floor(fx["grad_norms"].values())
    for k, g in fx["grad_small"].items():
        if float(g.norm()) < floor:
            assert float(P[k].grad.norm()) < 2 * floor, k
            continue
        torch.testing.assert_close(P[k].grad, g, atol=1e-4 * float(g.abs().max()) + 1e-7, rtol=2e-3, msg=lambda m, k=k: f"{k}: {m}")
    for k, b in fx["buffers_after"].items():
        torch.testing.assert_close(P[k].detach(), b, atol=1e-5, rtol=1e-4)


# ------------------------------------------------------------------------------------------- transformer rows (a10-a12)
@pytest.fixture(scope="module")
def tfx(golden_dir):
    return torch.load(os.path.join(golden_dir, "transformer_fp32.pt"), weights_only=False)


def _check_nobuf(P, fx, x, y, prefix="m."):
    torch.testing.assert_close(y, fx["y"], **TOL)
    torch.testing.assert_close(x.grad, fx["gx"], **TOL)
    for k, g in fx["grads"].items():
        torch.testing.assert_close(*at_sample(P[prefix + k].grad, g), atol=5e-5, rtol=5e-4, msg=lambda m, k=k: f"{k}: {m}")


@pytest.mark.parametrize("name", ["mha", "mha_hd32", "mha_causal", "mha_padding"])
def test_multi_head_attention(tfx, name):
    fx = tfx[name]
    c = fx["cfg"]
    P = {}
    O.multi_head_attention_shapes(P, "m", c["c"])
    P = O.clone_params(O.seeded_fill_(P, fx["seed"]))
    x, y = _run(lambda P, x: O.multi_head_attention(P, "m", x, c["heads"], key_padding_mask=fx.get("key_padding_mask"),
                                                     attn_mask=fx.get("attn_mask")), P, fx)
    _check_nobuf(P, fx, x, y)


@pytest.mark.parametrize("name", ["enc_swish", "enc_gelu"])
def test_transformer_encoder(tfx, name):
    fx = tfx[name]
    c = fx["cfg"]
    P = {}
    O.transformer_encoder_shapes(P, "m", c["c"], c["ffn"])
    P = O.clone_params(O.seeded_fill_(P, fx["seed"]))
    x, y = _run(lambda P, x: O.transformer_encoder(P, "m", x, c["heads"], act=c["act"], eps=c["eps"]), P, fx)
    _check_nobuf(P, fx, x, y)


# ---------------------------------------------------------------------------------------- round-2 fixtures (make_golden_r2.py)
@pytest.fixture(scope="module")
def standalone(golden_dir):
    return torch.load(os.path.join(golden_dir, "standalone_fp32.pt"), weights_only=False)


@pytest.mark.parametrize("name", ["lsa_cross", "laffn_cross"])
def test_cross_attention(standalone, name):
    """LinearSelfAttention / LinearAttnFFN cross-attention branch against the real reference (linear_attention.py:163-207)."""
    fx = standalone[name]
    shapes = {}
    if name == "lsa_cross":
        O._conv_bn(shapes, "m.qkv_proj", 16, 33, 1, norm=False, bias=True)
        O._conv_bn(shapes, "m.out_proj", 16, 16, 1, norm=False, bias=True)
        fn = O.linear_self_attention
    else:
        O.linear_attn_ffn_shapes(shapes, "m", fx["cfg"]["d"], fx["cfg"]["ffn"])
        fn = O.linear_attn_ffn
    P = O.clone_params(O.seeded_fill_(shapes, fx["seed"]))
    x, xp = fx["x"].clone().requires_grad_(True), fx["x_prev"].clone().requires_grad_(True)
    y = fn(P, "m", x, xp)
    y.backward(fx["gy"])
    assert torch.allclose(y, fx["y"], atol=2e-5, rtol=2e-5)
    assert torch.allclose(x.grad, fx["gx"], atol=2e-5, rtol=2e-4) and torch.allclose(xp.grad, fx["gx_prev"], atol=2e-5, rtol=2e-4)
    for k, g in fx["grads"].items():
        assert torch.allclose(P["m." + k].grad, g, atol=5e-5, rtol=5e-4), k


def test_model_batch16_fixture(golden_dir):
    """The well-conditioned end-to-end fixture (batch 16, 128x128, train mode): oracle == real reference (logits, loss, gradients)."""
    import torch.nn.functional as F
    fx = torch.load(os.path.join(golden_dir, "mobilevit_v2_b16_fp32.pt"), weights_only=False)
    P = O.clone_params(O.seeded_fill_(O.mobilevit_v2_shapes(fx["width"]), fx["seed"]))
    x = O.seeded_input((fx["batch"], 3, fx["res"], fx["res"]), fx["x_seed"])
    logits = O.mobilevit_v2_forward(P, x, width_multiplier=fx["width"], training=True)
    loss = F.cross_entropy(logits, fx["labels"], label_smoothing=0.1)
    loss.backward()
    assert float((logits - fx["logits"]).norm() / fx["logits"].norm()) <= 2e-5
    assert abs(float(loss) - float(fx["loss"])) <= 1e-5
    for k, n in fx["grad_norms"].items():
        assert abs(float(P[k].grad.norm()) - n) <= 2e-3 * n + 1e-7, k
    floor = _noise_floor(fx["grad_norms"].values())
    for k, g in fx["grads"].items():
        if fx["grad_norms"][k] < floor:
            assert float(P[k].grad.norm()) < 2 * floor, k
            continue
        ours, g = at_sample(P[k].grad, g)
        e = float((ours - g.float()).norm() / (g.float().norm() + 1e-12))
        assert e <= (2e-3 if g.dtype == torch.float16 else 2e-4), (k, e)


def test_vit_small_fixture(golden_dir):
    """VisionTransformer restatement (conv stem, cls / positional embedding, 12 encoders, post norm, classifier) == the real reference."""
    import torch.nn.functional as F
    fx = torch.load(os.path.join(golden_dir, "vit_small_fp32.pt"), weights_only=False)
    shapes = O.vit_shapes(fx["mode"])
    assert {k: list(v.shape) for k, v in shapes.items()} == {k: s for k, s in fx["keys"]}
    P = O.clone_params(O.seeded_fill_(shapes, fx["seed"]))
    x = O.seeded_input((2, 3, 224, 224), fx["x_seed"])
    logits = O.vit_forward(P, x, mode=fx["mode"], training=True)
    loss = F.cross_entropy(logits, fx["labels"], label_smoothing=0.1)
    loss.backward()
    assert float((logits - fx["logits"]).norm() / fx["logits"].norm()) <= 2e-5
    assert abs(float(loss) - float(fx["loss"])) <= 1e-5
    for k, n in fx["grad_norms"].items():
        assert abs(float(P[k].grad.norm()) - n) <= 2e-3 * n + 1e-7, k
    for k, g in fx["grads"].items():
        assert float((P[k].grad - g).norm() / (g.norm() + 1e-12)) <= 5e-4, k


def test_mobilevit_v1_xxs_fixture(golden_dir):
    """MobileViT-v1 XXS (BASELINE.json configs[0]): eval forward at 1x3x256x256 and a train-mode forward/backward == the real reference."""
    import torch.nn.functional as F
    fx = torch.load(os.path.join(golden_dir, "mobilevit_v1_xxs_fp32.pt"), weights_only=False)
    shapes = O.mobilevit_v1_shapes(fx["mode"])
    assert {k: list(v.shape) for k, v in shapes.items()} == {k: s for k, s in fx["keys"]}
    P = O.clone_params(O.seeded_fill_(shapes, fx["seed"]))
    with torch.no_grad():
        ev = O.mobilevit_v1_forward(P, O.seeded_input((1, 3, 256, 256), fx["eval_x_seed"]), mode=fx["mode"], training=False)
    assert float((ev - fx["eval_logits"]).norm() / fx["eval_logits"].norm()) <= 2e-5
    logits = O.mobilevit_v1_forward(P, O.seeded_input((4, 3, 192, 192), fx["x_seed"]), mode=fx["mode"], training=True)
    loss = F.cross_entropy(logits, fx["labels"], label_smoothing=0.1)
    loss.backward()
    assert float((logits - fx["logits"]).norm() / fx["logits"].norm()) <= 5e-5
    assert abs(float(loss) - float(fx["loss"])) <= 1e-5
    floor = _noise_floor(g.norm() for g in fx["grads"].values())
    for k, g in fx["grads"].items():
        if float(g.norm()) < floor:
            assert float(P[k].grad.norm()) < 2 * floor, k
            continue
        assert float((P[k].grad - g).norm() / (g.norm() + 1e-12)) <= 2e-3, k


def test_clip_small_fixture(golden_dir):
    """CLIP restatement (ViT image tower + projection head, causal text transformer + EOT gather + projection, contrastive loss with the
    learnable temperature) == the real reference at a reduced geometry."""
    fx = torch.load(os.path.join(golden_dir, "clip_small_fp32.pt"), weights_only=False)
    shapes = O.clip_shapes("small", proj=128, text_dim=256, text_layers=4, vocab=1000, ctx=16)
    assert {k: list(v.shape) for k, v in shapes.items()} == {k: s for k, s in fx["keys"]}
    P = O.clone_params(O.seeded_fill_(shapes, fx["seed"]))
    img, txt = O.clip_forward(P, O.seeded_input((8, 3, 224, 224), fx["x_seed"]), fx["tokens"], vit_mode="small", text_layers=4, text_heads=4)
    loss = O.clip_loss(img, txt, P["logit_scale"])
    loss.backward()
    assert float((img - fx["image_features"]).norm() / fx["image_features"].norm()) <= 2e-5
    assert float((txt - fx["text_features"]).norm() / fx["text_features"].norm()) <= 2e-5
    assert abs(float(loss) - float(fx["loss"])) <= 1e-5
    for k, n in fx["grad_norms"].items():
        assert abs(float(P[k].grad.norm()) - n) <= 3e-3 * n + 1e-7, k


def test_dilated_backbone_fixture(golden_dir):
    """SURVEY.md 8f row 4: MobileViTv2 as a segmentation backbone (output_stride 8 / 16: layer_4 / layer_5 dilate instead of striding).
    Oracle end points and gradients == the real reference (tests/golden/make_golden_dilated.py)."""
    fx = torch.load(os.path.join(golden_dir, "mobilevit_v2_dilated_fp32.pt"), weights_only=False)
    for os_ in (8, 16):
        rec = fx[f"os{os_}"]
        P = O.clone_params(O.seeded_fill_(O.mobilevit_v2_shapes(fx["width"]), fx["seed"]))
        x = O.seeded_input((fx["batch"], 3, fx["res"], fx["res"]), fx["x_seed"])
        _, st = O.mobilevit_v2_forward(P, x, width_multiplier=fx["width"], training=True, return_stages=True, output_stride=os_)
        ends = {"out_l3": st["layer_3.1"], "out_l4": st["layer_4.1"], "out_l5": st["layer_5.1"]}
        for k, v in rec["ends"].items():
            assert tuple(ends[k].shape) == ref_shape(v), (os_, k, ends[k].shape, ref_shape(v))
            ours, v = at_sample(ends[k], v)
            assert float((ours - v).norm() / v.norm()) <= 2e-5, (os_, k)
        if "grads" in rec:
            gy4, gy5 = (O.seeded_input(tuple(ends[k].shape), sd) for k, sd in zip(("out_l4", "out_l5"), rec["gy_seeds"]))
            ((ends["out_l4"] * gy4).sum() + (ends["out_l5"] * gy5).sum()).backward()
            for k, n in rec["grad_norms"].items():
                assert abs(float(P[k].grad.norm()) - n) <= 2e-3 * n + 1e-6, k
            for k, g in rec["grads"].items():
                ours, g = at_sample(P[k].grad, g)
                assert float((ours - g).norm() / (g.norm() + 1e-12)) <= 5e-4, k

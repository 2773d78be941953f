"""EfficientNet without a GPU: the fp32 restatement (tests/efficientnet_ref.py) pinned to the fixtures generated from the real reference
(tests/golden/make_golden_efficientnet.py), and the drop-in modules' constructor / child-tree / state_dict contract for b0 .. b3."""
import hashlib
import inspect
import json
import os

import pytest
import torch

import efficientnet_ref as E
from golden_sample import at_sample
from oracle import cvnets_oracle as O

TOL = dict(atol=2e-5, rtol=2e-4)


@pytest.fixture(scope="module")
def fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "efficientnet_fp32.pt"), weights_only=False)


def _check(P, f, fn, prefix="m."):
    x = O.seeded_input(f["x_shape"], f["x_seed"]).requires_grad_(True)
    y = fn(P, x)
    y.backward(O.seeded_input(tuple(y.shape), f["gy_seed"]))
    torch.testing.assert_close(*at_sample(y.detach(), f["y"]), **TOL)
    torch.testing.assert_close(*at_sample(x.grad, f["gx"]), **TOL)
    for k, g in f["grads"].items():
        torch.testing.assert_close(*at_sample(P[prefix + k].grad, g), atol=5e-5, rtol=5e-4, msg=lambda m, k=k: f"{k}: {m}")
    for k, b in f["buffers"].items():
        torch.testing.assert_close(*at_sample(P[prefix + k].detach(), b), **TOL, msg=lambda m, k=k: f"{k}: {m}")


@pytest.mark.parametrize("name", ["dw5_s1", "dw5_s2"])
def test_depthwise_5x5_conv_layer(fx, name):
    f = fx[name]
    c = f["cfg"]
    P = {}
    O._conv_bn(P, "m", c["c"], c["c"], 5, groups=c["c"])
    P = O.clone_params(O.seeded_fill_(P, f["seed"]))
    _check(P, f, lambda P, x: O.conv_layer_2d(P, "m", x, stride=c["stride"], groups=c["c"], use_act=False))


@pytest.mark.parametrize("name", ["eb_e1_k3", "eb_e6_k5_s2", "eb_e6_k5_res"])
def test_efficientnet_block(fx, name):
    f = fx[name]
    c = f["cfg"]
    P = {}
    E.efficientnet_block_shapes(P, "m", c["cin"], c["cout"], c["expand_ratio"], c["kernel_size"])
    P = O.clone_params(O.seeded_fill_(P, f["seed"]))
    _check(P, f, lambda P, x: E.efficientnet_block(P, "m", x, stride=c["stride"]))


def test_efficientnet_b0(fx):
    f = fx["b0_64"]
    P = O.clone_params(O.seeded_fill_(E.efficientnet_shapes("b0"), f["seed"]))
    _check(P, f, lambda P, x: E.efficientnet_forward(P, x, mode="b0"), prefix="")


def _params(f):
    return [p for p in inspect.signature(f).parameters if p not in ("args", "kwargs")]


@pytest.mark.parametrize("mode", ["b0", "b1", "b2", "b3"])
def test_model_contract(fx, mode):
    """Constructor parameters, child tree, state_dict [key, shape, dtype] (b0 as a list, every mode as a digest), per-block kernel sizes and stochastic-depth probabilities (rounded
    to 4 digits as the reference rounds them) against the reference classes; the restatement's shapes agree too."""
    import ml_cvnets_b200 as m
    ref = fx["contract"]
    assert _params(m.EfficientNetBlock.__init__) == ref["block_init"]
    assert _params(m.EfficientNet.__init__) == ref["model_init"]
    r = ref["models"][mode]
    model = m.EfficientNet(m.default_effnet_opts(mode, **{"model.classification.efficientnet.stochastic_depth_prob": 0.2}))
    entries = [[k, list(v.shape), str(v.dtype)] for k, v in model.state_dict().items()]
    if mode == "b0":
        assert entries == ref["b0_state_dict"]
    digest = {"n_entries": len(entries), "sha256": hashlib.sha256(json.dumps(entries, separators=(",", ":")).encode()).hexdigest()}
    assert digest == r["state_dict"]
    assert [n for n, _ in model.named_children()] == r["children"]
    blocks = [b for n in ("layer_1", "layer_2", "layer_3", "layer_4", "layer_5") for b in getattr(model, n)]
    assert [float(b.stochastic_depth.p) for b in blocks] == r["sd_probs"]
    assert [int(b.kernel_size) for b in blocks] == r["kernels"]
    assert repr(model.layer_4[3]) == r["block_repr"]
    shapes = E.efficientnet_shapes(mode)
    assert {k: list(v.shape) for k, v in shapes.items()} == {k: s for k, s, _ in entries}


def test_cpu_tensors_raise_and_optimizer_choice_is_checked():
    import ml_cvnets_b200 as m
    opts = m.default_effnet_opts("b0")
    blk = m.EfficientNetBlock(0.1, opts=opts, in_channels=40, out_channels=40, kernel_size=5, stride=1, expand_ratio=6, use_se=True,
                              squeeze_factor=24, act_fn_name="swish", se_scale_fn_name="sigmoid")
    with pytest.raises(RuntimeError):
        blk(torch.zeros(2, 40, 8, 8))
    model = m.EfficientNet(opts)
    with pytest.raises(RuntimeError):
        model(torch.zeros(1, 3, 64, 64))
    with pytest.raises(ValueError):
        m.TrainStep(model, optimizer="lamb")

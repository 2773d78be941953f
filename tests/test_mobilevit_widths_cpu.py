"""MobileViTv2 at the published widths the other fixtures do not hold (0.75, 1.25, 1.5, 1.75, 2.0), CPU only: the fp32 oracle against the
real reference's fixtures (tests/golden/make_golden_widths.py), the drop-in model's state_dict against the reference's key / shape / dtype
contract, and the configuration table at all seven widths."""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O
from test_oracle_golden import _noise_floor

WIDTHS = ["0.75", "1.25", "1.5", "1.75", "2.0"]


def load_width_fixture(golden_dir, width):
    """the real reference's record at one width (tests/golden/make_golden_widths.py writes one file per width)"""
    return torch.load(os.path.join(golden_dir, f"mobilevit_v2_w{width}_fp32.pt"), weights_only=False)


@pytest.fixture(scope="module")
def wfx(golden_dir):
    return {w: load_width_fixture(golden_dir, w) for w in WIDTHS}


@pytest.fixture(scope="module")
def contract(golden_dir):
    with open(os.path.join(golden_dir, "state_dict_contract_widths.json")) as f:
        return json.load(f)


def test_fixture_holds_every_width(wfx, contract):
    assert sorted(contract, key=float) == WIDTHS
    for w in WIDTHS:
        assert wfx[w]["width"] == float(w) and wfx[w]["res"] == 128


@pytest.mark.parametrize("width", WIDTHS)
def test_oracle_matches_reference(wfx, width):
    """The tolerances of test_oracle_golden.py::test_mobilevit_v2_model."""
    fx = wfx[width]
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
        assert abs(float(v.norm()) - fx["stage_norms"][name]) <= 1e-4 * fx["stage_norms"][name], name
        torch.testing.assert_close(v.flatten()[:: max(1, v.numel() // 512)][:512], fx["stage_sample"][name], atol=1e-4, rtol=1e-3)
    assert fx["grad_norms"].keys() == {k for k, p in P.items() if p.requires_grad}
    for k, n in fx["grad_norms"].items():
        assert abs(float(P[k].grad.norm()) - n) <= 2e-3 * n + 1e-6, (k, float(P[k].grad.norm()), n)
    floor = _noise_floor(fx["grad_norms"].values())
    assert len(fx["grad_small"]) > 100
    for k, g in fx["grad_small"].items():
        if float(g.norm()) < floor:
            assert float(P[k].grad.norm()) < 2 * floor, k
            continue
        torch.testing.assert_close(P[k].grad, g, atol=1e-4 * float(g.abs().max()) + 1e-7, rtol=2e-3, msg=lambda m, k=k: f"{k}: {m}")
    for k, b in fx["buffers_after"].items():
        torch.testing.assert_close(P[k].detach(), b, atol=1e-5, rtol=1e-4)


@pytest.mark.parametrize("width", WIDTHS)
def test_state_dict_contract(contract, width):
    import ml_cvnets_b200 as m
    entries = contract[width]
    sd = m.MobileViTv2(m.default_opts(width_multiplier=float(width))).state_dict()
    assert list(sd.keys()) == [e[0] for e in entries]
    for k, shape, dtype in entries:
        assert list(sd[k].shape) == shape and str(sd[k].dtype) == "torch." + dtype, k
    P = O.mobilevit_v2_shapes(float(width))
    assert {k: list(v.shape) for k, v in P.items()} == {k: shape for k, shape, _ in entries}


@pytest.mark.parametrize("width", [0.5, 0.75, 1.0, 1.25, 1.5, 1.75, 2.0])
def test_configuration_matches_oracle(width):
    import ml_cvnets_b200 as m
    # the reference's table also carries last_layer_exp_factor, which its MobileViTv2 never reads; the oracle leaves it out
    assert m.get_configuration(m.default_opts(width_multiplier=width)) == {**O.mobilevit_v2_config(width), "last_layer_exp_factor": 4}

"""Gradient accumulation without a GPU: the fp32 restatement of the reference's accumulating training loop (tests/accum_ref.py) against the
fixture generated from the real reference (tests/golden/make_golden_accum.py: EfficientNet-b0, accum_freq 2, two windows, SGD-Nesterov with
the reference's parameter groups, its EMA).  This pins the semantics the library's TrainStep(accum_freq=...) follows: gradients summed, not
averaged; one optimizer update and one EMA update per window; BatchNorm statistics moving on every micro-batch.  Also the public signature and
the C ABI declaration of the accumulate kernel."""
import inspect
import os
import re

import pytest
import torch

import accum_ref as A
import efficientnet_ref as E
from oracle import cvnets_oracle as O

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = dict(atol=2e-5, rtol=2e-4)


@pytest.fixture(scope="module")
def fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "accum_fp32.pt"), weights_only=False)


def _inputs(fx):
    c = fx["cfg"]
    xs = [O.seeded_input((c["batch"], 3, c["crop"], c["crop"]), s) for s in c["x_seeds"]]
    return xs, fx["targets"]


def _run(fx, accum_freq=None):
    c = fx["cfg"]
    P = O.clone_params(O.seeded_fill_(E.efficientnet_shapes(c["mode"], c["n_classes"]), c["param_seed"]))
    xs, ys = _inputs(fx)
    return A.train_windows(P, xs, ys, accum_freq=accum_freq or c["accum_freq"], lr=c["lr"], momentum=c["momentum"],
                           weight_decay=c["weight_decay"], label_smoothing=c["label_smoothing"], ema_momentum=c["ema_momentum"], mode=c["mode"])


@pytest.fixture(scope="module")
def run(fx):
    return _run(fx)


def test_restatement_reproduces_the_reference(fx, run):
    losses, micro, windows = run
    assert fx["cfg"]["accum_freq"] == 2 and len(fx["micro"]) == 4 and len(fx["windows"]) == 2
    torch.testing.assert_close(torch.tensor(losses), torch.tensor(fx["losses"]), **TOL)
    for i, (state, want) in enumerate(zip(micro, fx["micro"])):
        torch.testing.assert_close(A.flat_sample([state[k] for k in fx["bn_keys"]]), want, **TOL, msg=lambda m, i=i: f"micro-batch {i}: {m}")
    for i, ((state, mom, ema), want) in enumerate(zip(windows, fx["windows"])):
        torch.testing.assert_close(A.flat_sample([state[k] for k in fx["param_keys"]]), want["params"], **TOL,
                                   msg=lambda m, i=i: f"window {i} parameters: {m}")
        torch.testing.assert_close(A.flat_sample([mom[k] for k in fx["param_keys"]]), want["momentum"], atol=2e-5, rtol=1e-3,
                                   msg=lambda m, i=i: f"window {i} momentum: {m}")
        torch.testing.assert_close(A.flat_sample([ema[k] for k in fx["ema_keys"]]), want["ema"], **TOL,
                                   msg=lambda m, i=i: f"window {i} EMA: {m}")


def test_fixture_pins_summed_gradients_and_update_cadence(fx, run):
    """The fixture tells the semantics apart: the same micro-batches without accumulation (one update each) land elsewhere, the parameters
    move only at a window's end, and the statistics move on every micro-batch."""
    _, micro, _ = run
    _, _, per_batch = _run(fx, accum_freq=1)
    want = fx["windows"][0]["params"]
    assert not torch.allclose(A.flat_sample([per_batch[1][0][k] for k in fx["param_keys"]]), want, **TOL)
    inside = A.flat_sample([micro[0][k] for k in fx["param_keys"]])
    c = fx["cfg"]
    P0 = O.seeded_fill_(E.efficientnet_shapes(c["mode"], c["n_classes"]), c["param_seed"])
    assert torch.equal(inside, A.flat_sample([P0[k] for k in fx["param_keys"]])), "parameters moved inside the window"
    stats = fx["micro"]
    assert all(not torch.equal(a, b) for a, b in zip(stats, stats[1:]))


def test_train_step_signature():
    import ml_cvnets_b200 as m
    p = inspect.signature(m.TrainStep).parameters["accum_freq"]
    assert p.default == 1 and p.kind == inspect.Parameter.KEYWORD_ONLY
    assert callable(m.TrainStep.zero_grad)


def test_accumulate_declared_in_the_abi():
    hdr = open(os.path.join(REPO, "include", "cvnets_b200.h")).read()
    assert re.search(r"CVB_API int cvb_grad_accumulate\(float\* acc, const float\* g, int64_t n, cvb_stream_t stream\);", hdr)
    assert re.search(r"#define CVB_ABI_VERSION 12\b", hdr)


@pytest.mark.parametrize("bad", [0, -2, 1.5, True])
def test_accum_freq_below_one_or_not_an_integer_raises(bad):
    import ml_cvnets_b200 as m
    with pytest.raises(ValueError, match="accum_freq"):
        m.TrainStep(torch.nn.Linear(2, 2), accum_freq=bad)

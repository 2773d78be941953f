"""Classification validation without a GPU: the restatements of tests/eval_ref.py against the fixture generated from the real reference
(tests/golden/make_golden_eval.py: its EMA of the whole state, its eval-mode CrossEntropy and top_k_accuracy), the rank rule on ties, the
C ABI declarations of the two new entry points, and the argument checks of their wrappers."""
import os
import re

import pytest
import torch

import eval_ref as E

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "eval_fp32.pt"), weights_only=False)


def test_ema_restatement_matches_reference_bitwise(fx):
    ema = fx["ema_init"]
    assert any(not v.is_floating_point() for v in ema.values()), "the fixture must cover num_batches_tracked"
    for live, want in zip(fx["live_states"], fx["ema_states"]):
        ema = E.ema_state(ema, live, fx["momentum"])
        assert set(ema) == set(want)
        for k in want:
            assert ema[k].dtype == want[k].dtype and torch.equal(ema[k], want[k]), k


def test_ema_flat_is_the_state_update(fx):
    """The flat-buffer form (cvb_ema_update's order) gives the same floats as the per-tensor state update."""
    ema, live = fx["ema_init"], fx["live_states"][0]
    keys = [k for k, v in ema.items() if v.is_floating_point()]
    flat = E.ema_flat(torch.cat([ema[k].reshape(-1) for k in keys]), torch.cat([live[k].reshape(-1) for k in keys]), fx["momentum"])
    want = torch.cat([E.ema_state(ema, live, fx["momentum"])[k].reshape(-1) for k in keys])
    assert torch.equal(flat, want)


def test_metrics_restatement_matches_reference(fx):
    parts = []
    for b in fx["batches"]:
        p = E.cls_metrics(b["logits"], b["target"])
        n = b["target"].shape[0]
        assert p["n"] == n
        assert p["loss_sum"] / n == pytest.approx(b["loss"], rel=1e-6)
        assert 100.0 * p["top1"] / n == pytest.approx(b["top1"], rel=1e-6)
        assert 100.0 * p["top5"] / n == pytest.approx(b["top5"], rel=1e-6)
        parts.append(p)
    got = E.summarize(parts)
    assert [b["target"].shape[0] for b in fx["batches"]][-1] < fx["batches"][0]["target"].shape[0], "the last batch must be ragged"
    for k in ("loss", "top1", "top5"):
        assert got[k] == pytest.approx(fx["val"][k], rel=1e-6), k
    assert 0 < got["top1"] < got["top5"] < 100


def test_metrics_skip_ignored_rows(fx):
    b = fx["batches"][0]
    t = b["target"].clone()
    t[::3] = -1
    p = E.cls_metrics(b["logits"], t)
    q = E.cls_metrics(b["logits"][t != -1], b["target"][t != -1])
    assert p == q and p["n"] == int((t != -1).sum())


def test_rank_rule_counts_ties_for_the_target():
    """fewer than k classes strictly above: a tie at the k-th place is a hit; one more class above it is a miss"""
    row = torch.tensor([[5.0, 5.0, 4.0, 4.0, 4.0, 4.0, 4.0, 1.0]])
    assert E.cls_metrics(row, torch.tensor([1]))["top1"] == 1  # tied with class 0 for the first place
    assert E.cls_metrics(row, torch.tensor([6]))["top5"] == 1  # two classes above, four tied with it
    assert E.cls_metrics(row, torch.tensor([7]))["top5"] == 0  # seven above
    few = torch.tensor([[0.0, 3.0, 1.0]])
    assert E.cls_metrics(few, torch.tensor([0]))["top5"] == 1  # fewer than five classes: every counted row is a top-5 hit


def test_header_declares_the_validation_entry_points():
    hdr = open(os.path.join(REPO, "include", "cvnets_b200.h")).read()
    for name in ("cvb_cls_metrics", "cvb_ema_update"):
        assert re.search(r"CVB_API\s+int\s+" + name + r"\s*\(", hdr), name
    from ml_cvnets_b200 import _lib
    assert "cvb_cls_metrics" in _lib.EXPORTS and "cvb_ema_update" in _lib.EXPORTS
    import ctypes
    assert _lib._PROTOTYPES["cvb_ema_update"][1][3] is ctypes.c_double


def test_wrappers_reject_bad_arguments_before_launching():
    from ml_cvnets_b200 import ops
    logits = torch.zeros(4, 10, dtype=torch.bfloat16)
    y = torch.zeros(4, dtype=torch.int64)
    acc, cnt = torch.zeros(1, dtype=torch.float64), torch.zeros(3, dtype=torch.int64)
    scratch, ticket = torch.zeros(4), torch.zeros(1, dtype=torch.int32)
    with pytest.raises(ValueError, match="logits"):
        ops.cls_metrics(logits.float(), y, acc, cnt, scratch, ticket)
    with pytest.raises(ValueError, match="target"):
        ops.cls_metrics(logits, y.int(), acc, cnt, scratch, ticket)
    with pytest.raises(ValueError, match="loss_sum"):
        ops.cls_metrics(logits, y, acc.float(), cnt, scratch, ticket)
    with pytest.raises(ValueError, match="row_loss"):
        ops.cls_metrics(logits, y, acc, cnt, scratch[:3], ticket)
    with pytest.raises(ValueError, match="same size"):
        ops.ema_update(torch.zeros(4), torch.zeros(5), 0.1)
    with pytest.raises(ValueError, match="momentum"):
        ops.ema_update(torch.zeros(4), torch.zeros(4), 1.5)


def test_eval_step_and_ema_options_are_public():
    import inspect

    import ml_cvnets_b200 as m
    assert "EvalStep" in m.__all__
    sig = inspect.signature(m.TrainStep.__init__)
    assert sig.parameters["ema_buffers"].default is False
    for name in ("update", "capture", "compute", "reset"):
        assert callable(getattr(m.EvalStep, name))

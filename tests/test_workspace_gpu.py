"""StepWorkspace arena planning (-m gpu): each module's slice of the step arena is planned from the record of what the module carved, a
call that outgrows its slice carves tensors of its own until the next eager step re-plans, and none of it changes a gradient bit."""
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import cvnets_oracle as O  # noqa: E402
from test_engine_gpu import _small_model  # noqa: E402

pytestmark = pytest.mark.gpu

RES = 128
SCALE = 65536.0  # TrainStep's initial loss scale: the flat gradients it leaves are scaled by it


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as m
    return m


@pytest.fixture
def own_carves(pkg, monkeypatch):
    """Records every carve that got a tensor of its own instead of a slice of the planned buffers."""
    from ml_cvnets_b200.workspace import Arena
    calls = []
    own = Arena._own

    def counting(n, like):
        calls.append(n)
        return own(n, like)

    monkeypatch.setattr(Arena, "_own", staticmethod(counting))
    return calls


def _batch(B):
    return O.seeded_input((B, 3, RES, RES), 20 + B).cuda(), (torch.arange(B, device="cuda") * 37) % 1000


def _check_plan(ws):
    """Every slice holds its record (rounded up to 32 bytes), and the slices tile the two buffers without overlap."""
    plan = list(ws._plan.values())
    assert any(rec[0] for rec, *_ in plan) and any(rec[1] for rec, *_ in plan)
    for rec, o32, n32, o64, n64 in plan:
        assert rec[0] <= n32 < rec[0] + 8 and rec[1] <= n64 < rec[1] + 4, (rec, n32, n64)
    for offs, total in (([(o, n) for _, o, n, _, _ in plan], ws._buf32.numel()), ([(o, n) for _, _, _, o, n in plan], ws._buf64.numel())):
        offs.sort()
        assert all(o + n <= o2 for (o, n), (o2, _) in zip(offs, offs[1:])) and offs[-1][0] + offs[-1][1] <= total


def test_planned_arena_holds_every_carve_from_the_second_step(pkg, own_carves):
    model = _small_model(pkg)
    ts = pkg.TrainStep(model, lr=0.0, weight_decay=0.0)
    x, y = _batch(16)
    counts = []
    for _ in range(3):
        own_carves.clear()
        ts.step(x, y)
        counts.append(len(own_carves))
    assert counts[0] > 0 and counts[1:] == [0, 0], counts
    _check_plan(ts.ws)


def test_batch_size_changes_replan_and_keep_gradients_bitwise(pkg, own_carves):
    """Up from 8 to 16 (the batch-sized carves outgrow their slices: own tensors, then a re-plan), down to 4 (fits the planned slices),
    back to 16: every step's gradients equal the plain autograd path's bit for bit."""
    model = _small_model(pkg)
    ts = pkg.TrainStep(model, lr=0.0, weight_decay=0.0)  # lr 0: parameters stay put, gradients can be compared after each step
    counts = []
    for it, B in enumerate((8, 16, 16, 4, 16)):
        x, y = _batch(B)
        own_carves.clear()
        ts.step(x, y)
        counts.append(len(own_carves))
        ref = _small_model(pkg)
        (pkg.cross_entropy(ref(x), y, label_smoothing=0.1) * SCALE).backward()
        bad = [k for (k, p), (_, q) in zip(model.named_parameters(), ref.named_parameters()) if not torch.equal(p.grad, q.grad)]
        assert not bad, f"step {it} (batch {B}): {len(bad)} workspace gradients differ from the autograd path's, e.g. {bad[:5]}"
    assert counts[0] > 0 and counts[1] > 0 and counts[2:] == [0, 0, 0], counts
    _check_plan(ts.ws)

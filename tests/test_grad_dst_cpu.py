"""functional._Dst on CPU tensors (no step workspace): gradient destinations are named by their parameter, never by a position in the
module's parameter list, and ``finish`` hands the gradients back in the order it is asked for."""
from types import SimpleNamespace

import pytest
import torch

from ml_cvnets_b200.functional import _Dst
from ml_cvnets_b200.ops import PreparedWeights as PW


def _params():
    g = torch.Generator().manual_seed(0)
    w = torch.nn.Parameter(torch.randn(4, 3, generator=g))
    gamma = torch.nn.Parameter(torch.randn(4, generator=g))
    beta = torch.nn.Parameter(torch.randn(4, generator=g))
    return w, gamma, beta


@pytest.mark.parametrize("order", [(0, 1, 2), (2, 0, 1), (1, 2, 0)])
def test_finish_returns_gradients_in_argument_order(order):
    w, gamma, beta = _params()
    D = _Dst(SimpleNamespace(), [(w, gamma, beta)[i] for i in order], "cpu", True)
    dw, dbeta = D.mat(w, 4, 3), D.mat(beta, 1, 4)
    dw.copy_(torch.arange(12.0).view(4, 3))
    dbeta.fill_(-1.0)
    gw, none, gbeta = D.finish(w, None, beta)
    assert none is None
    assert gw.shape == w.shape and gw.data_ptr() == dw.data_ptr() and torch.equal(gw, torch.arange(12.0).view(4, 3))
    assert gbeta.shape == beta.shape and gbeta.data_ptr() == dbeta.data_ptr() and torch.equal(gbeta, torch.full((4,), -1.0))


def test_padded_carve_returns_its_first_rows_in_the_parameter_shape():
    w, _, b = _params()  # w [4, 3] and b [4], as a classifier's weight and bias padded to 8 output rows
    D = _Dst(SimpleNamespace(), [w, b], "cpu", True)
    vw, vb = D.padded(w, 4, 3, 8), D.padded(b, 4, 1, 8)
    assert vw.shape == (8, 3) and vb.shape == (8, 1)
    vw.copy_(torch.arange(24.0).view(8, 3))
    vb.copy_(torch.arange(8.0).view(8, 1))
    gw, gb = D.finish(w, b)
    assert gw.shape == w.shape and gw.data_ptr() == vw.data_ptr() and torch.equal(gw, torch.arange(12.0).view(4, 3))
    assert gb.shape == b.shape and torch.equal(gb, torch.arange(4.0))


def test_late64_gradient_is_fp32_after_finish():
    _, gamma, beta = _params()
    cfg = SimpleNamespace()
    for _ in range(2):  # the first call's carve is a tensor of its own, the second is a slice of the arena's buffer
        D = _Dst(cfg, [gamma, beta], "cpu", True)
        cs = D.ar.f64(2, 4)
        cs.copy_(torch.tensor([[1.5, 2.0, 3.0, 4.0], [-1.0, -2.0, -3.0, -4.0]], dtype=torch.float64))
        D.late64(gamma, cs[1])
        D.late64(beta, cs[0])
        ggamma, gbeta = D.finish(gamma, beta)
        assert ggamma.dtype == gbeta.dtype == torch.float32 and ggamma.shape == gbeta.shape == (4,)
        assert torch.equal(ggamma, cs[1].float()) and torch.equal(gbeta, cs[0].float())


def test_parameter_not_in_plist_fails():
    w, gamma, beta = _params()
    D = _Dst(SimpleNamespace(), [w, gamma], "cpu", True)
    for stranger in (beta, w.detach(), torch.nn.Parameter(w.detach().clone())):  # same shape, or even the same values, is not enough
        with pytest.raises(AssertionError, match="not in the plist"):
            D.mat(stranger, 4, 3)
        with pytest.raises(AssertionError, match="not in the plist"):
            D.padded(stranger, 4, 3, 8)
        with pytest.raises(AssertionError, match="not in the plist"):
            D.late64(stranger, D.ar.f64(4))
        with pytest.raises(AssertionError, match="not in the plist"):
            D.unprep(stranger, D.ar.f32(4, 3), 4, 3, 3, PW.KIND_ROWMAJOR)
    with pytest.raises(AssertionError, match="not in the plist"):
        D.bn_bwd(None, 1, None, False, gamma, beta)


def test_duplicate_plist_entry_fails():
    w, gamma, beta = _params()
    with pytest.raises(AssertionError, match="appears twice"):
        _Dst(SimpleNamespace(), [w, gamma, beta, gamma], "cpu", True)

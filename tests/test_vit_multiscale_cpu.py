"""CPU checks for multi-scale ViT training: the oracle's ViT with interpolated positional embeddings (tests/vit_multiscale_ref.py) reproduces the
real reference at the sampler's crops (tests/golden/make_golden_vit_multiscale.py), and the library exports the interpolating token kernels
at ABI 12."""
import os
import re
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_sample import at_sample  # noqa: E402
from vit_multiscale_ref import vit_forward_any_size, vit_pos_embed  # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("crop", ["320x320", "128x128", "256x320"])
def test_oracle_vit_multiscale_fixture(golden_dir, crop):
    fx = torch.load(os.path.join(golden_dir, "vit_multiscale_fp32.pt"), weights_only=False)
    shapes = O.vit_shapes(fx["mode"])
    assert {k: list(v.shape) for k, v in shapes.items()} == {k: s for k, s in fx["keys"]}
    c = fx["crops"][crop]
    P = O.clone_params(O.seeded_fill_(shapes, fx["seed"]))
    x = O.seeded_input((2, 3) + tuple(c["size"]), c["x_seed"])
    logits = vit_forward_any_size(P, x, mode=fx["mode"], training=True)
    loss = F.cross_entropy(logits, c["labels"], label_smoothing=0.1)
    loss.backward()
    assert float((logits - c["logits"]).norm() / c["logits"].norm()) <= 2e-5
    assert abs(float(loss) - float(c["loss"])) <= 1e-5
    for k, n in c["grad_norms"].items():
        assert abs(float(P[k].grad.norm()) - n) <= 2e-3 * n + 1e-7, k
    for k, g in c["grads"].items():
        ours, g = at_sample(P[k].grad, g)
        assert float((ours - g).norm() / (g.norm() + 1e-12)) <= 5e-4, k


def test_positional_table_is_resized_only_when_needed():
    pe = torch.randn(1, 1, 196, 8)
    P = O.clone_params(O.seeded_fill_(O.vit_shapes("tiny", n_classes=10), 3), requires_grad=False)
    x = O.seeded_input((1, 3, 224, 224), 4)
    assert torch.equal(vit_forward_any_size(P, x, mode="tiny"), O.vit_forward(P, x, mode="tiny"))
    assert torch.equal(vit_pos_embed(pe, 196), pe.reshape(1, 196, 8))
    for n in (64, 320, 400):
        assert torch.equal(vit_pos_embed(pe, n), F.interpolate(pe, size=(n, 8), mode="bilinear").reshape(1, n, 8))


def test_abi_12_exports_interpolating_token_kernels():
    import __graft_entry__ as ge
    ge.build()
    from ml_cvnets_b200 import _lib
    lib = _lib.load()
    assert _lib.ABI_VERSION == 12 and lib.cvb_abi_version() == 12
    hdr = open(os.path.join(REPO, "include", "cvnets_b200.h")).read()
    for name in ("cvb_vit_tokens_interp_fwd", "cvb_vit_tokens_interp_bwd"):
        assert re.search(r"CVB_API\s+int\s+" + name + r"\s*\(", hdr), name
        assert name in _lib.EXPORTS and hasattr(lib, name), name

"""CPU checks for CLIP zero-shot evaluation: the fp32 restatement (tests/clip_zeroshot_ref.py) reproduces the real reference's class table,
zero-shot logits, top-k and 3-D text output (tests/golden/make_golden_clip_zeroshot.py); encoding a causal prefix equals full-length
encoding to fp32 rounding; the library exports the zero-shot kernels at ABI 11."""
import os
import re
import sys

import torch

from oracle import cvnets_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from clip_zeroshot_ref import image_features, text_features, text_projected, zero_shot_table  # noqa: E402

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
KW = dict(text_layers=4, text_heads=4)


def _fixture(golden_dir):
    fx = torch.load(os.path.join(golden_dir, "clip_zeroshot_fp32.pt"), weights_only=False)
    shapes = O.clip_shapes("small", proj=128, text_dim=256, text_layers=4, vocab=1000, ctx=16)
    return fx, O.clone_params(O.seeded_fill_(shapes, fx["seed"]), requires_grad=False)


def _rel(a, b):
    return float((a - b).norm() / b.norm())


def test_restatement_reproduces_reference_zero_shot(golden_dir):
    fx, P = _fixture(golden_dir)
    assert fx["split_gap"] <= 1e-6
    table = zero_shot_table(P, fx["tokens"], **KW)
    assert table.shape == (128, 12)
    assert _rel(table, fx["table"]) <= 1e-5 and _rel(table, fx["table_split5"]) <= 1e-5
    img = image_features(P, O.seeded_input((8, 3, 224, 224), fx["x_seed"]))
    logits = 100.0 * img @ table
    assert _rel(logits, fx["zero_shot_image_logits"]) <= 1e-5
    pred = logits.topk(5, 1, True, True).indices
    hit = pred.eq(fx["labels"].view(-1, 1))
    assert 100.0 * float(hit[:, :1].sum()) / 8 == fx["top1"] and 100.0 * float(hit.sum()) / 8 == fx["top5"]


def test_restatement_reproduces_reference_3d_batch(golden_dir):
    fx, P = _fixture(golden_dir)
    out = text_features(P, fx["tokens_3d"], **KW)
    assert out.shape == (3, 2, 128)
    assert _rel(out, fx["text_3d"]) <= 1e-5


def test_causal_prefix_equals_full_length(golden_dir):
    """The end-of-text feature of a causal text tower depends only on tokens 0..eot: running a row at any prefix that contains its
    end-of-text token gives the full-length result up to fp32 rounding."""
    fx, P = _fixture(golden_dir)
    rows = fx["tokens"][0].reshape(-1, 16)
    full = text_projected(P, rows, **KW)
    eot = rows.argmax(dim=-1)
    for Lp in (8, 12, 16):
        sel = eot < Lp
        assert int(sel.sum()) > 0
        pre = text_projected(P, rows[sel], length=Lp, **KW)
        assert float((pre - full[sel]).abs().max()) <= 1e-5 * float(full.abs().max()), Lp
    exact = torch.stack([text_projected(P, rows[i:i + 1], length=int(eot[i]) + 1, **KW)[0] for i in range(rows.shape[0])])
    assert _rel(exact, full) <= 1e-6


def test_abi_11_exports_zero_shot_kernels():
    import __graft_entry__ as ge
    ge.build()
    from ml_cvnets_b200 import _lib
    lib = _lib.load()
    assert _lib.ABI_VERSION == 11 and lib.cvb_abi_version() == 11
    hdr = open(os.path.join(REPO, "include", "cvnets_b200.h")).read()
    for name in ("cvb_zs_class_embed", "cvb_zs_logits_topk"):
        assert re.search(r"CVB_API\s+int\s+" + name + r"\s*\(", hdr), name
        assert name in _lib.EXPORTS and hasattr(lib, name), name

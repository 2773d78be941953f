"""MobileViT-v1 at the variable-batch sampler's crops (160 - 320 px), CPU only.

Pins the resize-aware oracle (tests/mit_multiscale_ref.py) to the real reference's fixtures (tests/golden/make_golden_mit_multiscale.py),
checks the recipe's (crop, batch) table, and that every MobileViTBlock of XXS, XS and S at every pair it trains on reaches an attention
kernel whose shared memory holds the sequence (ops.mha_max_seq, a restatement of csrc/mha.cu's budget)."""
import os

import pytest
import torch
import torch.nn.functional as F

from mit_multiscale_ref import FIXTURES, PATCH, RECIPE_PAIRS, S_PAIRS, blocks, fixture_name, fold, mobilevit_v1_forward, unfold
from oracle import cvnets_oracle as O
from test_oracle_golden import _noise_floor

MODE_PAIRS = {"xx_small": RECIPE_PAIRS, "x_small": RECIPE_PAIRS, "small": S_PAIRS}


def test_recipe_pairs():
    """the sampler of config/classification/imagenet/mobilevit.yaml: crop 256, batch 128, 5 scales from 160 to 320, check_scale 32"""
    import ml_cvnets_b200 as m
    assert m.variable_batch_pairs(256, 256, 128, 5, 32, 160, 320, 160, 320) == [(c, c, b) for c, b in RECIPE_PAIRS]


def test_block_geometry():
    """layer 3 (stride 8) tokens and the layer-5 (stride 32) map of each pair; the maps that are not multiples of the patch"""
    assert [blocks("xx_small", c)[0][2] for c, _ in RECIPE_PAIRS] == [100, 144, 256, 324, 400]
    assert [blocks("xx_small", c)[2][1] for c, _ in RECIPE_PAIRS] == [5, 6, 8, 9, 10]
    odd = {(c, li) for c, _ in RECIPE_PAIRS for li, H, *_ in blocks("xx_small", c) if H % PATCH}
    assert odd == {(160, 5), (288, 5)}


@pytest.mark.parametrize("mode", sorted(MODE_PAIRS))
def test_attention_fits_at_every_pair(mode):
    """each block's sequence fits the shared memory of the kernel its head dim routes to, forward and backward; the recipes' head dims at
    layer 3 are 16 / 24 / 36 and reach 400 tokens at 320 px"""
    from ml_cvnets_b200 import ops
    seen = set()
    for crop, _ in MODE_PAIRS[mode]:
        for li, H, N, d, hd in blocks(mode, crop):
            assert N != d, (mode, crop, li)
            assert hd != 64
            assert N <= ops.mha_max_seq(hd, backward=True) <= ops.mha_max_seq(hd, backward=False), (mode, crop, li, hd, N)
            seen.add((hd, N))
    assert max(N for _, N in seen) == 400
    assert {hd for hd, N in seen if N == 400} == {"xx_small": {16}, "x_small": {24}, "small": {36}}[mode]


def test_small_at_192_collides():
    """MobileViT-S at 192 px: 144 tokens of width 144 in layer 3 (the refusal the S table drops the pair for)"""
    li, H, N, d, hd = blocks("small", 192)[0]
    assert (li, N, d) == (3, 144, 144)


def test_mha_limits():
    """the shared-memory limits of the mma.sync attention kernels: S <= 1152 / 704 / 448 / 384 at padded head dims 16 / 32 / 48 / 64"""
    from ml_cvnets_b200 import ops
    assert [ops.mha_max_seq(hd) for hd in (2, 16, 18, 32, 34, 36, 48, 50, 62)] == [1152, 1152, 704, 704, 448, 448, 448, 384, 384]
    assert ops.mha_max_seq(64) is None


def test_unfold_fold_identity_at_multiples():
    """at multiples of the patch the resize-aware unfold / fold are the oracle's reshapes and invert each other exactly"""
    fm = torch.randn(2, 24, 8, 6)
    t, info = unfold(fm)
    assert t.shape == (2 * PATCH * PATCH, 12, 24)
    assert torch.equal(fold(t, info), fm)
    t5, info5 = unfold(torch.randn(2, 24, 5, 7))
    assert t5.shape == (8, 12, 24) and info5[4:] == (6, 8)
    assert fold(t5, info5).shape == (2, 24, 5, 7)


@pytest.mark.parametrize("mode,crop", FIXTURES)
def test_oracle_matches_reference(golden_dir, mode, crop):
    """eval forward at 1 x crop^2 and a train-mode forward / backward at batch 2: the tolerances of test_mobilevit_v1_modes_cpu.py"""
    from golden_sample import at_sample
    fx = torch.load(os.path.join(golden_dir, fixture_name(mode, crop)), weights_only=False)
    assert fx["mode"] == mode and fx["res"] == crop
    shapes = O.mobilevit_v1_shapes(mode)
    assert {k: list(v.shape) for k, v in shapes.items()} == {k: s for k, s in fx["keys"]}
    P = O.clone_params(O.seeded_fill_(shapes, fx["seed"]))
    with torch.no_grad():
        ev = mobilevit_v1_forward(P, O.seeded_input((1, 3, crop, crop), fx["eval_x_seed"]), mode=mode, training=False)
    assert float((ev - fx["eval_logits"]).norm() / fx["eval_logits"].norm()) <= 2e-5
    logits = mobilevit_v1_forward(P, O.seeded_input((fx["batch"], 3, crop, crop), fx["x_seed"]), mode=mode, training=True)
    loss = F.cross_entropy(logits, fx["labels"], label_smoothing=0.1)
    loss.backward()
    assert float((logits.detach() - fx["logits"]).norm() / fx["logits"].norm()) <= 5e-5
    assert abs(float(loss) - float(fx["loss"])) <= 1e-5
    assert fx["grad_norms"].keys() == {k for k, p in P.items() if p.requires_grad}
    for k, n in fx["grad_norms"].items():
        assert abs(float(P[k].grad.norm()) - n) <= 2e-3 * n + 1e-6, (k, float(P[k].grad.norm()), n)
    floor = _noise_floor(fx["grad_norms"].values())
    for k, g in fx["grads"].items():
        if fx["grad_norms"][k] < floor:
            assert float(P[k].grad.norm()) < 2 * floor, k
            continue
        ours, ref = at_sample(P[k].grad, g)
        assert float((ours - ref).norm() / (ref.norm() + 1e-12)) <= 2e-3, k


def test_fixture_sizes(golden_dir):
    for mode, crop in FIXTURES:
        assert os.path.getsize(os.path.join(golden_dir, fixture_name(mode, crop))) < 1 << 20

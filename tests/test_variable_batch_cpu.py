"""engine.variable_batch_pairs against the reference's variable-batch sampler: the (h, w, batch) table of every ``sampler.vbs`` block in the
recipes this library trains (tests/golden/variable_batch_pairs.json, written by tests/golden/make_golden_variable_batch.py)."""
import json
import os

import pytest

with open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "variable_batch_pairs.json")) as _f:
    TABLES = json.load(_f)


@pytest.mark.parametrize("entry", TABLES, ids=[t["recipe"] for t in TABLES])
def test_variable_batch_pairs_match_reference_sampler(entry):
    from ml_cvnets_b200 import variable_batch_pairs
    assert variable_batch_pairs(**entry["args"]) == [tuple(p) for p in entry["pairs"]]


def test_fixture_covers_the_trained_recipes():
    names = {t["recipe"] for t in TABLES}
    for r in ("efficientnet_b0", "efficientnet_b1", "efficientnet_b2", "efficientnet_b3", "vit/classification/vit_base", "imagenet/vit.yaml",
              "clip/clip_vit_base", "clip/clip_vit_huge", "clip_finetune_imagenet/clip_vit_base", "clip_finetune_imagenet/clip_vit_huge",
              "multi_modal_img_text/clip_vit"):
        assert any(r in n for n in names), r


def test_defaults_are_the_reference_samplers():
    """max_scales 5, check_scale 32 and crops 160..320 are image_batch_pairs' defaults; a base crop already on the grid is not doubled."""
    from ml_cvnets_b200 import variable_batch_pairs
    assert variable_batch_pairs(224, 224, 256) == [(160, 160, 501), (192, 192, 348), (224, 224, 256), (256, 256, 196), (288, 288, 154),
                                                   (320, 320, 125)]

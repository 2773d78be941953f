"""CPU checks for the ViT-H/16 recipes: the state_dict contract of VisionTransformer(mode="huge") and of the CLIP ViT-H/16 recipe model against
the real reference, and the oracle's ViT-H (tests/vit_multiscale_ref.py) against the reference's checkpointed ViT-H at 128 x 128
(tests/golden/make_golden_vit_huge.py)."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from golden_sample import at_sample  # noqa: E402
from vit_huge_ref import vit_huge_forward, vit_huge_shapes  # noqa: E402

AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True}


@pytest.fixture(scope="module")
def fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "vit_huge_fp32.pt"), weights_only=False)


def test_vit_huge_state_dict_matches_reference(fx):
    import ml_cvnets_b200 as m
    model = m.VisionTransformer(m.default_vit_opts("huge", **{"model.classification.gradient_checkpointing": True}))
    assert model.gradient_checkpointing and model.checkpoint_segments == fx["segments"]
    ours = [[k, list(v.shape)] for k, v in model.state_dict().items()]
    assert sorted(ours) == sorted(fx["keys"])
    assert {k: list(v.shape) for k, v in vit_huge_shapes().items()} == {k: s for k, s in fx["keys"]}


def test_clip_vit_huge_recipe_state_dict_matches_reference(fx):
    import ml_cvnets_b200 as m
    opts = m.default_clip_opts("huge", projection_dim=512, text_dim=768, text_layers=12, text_heads=12, **AUG,
                               **{"model.classification.gradient_checkpointing": True, "model.text.transformer.gradient_checkpoint": True})
    model = m.CLIP(opts)
    assert model.image_encoder.gradient_checkpointing and model.text_encoder.gradient_checkpoint
    ours = [[k, list(v.shape)] for k, v in model.state_dict().items()]
    assert sorted(ours) == sorted(fx["clip_keys"])


def test_checkpoint_segments_are_checked():
    import ml_cvnets_b200 as m
    with pytest.raises(ValueError, match="checkpoint_segments"):
        m.VisionTransformer(m.default_vit_opts("tiny", **{"model.classification.gradient_checkpointing": True,
                                                          "model.classification.vit.checkpoint_segments": 13}))


def test_oracle_reproduces_reference_vit_huge_at_128(fx):
    c = fx["crops"]["128x128"]
    P = O.clone_params(O.seeded_fill_(vit_huge_shapes(), fx["seed"]))
    x = O.seeded_input((2, 3) + tuple(c["size"]), c["x_seed"])
    logits = vit_huge_forward(P, x, training=True)
    loss = F.cross_entropy(logits, c["labels"], label_smoothing=0.1)
    loss.backward()
    assert float((logits - c["logits"]).norm() / c["logits"].norm()) <= 2e-5
    assert abs(float(loss) - float(c["loss"])) <= 1e-5
    for k, n in c["grad_norms"].items():
        assert abs(float(P[k].grad.norm()) - n) <= 2e-3 * n + 1e-7, k
    for k, g in c["grads"].items():
        ours, g = at_sample(P[k].grad, g)
        assert float((ours - g).norm() / (g.norm() + 1e-12)) <= 5e-4, k

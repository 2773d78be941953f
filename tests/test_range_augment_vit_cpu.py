"""RangeAugment on VisionTransformer / CLIP without a GPU, against the fixture generated from the real reference
(tests/golden/make_golden_range_augment_vit.py): the oracle composition -- tests/range_augment_ref.py's augmentor fed the reference's draws, then
the ViT / CLIP oracle, the cross entropy or the contrastive loss and the PSNR loss -- reproduces the reference's training step; the drop-in models
have the reference's state_dict keys in order and give the sampler parameters the reference's weight decay."""
import os

import pytest
import torch
import torch.nn.functional as F

import range_augment_ref as R
from golden_sample import at_sample
from ml_cvnets_b200 import CLIP, VisionTransformer, default_clip_opts, default_vit_opts
from ml_cvnets_b200.engine import cosine_curriculum
from oracle import cvnets_oracle as O
from vit_multiscale_ref import vit_forward_any_size

TOL = dict(atol=2e-5, rtol=2e-4)
AUG = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
       "model.learn_augmentation.noise": True, "model.learn_augmentation.lr_multiplier": 1.0}
CLIP_KW = dict(projection_dim=64, text_dim=128, text_layers=2, text_heads=4, vocab_size=1000, context_length=16)


@pytest.fixture(scope="module")
def fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "range_augment_vit_fp32.pt"), weights_only=False)


def _image(f):
    """The generator's input image (make_golden_range_augment.image): uniform in [0, 1] with exact 0 and 1 pixels."""
    x = torch.rand(*f["x_shape"], generator=torch.Generator().manual_seed(f["x_seed"]))
    x[0, 0, :2] = 0.0
    x[0, 1, :2] = 1.0
    assert float(x.double().sum()) == pytest.approx(f["x_sum"], rel=1e-12)
    return x


def _target(fx):
    start, end = fx["target"]
    return float(cosine_curriculum(R.psnr_to_mse(start), R.psnr_to_mse(end), fx["period"])[fx["epoch"]])


def _check_grads(ours, ref):
    for k, g in ours.items():
        torch.testing.assert_close(g, ref[k], atol=2e-5 * max(1.0, float(ref[k].abs().max())), rtol=2e-3, msg=lambda m, k=k: f"{k}: {m}")


def test_vit_oracle_matches_reference(fx):
    f = fx["vit"]
    x = _image(f)
    P = O.seeded_fill_(O.vit_shapes(f["mode"], n_classes=10), f["seed"])
    P.update(R.seeded_aug_params(f["aug_seed"]))
    Pc = O.clone_params(P)
    x_aug = R.augment(x, R.raw_from(Pc), f["draws"])
    torch.testing.assert_close(*at_sample(x_aug, f["x_aug"]), **TOL)
    logits = vit_forward_any_size(Pc, x_aug, mode=f["mode"])
    torch.testing.assert_close(logits, f["logits"], atol=1e-4, rtol=1e-3)
    ce = F.cross_entropy(logits, f["y"], label_smoothing=0.1)
    na = R.na_loss(x_aug, x, _target(fx))
    torch.testing.assert_close(ce, f["ce"], **TOL)
    torch.testing.assert_close(na, f["na"], **TOL)
    names = list(f["grads"])
    _check_grads(dict(zip(names, torch.autograd.grad(ce + na, [Pc[k] for k in names]))), f["grads"])


def test_clip_oracle_matches_reference(fx):
    f = fx["clip"]
    x = _image(f)
    P = O.seeded_fill_(O.clip_shapes(f["vit_mode"], proj=64, text_dim=128, text_layers=2, vocab=1000, ctx=16), f["seed"])
    P.update({"image_encoder." + k: v for k, v in R.seeded_aug_params(f["aug_seed"]).items()})
    Pc = O.clone_params(P)
    raw = R.raw_from({k[len("image_encoder."):]: v for k, v in Pc.items() if k.startswith("image_encoder.neural_augmentor.")})
    x_aug = R.augment(x, raw, f["draws"])
    torch.testing.assert_close(*at_sample(x_aug, f["x_aug"]), **TOL)
    img, txt = O.clip_forward(Pc, x_aug, f["tokens"], vit_mode=f["vit_mode"], text_layers=2, text_heads=4)
    torch.testing.assert_close(img, f["image"], atol=1e-5, rtol=1e-3)
    torch.testing.assert_close(txt, f["text"], atol=1e-5, rtol=1e-3)
    torch.testing.assert_close(torch.clamp(Pc["logit_scale"].exp(), 0, 100.0), f["logit_scale"], **TOL)
    loss = O.clip_loss(img, txt, Pc["logit_scale"])
    na = R.na_loss(x_aug, x, _target(fx))
    torch.testing.assert_close(loss, f["clip_loss"], **TOL)
    torch.testing.assert_close(na, f["na"], **TOL)
    names = list(f["grads"])
    _check_grads(dict(zip(names, torch.autograd.grad(loss + na, [Pc[k] for k in names]))), f["grads"])


def test_vit_keys_and_decay_match_reference(fx):
    f = fx["vit"]
    model = VisionTransformer(default_vit_opts(f["mode"], n_classes=10, **AUG))
    assert [(k, tuple(v.shape)) for k, v in model.state_dict().items()] == [tuple(kv) for kv in f["state_dict_keys"]]
    groups, _ = model.get_trainable_parameters(weight_decay=0.05, no_decay_bn_filter_bias=True)
    decay = {id(p): g["weight_decay"] for g in groups for p in g["params"]}
    params = dict(model.named_parameters())
    assert set(f["decay"]) == set(R.AUG_KEYS)
    for k, wd in f["decay"].items():
        assert decay[id(params[k])] == wd, k
    plain = list(VisionTransformer(default_vit_opts(f["mode"], n_classes=10)).state_dict())
    assert plain == [k for k in model.state_dict() if "neural_augmentor." not in k]


def test_clip_keys_and_decay_match_reference(fx):
    f = fx["clip"]
    model = CLIP(default_clip_opts(f["vit_mode"], **CLIP_KW, **AUG))
    assert [(k, tuple(v.shape)) for k, v in model.state_dict().items()] == [tuple(kv) for kv in f["state_dict_keys"]]
    params = dict(model.named_parameters())
    assert set(f["decay"]) == {"image_encoder." + k for k in R.AUG_KEYS}
    for k, wd in f["decay"].items():
        # the flat optimizers exempt exactly the 1-D parameters from weight decay (optim.py), as the reference's parameter_list does
        assert wd == 0.05 and params[k].dim() != 1, k
    groups, _ = model.image_encoder.get_trainable_parameters(weight_decay=0.05, no_decay_bn_filter_bias=True)
    decayed = {id(p) for g in groups if g["weight_decay"] > 0 for p in g["params"]}
    assert all(id(p) in decayed for p in model.image_encoder.neural_augmentor.parameters())
    plain = list(CLIP(default_clip_opts(f["vit_mode"], **CLIP_KW)).state_dict())
    assert plain == [k for k in model.state_dict() if "neural_augmentor." not in k]


def test_basic_mode_raises():
    with pytest.raises(NotImplementedError, match="basic"):
        VisionTransformer(default_vit_opts("tiny", n_classes=10, **{**AUG, "model.learn_augmentation.mode": "basic"}))

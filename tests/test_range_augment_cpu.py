"""RangeAugment without a GPU: the fp32 restatement (tests/range_augment_ref.py), fed the draws the reference made, against the fixture generated
from the real reference (tests/golden/make_golden_range_augment.py); the curriculum tables; the modules' state_dict contract; the options that
are out of scope."""
import os

import pytest
import torch

import range_augment_ref as R
from ml_cvnets_b200 import (DistributionNeuralAugmentor, EfficientNet, FlatSGD, MobileViT, MobileViTv2, NeuralAugmentationLoss, StepWorkspace,  # noqa: F401
                            build_neural_augmentor, default_opts)
from ml_cvnets_b200.engine import cosine_curriculum, linear_curriculum
from ml_cvnets_b200.models_effnet import default_effnet_opts
from ml_cvnets_b200.models_mit import default_mit_opts

TOL = dict(atol=2e-5, rtol=2e-4)


@pytest.fixture(scope="module")
def fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "range_augment_fp32.pt"), weights_only=False)


def _raw(rec, requires_grad=False):
    out = {}
    for name in R.NAMES:
        if rec["flags"][name]:
            out[name] = tuple(rec["raw"][f"{name}._{s}"].clone().requires_grad_(requires_grad) for s in ("low", "high"))
    return out


def test_fixture_covers_the_hard_cases(fx):
    orders = [t["draws"]["order"] for t in fx["trials"]]
    assert any(o.index("noise") < o.index("contrast") for o in orders if "contrast" in o), "no trial puts noise before contrast"
    assert any(len(o) == 2 for o in orders)
    assert any(t["x"].shape[0] % 2 for t in fx["trials"])


@pytest.mark.parametrize("trial", range(8))
def test_oracle_matches_reference(fx, trial):
    rec = fx["trials"][trial]
    raw = _raw(rec, requires_grad=True)
    x = rec["x"]
    y = R.augment(x, raw, rec["draws"])
    torch.testing.assert_close(y, rec["x_aug"], **TOL)
    for epoch, ref in rec["loss"].items():
        t = cosine_curriculum(R.psnr_to_mse(40), R.psnr_to_mse(10), 10)
        target = float(t[min(epoch, len(t) - 1)])
        torch.testing.assert_close(R.na_loss(y, x, target), ref, **TOL)
    t4 = float(cosine_curriculum(R.psnr_to_mse(40), R.psnr_to_mse(10), 10)[4])
    total = R.na_loss(y, x, t4) + 1e-3 * (rec["w"] * y).sum()
    params = [p for name in R.NAMES if name in raw for p in raw[name]]
    grads = torch.autograd.grad(total, params)
    keys = [f"{name}._{s}" for name in R.NAMES if name in raw for s in ("low", "high")]
    for k, g in zip(keys, grads):
        torch.testing.assert_close(g, rec["grads"][k], atol=1e-5, rtol=1e-3, msg=lambda m, k=k: f"{k}: {m}")


def test_oracle_efficientnet_b0_with_augmentor_matches_reference(fx):
    """The reference's EfficientNet-b0 with the augmentor at 2 x 3 x 64 x 64: the restatement (tests/efficientnet_ref.py + range_augment_ref), fed
    the reference's draws, reproduces its logits, augmented image, composite loss and the augmentor's gradients."""
    import torch.nn.functional as F
    import efficientnet_ref as E
    from oracle import cvnets_oracle as O
    f = fx["effnet_b0_64"]
    P = O.seeded_fill_(E.efficientnet_shapes("b0"), f["seed"])
    P.update(R.seeded_aug_params(f["aug_seed"]))
    Pc = O.clone_params(P)
    x_aug = R.augment(f["x"], R.raw_from(Pc), f["draws"])
    torch.testing.assert_close(x_aug, f["x_aug"], **TOL)
    logits = E.efficientnet_forward(Pc, x_aug, mode="b0")
    torch.testing.assert_close(logits, f["logits"], atol=1e-4, rtol=1e-3)
    ce = F.cross_entropy(logits, f["y"], label_smoothing=0.1)
    na = R.na_loss(x_aug, f["x"], float(cosine_curriculum(R.psnr_to_mse(40), R.psnr_to_mse(10), 10)[4]))
    torch.testing.assert_close(ce, f["ce"], **TOL)
    torch.testing.assert_close(na, f["na"], **TOL)
    grads = torch.autograd.grad(ce + na, [Pc[k] for k in R.AUG_KEYS])
    for k, g in zip(R.AUG_KEYS, grads):
        torch.testing.assert_close(g, f["grads"][k], atol=2e-5, rtol=2e-3, msg=lambda m, k=k: f"{k}: {m}")


@pytest.mark.parametrize("method,fn", [("cosine", cosine_curriculum), ("linear", linear_curriculum)])
def test_curriculum_tables(fx, method, fn):
    for (m, start, end, per), ref in fx["curricula"].items():
        if m != method:
            continue
        ours = fn(R.psnr_to_mse(start), R.psnr_to_mse(end), per)
        torch.testing.assert_close(ours, ref, atol=0, rtol=1e-6)
        loss = NeuralAugmentationLoss(target_value=(start, end), curriculum_method=method, period=per)
        torch.testing.assert_close(loss.table, ref, atol=0, rtol=1e-6)
        assert loss.table.numel() == per + 1  # the step past the end uses the last entry (kernel: min(step, T - 1))


def _opts(kind, **aug):
    kv = {f"model.learn_augmentation.{k}": v for k, v in aug.items()}
    if kind == "efficientnet":
        return default_effnet_opts("b0", n_classes=10, **kv)
    if kind == "mobilevit":
        return default_mit_opts("xx_small", n_classes=10, **kv)
    return default_opts(1.0, n_classes=10, **kv)


MODELS = {"efficientnet": EfficientNet, "mobilevit": MobileViT, "mobilevit_v2": MobileViTv2}
AUG = dict(mode="distribution", brightness=True, contrast=True, noise=True, lr_multiplier=1.0)


@pytest.mark.parametrize("kind", list(MODELS))
def test_state_dict_keys_match_reference(fx, kind):
    m = MODELS[kind](_opts(kind, **AUG))
    ours = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
    ref = fx["state_dict_keys"][kind]
    assert ours[:6] == ref[:6]
    assert [k for k, _ in ours[:6]] == [f"neural_augmentor.{n}._{s}" for n in R.NAMES for s in ("low", "high")]
    # the rest is each model's own contract (its CPU tests); the augmentor only prepends its six keys
    plain = [(k, tuple(v.shape)) for k, v in MODELS[kind](_opts(kind)).state_dict().items()]
    assert ours[6:] == plain
    assert not any(k.startswith("neural_augmentor") for k, _ in plain)
    assert [n for n, _ in m.named_parameters()][:6] == [k for k, _ in ours[:6]]


def test_initial_values_and_bounds():
    aug = build_neural_augmentor(_opts("efficientnet", **AUG))
    assert isinstance(aug, DistributionNeuralAugmentor)
    assert float(aug.brightness._low) == 0.5 and float(aug.brightness._high) == 1.5
    assert float(aug.noise._low) == 0.0 and abs(float(aug.noise._high) - 0.1) < 1e-7
    assert (aug.contrast.min_fn.min_val, aug.contrast.min_fn.max_val, aug.contrast.max_fn.min_val, aug.contrast.max_fn.max_val) == (0.1, 0.9, 1.1, 10.0)
    assert (aug.noise.min_fn.min_val, aug.noise.min_fn.max_val, aug.noise.max_fn.min_val, aug.noise.max_fn.max_val) == (0.0, 0.00005, 0.0001, 1.0)
    lo, hi = R.low_high("brightness", aug.brightness._low, aug.brightness._high)
    torch.testing.assert_close(aug.brightness.low, lo)
    torch.testing.assert_close(aug.brightness.high, hi)
    assert build_neural_augmentor(_opts("efficientnet")) is None


def test_out_of_scope_options_raise():
    with pytest.raises(NotImplementedError, match="basic"):
        build_neural_augmentor(_opts("efficientnet", mode="basic", brightness=True))
    with pytest.raises(NotImplementedError, match="lr_multiplier"):
        build_neural_augmentor(_opts("efficientnet", **dict(AUG, lr_multiplier=0.5)))
    with pytest.raises(NotImplementedError, match="lr_multiplier"):
        EfficientNet(_opts("efficientnet", **dict(AUG, lr_multiplier=2.0)))


def test_zero_dim_sampler_parameters_get_weight_decay():
    """no_decay_bn_filter_bias exempts len(shape) == 1 only (cvnets/misc/common.py:122-176): the 0-dim _low / _high ARE decayed."""
    m = MobileViTv2(_opts("mobilevit_v2", **AUG))
    groups, _ = m.get_trainable_parameters(weight_decay=0.05, no_decay_bn_filter_bias=True)
    decayed = {id(p) for g in groups if g["weight_decay"] > 0 for p in g["params"]}
    aug = list(m.neural_augmentor.parameters())
    assert len(aug) == 6 and all(p.dim() == 0 for p in aug)
    assert all(id(p) in decayed for p in aug)
    # FlatSGD / FlatAdamW apply the same rule per element: test_range_augment_gpu.py::test_flat_optimizers_decay_sampler_parameters

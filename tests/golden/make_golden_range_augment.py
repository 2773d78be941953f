"""RangeAugment fixtures FROM THE REAL REFERENCE (cvnets/neural_augmentor, loss_fn/neural_augmentation.py); see make_golden.py for the method.

The reference's DistributionNeuralAugmentor runs on CPU with ``random.shuffle``, ``torch.randperm``, ``torch.rand`` and ``torch.randn_like``
wrapped to record what it drew; the fixture stores those draws with the augmented image, the PSNR loss at several curriculum positions and the
gradients of the six sampler parameters, so tests/range_augment_ref.py can be pinned to it with the same draws.  It also stores one training
forward / backward of the reference's EfficientNet-b0 with the augmentor at 2 x 3 x 64 x 64 (logits, augmented_tensor, composite loss, the
augmentor's gradients), the reference's curriculum tables and the ``state_dict`` keys of the three conv-stem classifiers built with
``model.learn_augmentation`` set.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_range_augment.py
"""
import copy
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import O, make_opts, torch  # noqa: E402
from make_golden_efficientnet import effnet_opts  # noqa: E402
import efficientnet_ref as E  # noqa: E402
import range_augment_ref as R  # noqa: E402
import torch.nn.functional as F  # noqa: E402

import cvnets.neural_augmentor.neural_aug as NA  # noqa: E402
from cvnets import get_model  # noqa: E402
from cvnets.models.classification.efficientnet import EfficientNet  # noqa: E402
from loss_fn.neural_augmentation import CURRICULUM_METHOD, NeuralAugmentation  # noqa: E402


AUG_FLAGS = {"model.learn_augmentation.mode": "distribution", "model.learn_augmentation.brightness": True, "model.learn_augmentation.contrast": True,
             "model.learn_augmentation.noise": True, "model.learn_augmentation.lr_multiplier": 1.0}


def aug_opts(**flags):
    opts = copy.deepcopy(make_opts(1.0))
    setattr(opts, "model.learn_augmentation.mode", "distribution")
    for name in ("brightness", "contrast", "noise"):
        setattr(opts, f"model.learn_augmentation.{name}", flags.get(name, True))
    setattr(opts, "model.learn_augmentation.lr_multiplier", 1.0)
    return opts


def recorded_forward(aug, x):
    """Run the reference augmentor, returning (x_aug, draws) with draws in tests/range_augment_ref.py's layout."""
    log = {"order": None, "perm": [], "rand": [], "randn": []}
    real_shuffle, real_randperm, real_rand, real_randn_like = NA.random.shuffle, torch.randperm, torch.rand, torch.randn_like

    def shuffle(seq):
        real_shuffle(seq)
        log["order"] = [f.__name__[len("_apply_"):] for f in seq]

    def randperm(*a, **k):
        r = real_randperm(*a, **k)
        log["perm"].append(r.clone())
        return r

    def rand(*a, **k):
        r = real_rand(*a, **k)
        log["rand"].append(r.clone())
        return r

    def randn_like(*a, **k):
        r = real_randn_like(*a, **k)
        log["randn"].append(r.clone())
        return r

    NA.random.shuffle, torch.randperm, torch.rand, torch.randn_like = shuffle, randperm, rand, randn_like
    try:
        y = aug(x)
    finally:
        NA.random.shuffle, torch.randperm, torch.rand, torch.randn_like = real_shuffle, real_randperm, real_rand, real_randn_like
    n = max(1, x.shape[0] // 2)
    draws = {"order": log["order"]}
    for i, name in enumerate(log["order"]):
        draws[name] = {"idx": log["perm"][i][:n], "u": log["rand"][i].flatten()}
    if "noise" in draws:
        draws["noise"]["eps"] = log["randn"][0]
    return y, draws


def loss_opts(period, method="cosine", target=(40, 10)):
    opts = aug_opts()
    setattr(opts, "loss.neural_augmentation.perceptual_metric", "psnr")
    setattr(opts, "loss.neural_augmentation.target_value", list(target))
    setattr(opts, "loss.neural_augmentation.curriculum_method", method)
    setattr(opts, "loss.neural_augmentation.alpha", 100.0)
    setattr(opts, "scheduler.max_epochs", period)
    setattr(opts, "scheduler.is_iteration_based", False)
    return opts


def image(B, H, W, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(B, 3, H, W, generator=g)
    x[0, 0, :2] = 0.0  # exact 0 and 1 pixels: the clip passes their gradient (torch.clamp's inclusive bounds)
    x[0, 1, :2] = 1.0
    return x


def main():
    torch.manual_seed(0)
    fx = {"trials": [], "curricula": {}, "state_dict_keys": {}}
    period = 10
    crit = NeuralAugmentation(loss_opts(period))
    for trial in range(8):
        flags = {"brightness": True, "contrast": True, "noise": True}
        if trial == 6:
            flags["contrast"] = False
        B = 5 if trial % 2 else 6
        torch.manual_seed(1000 + trial)
        aug = NA.build_neural_augmentor(aug_opts(**flags))
        with torch.no_grad():  # trained-looking sampler parameters, not just the initial values
            for p in aug.parameters():
                p.add_(0.3 * torch.randn(()))
        x = image(B, 12, 16, 2000 + trial)
        y, draws = recorded_forward(aug, x)
        w = torch.randn(y.shape, generator=torch.Generator().manual_seed(3000 + trial))
        rec = {"x": x, "flags": flags, "raw": {k: v.detach().clone() for k, v in aug.state_dict().items()}, "draws": draws, "x_aug": y.detach().clone(),
               "loss": {}, "grads": {}}
        for epoch in (0, 4, period + 3):
            rec["loss"][epoch] = crit(x, {"augmented_tensor": y}, epoch=epoch).detach().clone()
        # gradient of L_na (epoch 4) plus a linear function of the augmented image (what the classifier's gradient looks like to the augmentor)
        total = crit(x, {"augmented_tensor": y}, epoch=4) + 1e-3 * (w * y).sum()
        grads = torch.autograd.grad(total, list(aug.parameters()))
        rec["w"] = w
        rec["grads"] = {k: g.clone() for (k, _), g in zip(aug.named_parameters(), grads)}
        fx["trials"].append(rec)
        print(trial, draws["order"], float(rec["loss"][4]), [float(g) for g in grads])
    # EfficientNet-b0 with the augmentor, 2 x 3 x 64 x 64, one training forward / backward of the composite loss (CE, label smoothing 0.1, +
    # the NA loss at epoch 4 of a 10-epoch cosine curriculum), seeded parameters (oracle.seeded_fill_ 81 + range_augment_ref.seeded_aug_params 82)
    opts = effnet_opts("b0")
    for k, v in AUG_FLAGS.items():
        setattr(opts, k, v)
    model = EfficientNet(opts).train()
    P = O.seeded_fill_(E.efficientnet_shapes("b0"), 81)
    P.update(R.seeded_aug_params(82))
    assert list(model.state_dict())[:6] == R.AUG_KEYS
    model.load_state_dict(P, strict=True)
    x = image(2, 64, 64, 181)
    yl = torch.tensor([3, 7])
    torch.manual_seed(5)
    out, draws = recorded_forward(model, x)
    ce = F.cross_entropy(out["logits"], yl, label_smoothing=0.1)
    na = crit(x, out, epoch=4)
    loss = ce + na
    aug_params = list(model.neural_augmentor.parameters())
    grads = torch.autograd.grad(loss, aug_params)
    fx["effnet_b0_64"] = {"x": x, "y": yl, "seed": 81, "aug_seed": 82, "draws": draws, "logits": out["logits"].detach().clone(),
                          "x_aug": out["augmented_tensor"].detach().clone(), "ce": ce.detach(), "na": na.detach(), "loss": loss.detach(),
                          "grads": {k: g.clone() for k, g in zip(R.AUG_KEYS, grads)}}
    print("effnet_b0_64", draws["order"], float(loss), [float(g) for g in grads])
    for method, fn in CURRICULUM_METHOD.items():
        for (start, end, per) in ((40, 10, 400), (40, 20, 7)):
            s_mse = 10.0 ** ((20.0 * torch.log10(torch.tensor(255.0, dtype=torch.float64)).item() - start) / 10.0)
            e_mse = 10.0 ** ((20.0 * torch.log10(torch.tensor(255.0, dtype=torch.float64)).item() - end) / 10.0)
            fx["curricula"][(method, start, end, per)] = fn(start=s_mse, end=e_mse, period=per)
    for name in ("mobilevit_v2", "mobilevit", "efficientnet"):
        opts = aug_opts()
        setattr(opts, "model.classification.name", name)
        setattr(opts, "model.classification.n_classes", 10)
        if name == "mobilevit":
            setattr(opts, "model.classification.mit.mode", "xx_small")
        if name == "efficientnet":
            setattr(opts, "model.classification.efficientnet.mode", "b0")
        m = get_model(opts)
        fx["state_dict_keys"][name] = [(k, tuple(v.shape)) for k, v in m.state_dict().items()]
        print(name, fx["state_dict_keys"][name][:8])
    torch.save(fx, os.path.join(HERE, "range_augment_fp32.pt"))


if __name__ == "__main__":
    main()

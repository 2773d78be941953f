"""Gradient-accumulation fixture FROM THE REAL REFERENCE (see make_golden.py for the method): EfficientNet-b0 (16 classes, no stochastic
depth, no classifier dropout) trained on the CPU in fp32 for two accumulation windows of ``common.accum_freq`` 2, micro-batches of 8 images
at 64 x 64, with the reference's SGD (optim/sgd.py: momentum 0.9, Nesterov, learning rate 0.005, weight decay 4e-5 on the parameter groups of
``get_trainable_parameters(no_decay_bn_filter_bias=True)``, built by ``optim.build_optimizer``), its label-smoothed ``CrossEntropy`` (0.1),
its ``EMA`` of the whole state (cvnets/misc/averaging_utils.py, momentum 0.1 so that two updates move it visibly) and a GradScaler that is
disabled, as the reference's is without mixed precision.

``Trainer.train_epoch`` needs a full option set, a data loader with ``samples_in_dataset``, log writers and checkpointing, so its loop is
restated here line by line (engine/training_engine.py; the learning-rate scheduler is constant and left out):
  :225  ``_zero_grad()`` at the start of the epoch
  :258  forward, :263  loss, :286  ``gradient_scaler.scale(loss).backward()`` on every batch (gradients are summed, the loss is not divided)
  :288  every ``accum_freq``-th batch: :304 ``gradient_scaler.step``, :306 ``update``, :308 ``_zero_grad()``, :312 ``model_ema.update_parameters``
(no ``common.grad_clip``: the EfficientNet recipes set none, so :289-295 do nothing).

Stored: the micro-batches' seeds, targets and losses; after every micro-batch the BatchNorm running statistics; after every window the
parameters, the momentum buffers and the floating-point entries of the EMA state_dict.  Each snapshot is ONE fp32 vector: per tensor, in
the order of its key list, at most 32 elements at the evenly strided positions of golden_sample.py (``flat_sample``).

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_accum.py
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import O, load_seeded, torch  # noqa: E402
from make_golden_efficientnet import effnet_opts  # noqa: E402
import accum_ref as A  # noqa: E402
import efficientnet_ref as E  # noqa: E402

from cvnets.misc.averaging_utils import EMA  # noqa: E402
from cvnets.models.classification.efficientnet import EfficientNet  # noqa: E402
from loss_fn.classification.cross_entropy import CrossEntropy  # noqa: E402
from optim import build_optimizer  # noqa: E402

CFG = dict(mode="b0", n_classes=16, crop=64, batch=8, accum_freq=2, windows=2, lr=0.005, momentum=0.9, weight_decay=4e-5, label_smoothing=0.1,
           ema_momentum=0.1, param_seed=83, x_seeds=[401, 402, 403, 404], y_seed=405)


def main():
    torch.manual_seed(0)
    opts = effnet_opts(CFG["mode"])
    setattr(opts, "model.classification.n_classes", CFG["n_classes"])
    for k, v in {"optim.name": "sgd", "optim.weight_decay": CFG["weight_decay"], "optim.no_decay_bn_filter_bias": True,
                 "optim.sgd.momentum": CFG["momentum"], "optim.sgd.nesterov": True, "scheduler.lr": CFG["lr"]}.items():
        setattr(opts, k, v)
    model = EfficientNet(opts)
    load_seeded(model, E.efficientnet_shapes(CFG["mode"], CFG["n_classes"]), CFG["param_seed"])
    model.train()
    optimizer = build_optimizer(model, opts)
    scaler = torch.amp.GradScaler("cpu", enabled=False)
    lopts = CrossEntropy.add_arguments(argparse.ArgumentParser()).parse_args([])
    setattr(lopts, "loss.classification.cross_entropy.label_smoothing", CFG["label_smoothing"])
    criteria = CrossEntropy(lopts)
    criteria.train()
    ema = EMA(model, ema_momentum=CFG["ema_momentum"], device="cpu")
    g = torch.Generator().manual_seed(CFG["y_seed"])
    n_micro = CFG["accum_freq"] * CFG["windows"]
    targets = [torch.randint(0, CFG["n_classes"], (CFG["batch"],), generator=g) for _ in range(n_micro)]
    bn_keys = [k for k in model.state_dict() if k.endswith(("running_mean", "running_var"))]
    ema_keys = [k for k, v in model.state_dict().items() if v.is_floating_point()]

    optimizer.zero_grad()  # :225
    micro, windows, losses = [], [], []
    for batch_id in range(n_micro):
        x = O.seeded_input((CFG["batch"], 3, CFG["crop"], CFG["crop"]), CFG["x_seeds"][batch_id])
        pred = model(x)
        loss = criteria(input_sample=x, prediction=pred, target=targets[batch_id], epoch=0, iterations=len(windows))
        scaler.scale(loss).backward()
        losses.append(float(loss.detach()))
        sd = model.state_dict()
        micro.append(A.flat_sample([sd[k] for k in bn_keys]))
        if (batch_id + 1) % CFG["accum_freq"] == 0:
            scaler.step(optimizer=optimizer)
            scaler.update()
            optimizer.zero_grad()
            ema.update_parameters(model)
            params = [p for _, p in model.named_parameters()]
            esd = ema.ema_model.state_dict()
            windows.append(dict(params=A.flat_sample(params), momentum=A.flat_sample([optimizer.state[p]["momentum_buffer"] for p in params]),
                                ema=A.flat_sample([esd[k] for k in ema_keys])))
    fx = dict(cfg=CFG, targets=targets, losses=losses, bn_keys=bn_keys, param_keys=[k for k, _ in model.named_parameters()], ema_keys=ema_keys,
              micro=micro, windows=windows)
    out = os.path.join(HERE, "accum_fp32.pt")
    torch.save(fx, out)
    print(out, os.path.getsize(out), "bytes; losses", losses)


if __name__ == "__main__":
    main()

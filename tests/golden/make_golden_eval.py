"""Golden fixture FROM THE REAL REFERENCE for classification validation (see make_golden.py for the method).

  * EMA of the whole state: the reference's ``EMA`` (cvnets/misc/averaging_utils.py) at momentum 0.1 around an InvertedResidual 16 -> 16
    (expand 2: three conv + BatchNorm pairs), fed a seeded sequence of 5 live state_dicts (weights, running statistics and a growing
    ``num_batches_tracked``); the EMA state after every update.
  * Validation metrics: the reference's ``CrossEntropy`` in eval mode (label smoothing 0.1 configured, switched off by eval) and
    ``top_k_accuracy`` (metrics/topk_accuracy.py) on three batches of 100 classes, the last one ragged (64, 64, 37 rows; the target's rank
    drawn from 0..11), averaged over the rows as the reference's AverageMetric does (sum of batch value * batch size / rows).  The logits
    are distinct multiples of 1/8 per row, exactly representable in bf16, so the ranking has no ties in fp32 or in bf16.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_eval.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import O, load_seeded, make_opts, strip, torch  # noqa: E402

import argparse  # noqa: E402

from cvnets.misc.averaging_utils import EMA  # noqa: E402
from cvnets.modules import InvertedResidual  # noqa: E402
from loss_fn.classification.cross_entropy import CrossEntropy  # noqa: E402
from metrics.topk_accuracy import top_k_accuracy  # noqa: E402

MOMENTUM = 0.1
N_CLASSES = 100
BATCHES = (64, 64, 37)


def live_states(model, n, gen):
    """n seeded state_dicts of the model: weights and running statistics drawn afresh, the counter growing as training would."""
    out = []
    for i in range(n):
        sd = {}
        for k, v in model.state_dict().items():
            if v.is_floating_point():
                r = torch.randn(v.shape, generator=gen)
                sd[k] = r.abs() + 0.5 if k.endswith("running_var") else r
            else:
                sd[k] = torch.full_like(v, 3 * (i + 1))
        out.append(sd)
    return out


def main():
    torch.manual_seed(0)
    opts = make_opts(1.0)
    P = {}
    O.inverted_residual_shapes(P, "m", 16, 16, expand_ratio=2)
    model = InvertedResidual(opts, 16, 16, stride=1, expand_ratio=2)
    load_seeded(model, strip("m.", P), 91)
    gen = torch.Generator().manual_seed(92)
    ema = EMA(model, ema_momentum=MOMENTUM, device="cpu")
    init = {k: v.clone() for k, v in ema.ema_model.state_dict().items()}
    states = live_states(model, 5, gen)
    ema_states = []
    for sd in states:
        model.load_state_dict(sd, strict=True)
        ema.update_parameters(model)
        ema_states.append({k: v.clone() for k, v in ema.ema_model.state_dict().items()})

    p = CrossEntropy.add_arguments(argparse.ArgumentParser())
    lopts = p.parse_args([])
    setattr(lopts, "loss.classification.cross_entropy.label_smoothing", 0.1)
    loss_fn = CrossEntropy(lopts)
    loss_fn.eval()
    batches = []
    tot = {"loss": 0.0, "top1": 0.0, "top5": 0.0}
    for b in BATCHES:
        perm = torch.stack([torch.randperm(N_CLASSES, generator=gen) for _ in range(b)])
        logits = (perm.float() - N_CLASSES / 2) / 8.0
        rank = torch.randint(0, 12, (b,), generator=gen)  # the target's rank: about 1 in 12 top-1 and 5 in 12 top-5 hits
        target = (perm == (N_CLASSES - 1 - rank)[:, None]).float().argmax(1)
        with torch.no_grad():
            loss = float(loss_fn(None, logits, target))
            top1, top5 = (float(a) for a in top_k_accuracy(logits, target, top_k=(1, 5)))
        batches.append(dict(logits=logits, target=target, loss=loss, top1=top1, top5=top5))
        for k, v in (("loss", loss), ("top1", top1), ("top5", top5)):
            tot[k] += v * b
    n = sum(BATCHES)
    fx = dict(momentum=MOMENTUM, ema_init=init, live_states=states, ema_states=ema_states, batches=batches,
              val={k: v / n for k, v in tot.items()}, n_rows=n)
    out_path = os.path.join(HERE, "eval_fp32.pt")
    torch.save(fx, out_path)
    print(out_path, os.path.getsize(out_path), "bytes; val", fx["val"])


if __name__ == "__main__":
    main()

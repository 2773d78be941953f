"""Generate the MobileViT-v1 fixtures at the variable-batch sampler's other crops FROM THE REAL REFERENCE (apple/ml-cvnets @ /root/reference).

Runs only in the build container, like make_golden_mit_modes.py: it builds the reference's own ``get_model`` in each mode, loads the
deterministic parameters of ``oracle.cvnets_oracle.seeded_fill_``, runs one eval forward at 1 x 3 x crop x crop and one train-mode forward /
backward at batch 2, every dropout 0, label smoothing 0.1.  The (mode, crop) list is ``tests/mit_multiscale_ref.FIXTURES``:
  XXS at 160 and 288 (the 5x5 / 9x9 stride-32 maps the reference resizes to 6x6 / 10x10) and 320 (400 tokens at head_dim 16),
  XS at 320 (head_dim 24 at 400 tokens), S at 160 (the resize at width 240) and 320 (head_dim 36 at 400 tokens).
Gradients above KEEP elements are stored as a fixed sample (tests/golden_sample.py), so every file stays under 1 MB.
``tests/test_mobilevit_v1_multiscale_cpu.py`` pins tests/mit_multiscale_ref.py to these files; ``tests/test_mobilevit_v1_multiscale_gpu.py``
compares the CUDA path with them.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_mit_multiscale.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from golden_sample import sample_large  # noqa: E402
from make_golden import O, get_model, load_seeded  # noqa: E402  (puts the reference on sys.path, changes into its root)
from make_golden_mit_modes import mit_opts  # noqa: E402
from mit_multiscale_ref import FIXTURES, fixture_name  # noqa: E402

BATCH = 2
KEEP = 2048    # gradients with at most this many elements are stored whole
SAMPLE = 512   # elements kept of each larger gradient


def main():
    torch.manual_seed(0)
    for i, (mode, crop) in enumerate(FIXTURES):
        seed, eval_x_seed, x_seed = 91 + i, 481 + i, 491 + i
        model = get_model(mit_opts(mode))
        load_seeded(model, O.mobilevit_v1_shapes(mode), seed)
        model.eval()
        with torch.no_grad():
            eval_logits = model(O.seeded_input((1, 3, crop, crop), eval_x_seed)).clone()
        model.train()
        x = O.seeded_input((BATCH, 3, crop, crop), x_seed)
        labels = torch.tensor([11 + i, 980 - i])
        logits = model(x)
        loss = F.cross_entropy(logits, labels, label_smoothing=0.1)
        loss.backward()
        grads = {k: p.grad for k, p in model.named_parameters()}
        fx = dict(mode=mode, res=crop, batch=BATCH, seed=seed, eval_x_seed=eval_x_seed, eval_logits=eval_logits, x_seed=x_seed, labels=labels,
                  logits=logits.detach().clone(), loss=loss.detach().clone(), keys=[[k, list(v.shape)] for k, v in model.state_dict().items()],
                  grad_norms={k: float(g.norm()) for k, g in grads.items()},
                  grads={k: sample_large(g.clone(), limit=KEEP, n=SAMPLE) for k, g in grads.items()})
        fn = os.path.join(HERE, fixture_name(mode, crop))
        torch.save(fx, fn)
        print(os.path.basename(fn), os.path.getsize(fn), "bytes")


if __name__ == "__main__":
    main()

"""Generate the MobileViT-v1 fixtures of the two modes the recipes train that mobilevit_v1_xxs_fp32.pt does not hold (x_small, small) FROM THE
REAL REFERENCE (apple/ml-cvnets @ /root/reference).

Runs only in the build container, like make_golden.py: it builds the reference's own ``get_model`` in each mode, loads the deterministic
parameters of ``oracle.cvnets_oracle.seeded_fill_`` (asserting the state_dict key / shape contract), runs one eval forward at 1x3x256x256 and
one train-mode forward / backward at batch 2, 256x256, every dropout 0, label smoothing 0.1.  256x256 keeps every token count (256 / 64 / 16)
away from every transformer dim (96 - 240): where they are equal the reference's LayerNorm takes its channel-first branch (layer_norm.py:52-65,
e.g. MobileViT-S at 192x192 has N = d = 144 in layer 3), which the library refuses.  It stores the fields of mobilevit_v1_xxs_fp32.pt, one file
per mode (``fixture_name``); gradients above KEEP elements are stored as a fixed sample (tests/golden_sample.py) so that every file stays
under 1 MB.  It also writes ``state_dict_contract_mit.json``: the reference's state_dict keys, shapes and dtypes per mode.
``tests/test_mobilevit_v1_modes_cpu.py`` pins the oracle to these files; ``tests/test_mobilevit_v1_modes_gpu.py`` compares the CUDA path with them.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_mit_modes.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from golden_sample import sample_large  # noqa: E402
from make_golden import O, get_model, load_seeded, make_opts  # noqa: E402  (puts the reference on sys.path, changes into its root)

MODES = ("x_small", "small")
RES, BATCH = 256, 2
KEEP = 2048    # gradients with at most this many elements are stored whole
SAMPLE = 512   # elements kept of each larger gradient


def fixture_name(mode):
    return {"x_small": "mobilevit_v1_xs_fp32.pt", "small": "mobilevit_v1_s_fp32.pt"}[mode]


def mit_opts(mode):
    opts = make_opts(1.0)
    for k, v in {"model.classification.name": "mobilevit", "model.classification.mit.mode": mode, "model.classification.mit.dropout": 0.0,
                 "model.classification.mit.attn_dropout": 0.0, "model.classification.mit.ffn_dropout": 0.0,
                 "model.classification.classifier_dropout": 0.0, "model.classification.n_classes": 1000}.items():
        setattr(opts, k, v)
    return opts


def main():
    torch.manual_seed(0)
    contract = {}
    for i, mode in enumerate(MODES):
        seed, eval_x_seed, x_seed = 81 + i, 381 + i, 391 + i
        model = get_model(mit_opts(mode))
        contract[mode] = [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in model.state_dict().items()]
        load_seeded(model, O.mobilevit_v1_shapes(mode), seed)
        model.eval()
        with torch.no_grad():
            eval_logits = model(O.seeded_input((1, 3, RES, RES), eval_x_seed)).clone()
        model.train()
        x = O.seeded_input((BATCH, 3, RES, RES), x_seed)
        labels = torch.tensor([7 + i, 990 - i])
        logits = model(x)
        loss = F.cross_entropy(logits, labels, label_smoothing=0.1)
        loss.backward()
        grads = {k: p.grad for k, p in model.named_parameters()}
        fx = dict(mode=mode, res=RES, batch=BATCH, seed=seed, eval_x_seed=eval_x_seed, eval_logits=eval_logits, x_seed=x_seed, labels=labels,
                  logits=logits.detach().clone(), loss=loss.detach().clone(), keys=[[k, list(v.shape)] for k, v in model.state_dict().items()],
                  grad_norms={k: float(g.norm()) for k, g in grads.items()},
                  grads={k: sample_large(g.clone(), limit=KEEP, n=SAMPLE) for k, g in grads.items()})
        torch.save(fx, os.path.join(HERE, fixture_name(mode)))
    with open(os.path.join(HERE, "state_dict_contract_mit.json"), "w") as f:
        json.dump(contract, f)
    for fn in [fixture_name(m) for m in MODES] + ["state_dict_contract_mit.json"]:
        print(fn, os.path.getsize(os.path.join(HERE, fn)), "bytes")


if __name__ == "__main__":
    main()

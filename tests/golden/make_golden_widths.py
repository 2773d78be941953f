"""Generate the MobileViTv2 fixtures of the published widths that mobilevit_v2_fp32.pt does not hold (0.75, 1.25, 1.5, 1.75, 2.0) FROM THE
REAL REFERENCE (apple/ml-cvnets @ /root/reference).

Runs only in the build container, like make_golden.py: it builds the reference's own ``get_model`` at each width, loads the deterministic
parameters of ``oracle.cvnets_oracle.seeded_fill_`` (asserting the state_dict key / shape contract), runs one train-mode forward and backward
at batch 2, 128x128 (at 64x64 the layer-5 attention would see a single patch) with label smoothing 0.1, and stores the same fields as
mobilevit_v2_fp32.pt, one file per width (``fixture_name``; every file in this directory stays under 1 MB).
``tests/test_mobilevit_widths_cpu.py`` pins the oracle to these files; ``tests/test_mobilevit_widths_gpu.py`` compares the CUDA path with them.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_widths.py
"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

import torch  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from make_golden import O, get_model, load_seeded, make_opts  # noqa: E402  (puts the reference on sys.path, changes into its root)

WIDTHS = (0.75, 1.25, 1.5, 1.75, 2.0)
RES, BATCH = 128, 2
KEEP = 1024  # gradients and buffers with at most this many elements are stored whole


def fixture_name(width):
    return f"mobilevit_v2_w{width}_fp32.pt"


def main():
    torch.manual_seed(0)
    contract = {}
    for i, width in enumerate(WIDTHS):
        seed, x_seed = 41 + i, 341 + i
        model = get_model(make_opts(width))
        sd = model.state_dict()
        contract[str(width)] = [[k, list(v.shape), str(v.dtype).replace("torch.", "")] for k, v in sd.items()]
        load_seeded(model, O.mobilevit_v2_shapes(width), seed)
        model.train()
        x = O.seeded_input((BATCH, 3, RES, RES), x_seed)
        labels = torch.tensor([5 + i, 990 - i])
        stage_out = {}
        hooks = [getattr(model, name).register_forward_hook(lambda mod, inp, out, name=name: stage_out.__setitem__(name, out.detach().clone()))
                 for name in ["conv_1", "layer_1", "layer_2", "layer_3", "layer_4", "layer_5"]]
        logits = model(x)
        loss = F.cross_entropy(logits, labels, label_smoothing=0.1)
        loss.backward()
        for h in hooks:
            h.remove()
        grads = {k: p.grad for k, p in model.named_parameters()}
        fx = dict(
            width=width, res=RES, seed=seed, x_seed=x_seed, labels=labels,
            logits=logits.detach().clone(), loss=loss.detach().clone(),
            stage_norms={k: float(v.norm()) for k, v in stage_out.items()},
            stage_sample={k: v.flatten()[:: max(1, v.numel() // 512)][:512].clone() for k, v in stage_out.items()},
            grad_norms={k: float(g.norm()) for k, g in grads.items()},
            grad_small={k: g.clone() for k, g in grads.items() if g.numel() <= KEEP},
            buffers_after={k: b.detach().clone() for k, b in model.named_buffers() if b.numel() <= KEEP},
        )
        torch.save(fx, os.path.join(HERE, fixture_name(width)))
    with open(os.path.join(HERE, "state_dict_contract_widths.json"), "w") as f:
        json.dump(contract, f)
    for fn in [fixture_name(w) for w in WIDTHS] + ["state_dict_contract_widths.json"]:
        print(fn, os.path.getsize(os.path.join(HERE, fn)), "bytes")


if __name__ == "__main__":
    main()

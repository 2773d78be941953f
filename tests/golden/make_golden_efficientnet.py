"""EfficientNet fixtures FROM THE REAL REFERENCE (cvnets/modules/efficientnet.py, cvnets/models/classification/efficientnet.py,
config/efficientnet.py); see make_golden.py for the method.  Inputs and output gradients are regenerated from their seeds and large
tensors are stored as fixed samples (golden_sample.py).  Writes efficientnet_fp32.pt with
  * stand-alone depthwise 5x5 ConvLayer2d + BN, stride 1 and 2;
  * EfficientNetBlock: expand 1 with a 3x3 kernel, expand 6 with 5x5 / stride 2, expand 6 with 5x5 / stride 1 and a residual;
  * EfficientNet-b0 at 2 x 3 x 64 x 64, forward and backward;
  * the module contract: EfficientNetBlock / EfficientNet constructor parameters, the b0 state_dict [key, shape, dtype] list, b0 .. b3
    state_dict digests and the per-block stochastic-depth probabilities at stochastic_depth_prob 0.2.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_efficientnet.py
"""
import copy
import hashlib
import inspect
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from make_golden import O, load_seeded, make_opts, run_module, strip, torch  # noqa: E402
from golden_sample import sample_large  # noqa: E402
import efficientnet_ref as E  # noqa: E402

from cvnets.layers import ConvLayer2d  # noqa: E402
from cvnets.models.classification.efficientnet import EfficientNet  # noqa: E402
from cvnets.modules import EfficientNetBlock  # noqa: E402

DW = {"dw5_s1": dict(c=144, stride=1, shape=(2, 144, 14, 12), seed=61), "dw5_s2": dict(c=240, stride=2, shape=(2, 240, 14, 14), seed=62)}
BLOCKS = {
    "eb_e1_k3": dict(cin=32, cout=16, expand_ratio=1, kernel_size=3, stride=1, shape=(2, 32, 16, 16), seed=71),
    "eb_e6_k5_s2": dict(cin=24, cout=40, expand_ratio=6, kernel_size=5, stride=2, shape=(2, 24, 16, 16), seed=72),
    "eb_e6_k5_res": dict(cin=40, cout=40, expand_ratio=6, kernel_size=5, stride=1, shape=(2, 40, 12, 10), seed=73),
}


def params(f):
    return [p for p in inspect.signature(f).parameters if p not in ("args", "kwargs")]


def compact(out, x_seed, gy_seed, limit=8192, n=4096, buffers=("",)):
    """x and gy are regenerated from their seeds (oracle.seeded_input); large outputs / gradients are stored as fixed samples, and only the
    buffers whose names end in one of ``buffers``."""
    out = dict(out, x_shape=tuple(out["x"].shape), x_seed=x_seed, gy_seed=gy_seed)
    del out["x"], out["gy"]
    for k in ("y", "gx"):
        out[k] = sample_large(out[k], limit, n)
    out["grads"] = {k: sample_large(v, limit, n) for k, v in out["grads"].items()}
    out["buffers"] = {k: sample_large(v, limit, n) for k, v in out["buffers"].items() if k.endswith(buffers)}
    return out


def sd_entries(mod):
    return [[k, list(v.shape), str(v.dtype)] for k, v in mod.state_dict().items()]


def sd_digest(mod):
    """Whole-model state_dicts are pinned by the SHA-256 of their canonical [key, shape, dtype] list, as in make_golden_contract.py."""
    e = sd_entries(mod)
    return {"n_entries": len(e), "sha256": hashlib.sha256(json.dumps(e, separators=(",", ":")).encode()).hexdigest()}


def effnet_opts(mode, sd=0.0):
    opts = copy.deepcopy(make_opts(1.0))
    for k, v in {"model.classification.name": "efficientnet", "model.classification.efficientnet.mode": mode,
                 "model.classification.efficientnet.stochastic_depth_prob": sd, "model.classification.classifier_dropout": 0.0,
                 "model.classification.n_classes": 1000}.items():
        setattr(opts, k, v)
    return opts


def main():
    torch.manual_seed(0)
    opts = effnet_opts("b0")
    fx = {}
    for name, c in DW.items():
        P = {}
        O._conv_bn(P, "m", c["c"], c["c"], 5, groups=c["c"])
        m = ConvLayer2d(opts, c["c"], c["c"], 5, stride=c["stride"], groups=c["c"], use_norm=True, use_act=False)
        load_seeded(m, strip("m.", P), c["seed"])
        fx[name] = dict(cfg={k: v for k, v in c.items() if k not in ("shape", "seed")}, seed=c["seed"],
                        **compact(run_module(m, O.seeded_input(c["shape"], 100 + c["seed"]), 200 + c["seed"]), 100 + c["seed"], 200 + c["seed"]))
    for name, c in BLOCKS.items():
        P = {}
        E.efficientnet_block_shapes(P, "m", c["cin"], c["cout"], c["expand_ratio"], c["kernel_size"])
        m = EfficientNetBlock(0.0, opts=opts, in_channels=c["cin"], out_channels=c["cout"], kernel_size=c["kernel_size"], stride=c["stride"],
                              expand_ratio=c["expand_ratio"], dilation=1, use_hs=False, use_se=True, use_input_as_se_dim=True,
                              squeeze_factor=c["expand_ratio"] * 4, act_fn_name="swish", se_scale_fn_name="sigmoid")
        load_seeded(m, strip("m.", P), c["seed"])
        fx[name] = dict(cfg={k: v for k, v in c.items() if k not in ("shape", "seed")}, seed=c["seed"], repr=repr(m),
                        **compact(run_module(m, O.seeded_input(c["shape"], 100 + c["seed"]), 200 + c["seed"]), 100 + c["seed"], 200 + c["seed"]))
    # whole model, b0 at 64 x 64
    model = EfficientNet(opts)
    P = E.efficientnet_shapes("b0")
    load_seeded(model, P, 81)
    # (the whole model keeps the running variances only: the running means follow the same batch statistics)
    fx["b0_64"] = dict(seed=81, **compact(run_module(model, O.seeded_input((2, 3, 64, 64), 181), 281), 181, 281, limit=256, n=128,
                                          buffers=("running_var",)))
    # contract
    contract = {"block_init": params(EfficientNetBlock.__init__), "model_init": params(EfficientNet.__init__), "models": {}}
    for mode in ("b0", "b1", "b2", "b3"):
        mm = EfficientNet(effnet_opts(mode, 0.2))
        contract["models"][mode] = {
            "state_dict": sd_digest(mm),
            "children": [n for n, _ in mm.named_children()],
            "sd_probs": [float(b.stochastic_depth.p) for n in ("layer_1", "layer_2", "layer_3", "layer_4", "layer_5") for b in getattr(mm, n)],
            "kernels": [int(b.kernel_size) for n in ("layer_1", "layer_2", "layer_3", "layer_4", "layer_5") for b in getattr(mm, n)],
            "block_repr": repr(getattr(mm, "layer_4")[3]),
        }
    contract["b0_state_dict"] = sd_entries(EfficientNet(effnet_opts("b0")))  # the readable list behind the b0 digest
    fx["contract"] = contract
    for k, v in fx.items():
        if "y" in v:
            print(k, v["x_shape"])
    torch.save(fx, os.path.join(HERE, "efficientnet_fp32.pt"))


if __name__ == "__main__":
    main()

"""Module-contract fixture FROM THE REAL REFERENCE (apple/ml-cvnets): constructor / forward signatures, state_dict keys, shapes and
dtypes, child trees and reprs of the reference classes this package replaces, so that tests/test_host_cpu.py checks the drop-ins
without a reference checkout.

    python tests/golden/make_golden_contract.py /path/to/ml-cvnets      # writes tests/golden/reference_contract.json
"""
import argparse
import hashlib
import inspect
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))


def params(f):
    return [p for p in inspect.signature(f).parameters if p not in ("args", "kwargs")]


def sd_entries(mod):
    return [[k, list(v.shape), str(v.dtype)] for k, v in mod.state_dict().items()]


def sd_digest(mod):
    """Whole-model state_dicts are pinned by the SHA-256 of their canonical [key, shape, dtype] list (tests/test_host_cpu.py recomputes it)."""
    e = sd_entries(mod)
    return {"n_entries": len(e), "sha256": hashlib.sha256(json.dumps(e, separators=(",", ":")).encode()).hexdigest()}


# the InvertedResidualSE configurations the contract covers (kwargs after (opts, 24, 24))
SE_CONFIGS = [dict(expand_ratio=4, stride=1, use_se=True, act_fn_name="hard_swish"), dict(expand_ratio=3, stride=2, use_se=True, act_fn_name="relu"),
              dict(expand_ratio=1, stride=1, use_se=False, act_fn_name="relu"), dict(expand_ratio=2, stride=1, use_se=True, kernel_size=5)]


def main():
    ref = os.path.abspath(sys.argv[1])
    sys.path.insert(0, ref)
    os.chdir(ref)
    import torch
    from cvnets import get_model, modeling_arguments
    from cvnets.layers import MultiHeadAttention as RefMHA
    from cvnets.modules import InvertedResidualSE as RefSE, SqueezeExcitation as RefSq, TransformerEncoder as RefEnc

    torch.manual_seed(0)
    out = {}
    opts = modeling_arguments(argparse.ArgumentParser()).parse_args([])
    # ---- classification models (the ones register.py registers replacements for)
    for k, v in {"dataset.category": "classification", "model.classification.name": "mobilevit_v2",
                 "model.classification.mitv2.width_multiplier": 1.0, "model.activation.name": "swish"}.items():
        setattr(opts, k, v)
    mv2 = get_model(opts)
    out["mobilevit_v2"] = {"n_params": sum(p.numel() for p in mv2.parameters()), "state_dict": sd_digest(mv2)}
    setattr(opts, "model.classification.mit.mode", "xx_small")
    setattr(opts, "model.classification.name", "mobilevit")
    out["mobilevit_xx_small"] = {"state_dict": sd_digest(get_model(opts))}
    for k, v in {"model.classification.vit.mode": "tiny", "model.classification.vit.norm_layer": "layer_norm_fp32", "model.activation.name": "gelu",
                 "model.classification.activation.name": "gelu", "model.classification.name": "vit"}.items():
        setattr(opts, k, v)
    out["vit_tiny"] = {"state_dict": sd_digest(get_model(opts))}
    # ---- MultiHeadAttention / TransformerEncoder
    opts = modeling_arguments(argparse.ArgumentParser()).parse_args([])
    enc = {"params": {"mha_init": params(RefMHA.__init__), "enc_init": params(RefEnc.__init__), "enc_forward": params(RefEnc.forward)},
           "mha_state_dict": [k for k in RefMHA(64, 4).state_dict()]}
    for act in ("swish", "gelu"):
        setattr(opts, "model.activation.name", act)
        b = RefEnc(opts, 64, 128, num_heads=4)
        enc[act] = {"state_dict": sd_entries(b), "eps": float(b.pre_norm_mha[0].eps), "repr_head": repr(b).split("(")[0]}
    out["transformer"] = enc
    # ---- InvertedResidualSE / SqueezeExcitation, and the dropout children of TransformerEncoder, under the default options
    opts = modeling_arguments(argparse.ArgumentParser()).parse_args([])
    se = {"params": {"se_init": params(RefSE.__init__), "sq_init": params(RefSq.__init__)}, "configs": [],
          "activation": getattr(opts, "model.activation.name")}
    e2 = RefEnc(opts, 64, 128, num_heads=4, dropout=0.1, ffn_dropout=0.2)
    se["dropout_children"] = {"pre_norm_ffn": [type(m).__name__ for m in e2.pre_norm_ffn],
                              "p": [e2.pre_norm_mha[2].p, e2.pre_norm_ffn[3].p, e2.pre_norm_ffn[5].p]}
    s2 = RefEnc(opts, 64, 128, num_heads=4, stochastic_dropout=0.2)
    se["stochastic"] = {"drop_path": type(s2.drop_path).__name__, "p": s2.drop_path.p, "state_dict_keys": list(s2.state_dict().keys())}
    for kw in SE_CONFIGS:
        b = RefSE(opts, 24, 24, **kw)
        se["configs"].append({"kwargs": kw, "state_dict": sd_entries(b), "children": [n for n, _ in b.block.named_children()],
                              "modules": list(b.block._modules), "repr": repr(b), "use_res_connect": bool(b.use_res_connect)})
    out["inverted_residual_se"] = se
    with open(os.path.join(HERE, "reference_contract.json"), "w") as f:
        json.dump(out, f, separators=(",", ":"))


if __name__ == "__main__":
    main()

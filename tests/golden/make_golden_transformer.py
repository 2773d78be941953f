"""Golden fixtures for the transformer rows (SURVEY.md 8a a10-a12) FROM THE REAL REFERENCE (apple/ml-cvnets @ /root/reference).

Same protocol as make_golden.py: the reference's own ``MultiHeadAttention`` / ``TransformerEncoder`` get the deterministic
parameters of ``oracle.cvnets_oracle.seeded_fill_`` (asserting the ``state_dict`` key/shape contract on the way), run forward +
backward in fp32 on CPU, and the results are stored in ``transformer_fp32.pt``.  Build container only.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_transformer.py
"""
import argparse
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
REPO = os.path.dirname(os.path.dirname(HERE))
REF = "/root/reference"
sys.path.insert(0, REPO)
sys.path.insert(0, REF)
sys.path.insert(0, os.path.dirname(HERE))
os.chdir(REF)

import torch  # noqa: E402
from golden_sample import sample_large  # noqa: E402

from cvnets import modeling_arguments  # noqa: E402
from cvnets.layers import MultiHeadAttention  # noqa: E402
from cvnets.modules import TransformerEncoder  # noqa: E402
from oracle import cvnets_oracle as O  # noqa: E402


def make_opts(act):
    opts = modeling_arguments(argparse.ArgumentParser()).parse_args([])
    setattr(opts, "model.activation.name", act)
    return opts


def load_seeded(module, P, seed):
    sd = module.state_dict()
    assert set(sd.keys()) == set(P.keys()), sorted(set(sd) ^ set(P))
    for k in sd:
        assert tuple(sd[k].shape) == tuple(P[k].shape), (k, sd[k].shape, P[k].shape)
    O.seeded_fill_(P, seed)
    module.load_state_dict({k: v.clone() for k, v in P.items()}, strict=True)


def run(module, x, gy_seed, **kw):
    module.train()
    module.zero_grad(set_to_none=True)
    x = x.clone().requires_grad_(True)
    y = module(x, **kw)
    gy = O.seeded_input(tuple(y.shape), gy_seed)
    y.backward(gy)
    return {"x": x.detach().clone(), "y": y.detach().clone(), "gy": gy, "gx": x.grad.clone(),
            "grads": {k: p.grad.clone() for k, p in module.named_parameters()}}


def strip(prefix, d):
    return {k[len(prefix):]: v for k, v in d.items()}


def main():
    torch.manual_seed(0)
    fx = {}
    # ---- MultiHeadAttention: plain, causal additive mask, key padding mask (multi_head_attention.py:197-224)
    for name, (c, heads, n, s, seed) in {"mha": (64, 4, 2, 20, 31), "mha_hd32": (64, 2, 3, 9, 32)}.items():
        P = {}
        O.multi_head_attention_shapes(P, "m", c)
        m = MultiHeadAttention(c, heads, attn_dropout=0.0, bias=True)
        load_seeded(m, strip("m.", P), seed)
        fx[name] = dict(cfg=dict(c=c, heads=heads), seed=seed, **run(m, O.seeded_input((n, s, c), 100 + seed), 200 + seed))
        if name == "mha":
            causal = torch.full((s, s), float("-inf")).triu(1)[None].repeat(n, 1, 1)
            fx["mha_causal"] = dict(cfg=dict(c=c, heads=heads), seed=seed, attn_mask=causal,
                                    **run(m, O.seeded_input((n, s, c), 100 + seed), 200 + seed, attn_mask=causal))
            kpm = torch.zeros(n, s, dtype=torch.bool)
            kpm[0, 15:] = True
            kpm[1, 18:] = True
            fx["mha_padding"] = dict(cfg=dict(c=c, heads=heads), seed=seed, key_padding_mask=kpm,
                                     **run(m, O.seeded_input((n, s, c), 100 + seed), 200 + seed, key_padding_mask=kpm))
    # ---- TransformerEncoder: MobileViT flavour (swish) and ViT flavour (gelu, eps as built by get_normalization_layer)
    for name, (c, ffn, heads, n, s, act, seed) in {"enc_swish": (64, 128, 4, 2, 20, "swish", 41), "enc_gelu": (128, 256, 2, 2, 12, "gelu", 42)}.items():
        opts = make_opts(act)
        P = {}
        O.transformer_encoder_shapes(P, "m", c, ffn)
        m = TransformerEncoder(opts, embed_dim=c, ffn_latent_dim=ffn, num_heads=heads, attn_dropout=0.0, dropout=0.0, ffn_dropout=0.0)
        load_seeded(m, strip("m.", P), seed)
        eps = m.pre_norm_mha[0].eps
        fx[name] = dict(cfg=dict(c=c, ffn=ffn, heads=heads, act=act, eps=eps), seed=seed,
                        **run(m, O.seeded_input((n, s, c), 100 + seed), 200 + seed))
    for rec in fx.values():
        rec["grads"] = {k: sample_large(g) for k, g in rec["grads"].items()}
    torch.save(fx, os.path.join(HERE, "transformer_fp32.pt"))
    print("wrote", sorted(fx.keys()))


if __name__ == "__main__":
    main()

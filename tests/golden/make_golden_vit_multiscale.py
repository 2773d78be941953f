"""Golden fixture FROM THE REAL REFERENCE for VisionTransformer at the variable-batch sampler's crops (see make_golden.py for the method).

The reference's ViT keeps 196 positional embeddings and resizes them with F.interpolate whenever the patch count differs
(cvnets/layers/positional_embedding.py:90-95).  "small" geometry (12 layers, head_dim 64, like base), train mode, batch 2, dropouts 0, at
  * 320 x 320: S = 401, table upsampled,
  * 128 x 128: S = 65, table downsampled,
  * 256 x 320: S = 321, a non-square crop above 256 tokens.
Stores logits, loss, every gradient norm and a fixed sample of every gradient (golden_sample.sample_large) per crop.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_vit_multiscale.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from golden_sample import sample_large  # noqa: E402
from make_golden import O, F, get_model, load_seeded, make_opts, torch  # noqa: E402

CROPS = ((320, 320), (128, 128), (256, 320))


def main():
    torch.manual_seed(0)
    opts = make_opts(1.0)
    for k, v in {"model.classification.name": "vit", "model.classification.vit.mode": "small", "model.classification.vit.norm_layer": "layer_norm_fp32",
                 "model.activation.name": "gelu", "model.classification.activation.name": "gelu", "model.classification.n_classes": 1000}.items():
        setattr(opts, k, v)
    model = get_model(opts)
    P = O.vit_shapes("small")
    seed = 61
    fx = dict(mode="small", seed=seed, keys=[[k, list(v.shape)] for k, v in model.state_dict().items()], crops={})
    for i, (h, w) in enumerate(CROPS):
        load_seeded(model, P, seed)
        model.train()
        model.zero_grad(set_to_none=True)
        x_seed = 361 + i
        x = O.seeded_input((2, 3, h, w), x_seed)
        labels = torch.tensor([17 + i, 503 + i])
        logits = model(x)
        loss = F.cross_entropy(logits, labels, label_smoothing=0.1)
        loss.backward()
        grads = {k: p.grad for k, p in model.named_parameters()}
        fx["crops"][f"{h}x{w}"] = dict(
            size=(h, w), x_seed=x_seed, labels=labels, logits=logits.detach().clone(), loss=loss.detach().clone(),
            grad_norms={k: float(g.norm()) for k, g in grads.items()},
            grads={k: sample_large(g.detach().clone(), limit=256, n=256) for k, g in grads.items()})
    out = os.path.join(HERE, "vit_multiscale_fp32.pt")
    torch.save(fx, out)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()

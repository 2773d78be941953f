"""Golden fixture FROM THE REAL REFERENCE for the ViT-H/16 recipes (see make_golden.py for the method).

  * ViT-H/16 classifier (32 layers, 1280 wide, 20 heads), train mode, ``gradient_checkpointing`` on with 4 segments (vit.py:526-533), batch 2,
    dropouts 0, at 128 x 128 (S = 65, table downsampled) and 320 x 320 (S = 401, table upsampled): logits, loss, every gradient norm and a
    fixed sample of every gradient (golden_sample.sample_large, 128 elements: the ~520 gradients of both crops stay under 1 MB) per crop.
  * the state_dict keys and shapes of the CLIP ViT-H/16 recipe model (examples/range_augment/clip/clip_vit_huge.yaml: 768-wide, 12-layer,
    12-head text tower, projection 512, RangeAugment augmentor, both towers checkpointed).

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_vit_huge.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from golden_sample import sample_large  # noqa: E402
from make_golden import O, F, get_model, load_seeded, make_opts, torch  # noqa: E402
from vit_huge_ref import vit_huge_shapes  # noqa: E402
from make_golden_range_augment_vit import CLIP, VIT, opts_with  # noqa: E402

CROPS = ((128, 128), (320, 320))
HUGE = {"model.classification.vit.mode": "huge", "model.classification.gradient_checkpointing": True,
        "model.classification.vit.checkpoint_segments": 4}
CLIP_HUGE = {"model.multi_modal_image_text.clip.projection_dim": 512, "model.text.transformer.model_dim": 768,
             "model.text.transformer.n_transformer_layers": 12, "model.text.transformer.n_heads_per_layer": 12,
             "model.text.transformer.gradient_checkpoint": True, "dataset.text_vocab_size": 49408, "dataset.text_context_length": 77,
             "model.learn_augmentation.mode": "distribution"}


def main():
    torch.manual_seed(0)
    opts = make_opts(1.0)
    for k, v in dict(VIT, **HUGE, **{"model.classification.n_classes": 1000}).items():
        setattr(opts, k, v)
    model = get_model(opts)
    assert model.gradient_checkpointing and model.checkpoint_segments == 4
    P = vit_huge_shapes()
    seed = 71
    fx = dict(mode="huge", seed=seed, segments=4, keys=[[k, list(v.shape)] for k, v in model.state_dict().items()], crops={})
    for i, (h, w) in enumerate(CROPS):
        load_seeded(model, P, seed)
        model.train()
        model.zero_grad(set_to_none=True)
        x_seed = 381 + i
        x = O.seeded_input((2, 3, h, w), x_seed)
        labels = torch.tensor([29 + i, 611 + i])
        logits = model(x)
        loss = F.cross_entropy(logits, labels, label_smoothing=0.1)
        loss.backward()
        grads = {k: p.grad for k, p in model.named_parameters()}
        fx["crops"][f"{h}x{w}"] = dict(
            size=(h, w), x_seed=x_seed, labels=labels, logits=logits.detach().clone(), loss=loss.detach().clone(),
            grad_norms={k: float(g.norm()) for k, g in grads.items()},
            grads={k: sample_large(g.detach().clone(), limit=256, n=128) for k, g in grads.items()})
        print(f"{h}x{w}", float(loss))
    del model
    copts = opts_with(dict(VIT, **CLIP))
    for k, v in dict(HUGE, **CLIP_HUGE).items():
        setattr(copts, k, v)
    clip = get_model(copts)
    fx["clip_keys"] = [[k, list(v.shape)] for k, v in clip.state_dict().items()]
    out = os.path.join(HERE, "vit_huge_fp32.pt")
    torch.save(fx, out)
    print(out, os.path.getsize(out), "bytes")


if __name__ == "__main__":
    main()

"""RangeAugment on the ViT / CLIP recipes, fixture FROM THE REAL REFERENCE (see make_golden.py for the method).

Builds the reference's ViT-tiny classifier (10 classes) and a small CLIP (ViT-tiny image tower, projection 64, 2-layer / 128-wide causal text
tower, vocabulary 1000, context 16), both with ``model.learn_augmentation.mode: distribution`` (brightness, contrast, noise), and records:
  * the ``state_dict`` keys in order with their shapes, and the weight decay the reference's ``get_trainable_parameters`` (weight decay 0.05,
    no_decay_bn_filter_bias) gives each augmentor parameter;
  * one training forward / backward on seeded parameters (oracle.seeded_fill_ + range_augment_ref.seeded_aug_params) with the augmentor's draws
    recorded (make_golden_range_augment.recorded_forward): the augmented image, the logits (ViT) or the image / text features and the logit
    scale (CLIP), the two loss terms -- cross entropy with label smoothing 0.1, or the contrastive loss (ContrastiveLossClip), and the PSNR loss
    at epoch 4 of a 10-epoch cosine curriculum from 40 to 20 dB (the recipes' target) -- and the gradients of the sampler parameters and of the
    stem conv weight under their sum.
The 'tiny' ViT's positional-embedding dropout (0.1) is set to 0 so that the recorded step is deterministic.  The input images are stored as
their seed (make_golden_range_augment.image, with their sum as a check) and the augmented images as a fixed sample (golden_sample.py); the
noise the augmentor drew is stored whole.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_range_augment_vit.py
"""
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from golden_sample import sample_large  # noqa: E402
from make_golden import O, get_model, torch  # noqa: E402
from make_golden_range_augment import image, loss_opts, recorded_forward  # noqa: E402
import range_augment_ref as R  # noqa: E402
import torch.nn.functional as F  # noqa: E402

from loss_fn.multi_modal_img_text.contrastive_loss_clip import ContrastiveLossClip  # noqa: E402
from loss_fn.neural_augmentation import NeuralAugmentation  # noqa: E402

VIT = {"model.classification.name": "vit", "model.classification.vit.mode": "tiny", "model.classification.vit.norm_layer": "layer_norm_fp32",
       "model.activation.name": "gelu", "model.classification.activation.name": "gelu"}
CLIP = {"dataset.category": "multi_modal_image_text", "model.multi_modal_image_text.name": "clip", "model.multi_modal_image_text.clip.projection_dim": 64,
        "model.image_projection_head.name": "simple_projection_nc2nc", "model.text.name": "transformer", "model.text.transformer.model_dim": 128,
        "model.text.transformer.n_transformer_layers": 2, "model.text.transformer.n_heads_per_layer": 4,
        "model.text.transformer.ffn_multiplier_per_layer": 4.0, "model.text.transformer.causal_masking": True,
        "model.text.transformer.norm_layer": "layer_norm_fp32", "dataset.text_vocab_size": 1000, "dataset.text_context_length": 16,
        "dataset.padding_index": None, "ddp.use_distributed": False, "ddp.rank": 0,
        "model.multi_modal_image_text.clip.cache_text_features_zero_shot": False}
EPOCH, PERIOD, TARGET = 4, 10, (40, 20)


def opts_with(kv):
    opts = loss_opts(PERIOD, target=TARGET)
    for k, v in kv.items():
        setattr(opts, k, v)
    return opts


def decay_of_augmentor(model):
    groups, _ = model.get_trainable_parameters(weight_decay=0.05, no_decay_bn_filter_bias=True)
    out = {}
    for g in groups:
        for name in g["param_names"]:
            if "neural_augmentor." in name:
                out[name] = float(g["weight_decay"])
    assert len(out) == 6, out
    return out


def tokens(B, L, seed):
    g = torch.Generator().manual_seed(seed)
    tok = torch.randint(1, 998, (B, L), generator=g)
    tok[torch.arange(B), torch.randint(2, L, (B,), generator=g)] = 999
    return tok


def main():
    torch.manual_seed(0)
    random.seed(0)  # the reference shuffles the augmentations' order with Python's generator
    fx = {"epoch": EPOCH, "period": PERIOD, "target": TARGET}
    crit = NeuralAugmentation(loss_opts(PERIOD, target=TARGET))

    # ViT-tiny classifier, 2 x 3 x 64 x 64 (the positional table is interpolated to 4 x 4 patches)
    opts = opts_with(dict(VIT, **{"model.classification.n_classes": 10}))
    model = get_model(opts).train()
    model.emb_dropout.p = 0.0
    keys = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
    P = O.seeded_fill_(O.vit_shapes("tiny", n_classes=10), 91)
    P.update(R.seeded_aug_params(92))
    model.load_state_dict(P, strict=True)
    x_seed = 191
    x = image(2, 64, 64, x_seed)
    y = torch.tensor([3, 7])
    torch.manual_seed(6)
    out, draws = recorded_forward(model, x)
    ce = F.cross_entropy(out["logits"], y, label_smoothing=0.1)
    na = crit(x, out, epoch=EPOCH)
    names = R.AUG_KEYS + ["patch_emb.0.block.conv.weight"]
    params = dict(model.named_parameters())
    grads = torch.autograd.grad(ce + na, [params[k] for k in names])
    fx["vit"] = {"mode": "tiny", "seed": 91, "aug_seed": 92, "state_dict_keys": keys, "decay": decay_of_augmentor(model), "x_shape": tuple(x.shape),
                 "x_seed": x_seed, "x_sum": float(x.double().sum()), "y": y, "draws": draws, "x_aug": sample_large(out["augmented_tensor"].detach().clone()),
                 "logits": out["logits"].detach().clone(), "ce": ce.detach(), "na": na.detach(), "grads": {k: g.clone() for k, g in zip(names, grads)}}
    print("vit", draws["order"], float(ce), float(na), [float(g) for g in grads[:6]])

    # small CLIP, ViT-tiny image tower at 2 x 3 x 224 x 224 (its 196-entry positional table as is)
    opts = opts_with(dict(VIT, **CLIP))
    model = get_model(opts).train()
    model.image_encoder.emb_dropout.p = 0.0
    keys = [(k, tuple(v.shape)) for k, v in model.state_dict().items()]
    P = O.clip_shapes("tiny", proj=64, text_dim=128, text_layers=2, vocab=1000, ctx=16)
    O.seeded_fill_(P, 93)
    P.update({"image_encoder." + k: v for k, v in R.seeded_aug_params(94).items()})
    model.load_state_dict(P, strict=True)
    x_seed = 193
    x = image(2, 224, 224, x_seed)
    tok = tokens(2, 16, 194)
    torch.manual_seed(7)
    out, draws = recorded_forward(lambda im: model({"image": im, "text": tok}), x)
    pred = dict(out)
    clip_loss = ContrastiveLossClip(opts)(None, pred)["total_loss"]
    na = crit(x, out, epoch=EPOCH)
    names = ["image_encoder." + k for k in R.AUG_KEYS] + ["image_encoder.patch_emb.0.block.conv.weight"]
    params = dict(model.named_parameters())
    grads = torch.autograd.grad(clip_loss + na, [params[k] for k in names])
    fx["clip"] = {"vit_mode": "tiny", "seed": 93, "aug_seed": 94, "state_dict_keys": keys, "decay": decay_of_augmentor(model), "x_shape": tuple(x.shape),
                  "x_seed": x_seed, "x_sum": float(x.double().sum()), "tokens": tok, "draws": draws,
                  "x_aug": sample_large(out["augmented_tensor"].detach().clone()), "image": out["image"].detach().clone(),
                  "text": out["text"].detach().clone(), "logit_scale": out["logit_scale"].detach().clone(), "clip_loss": clip_loss.detach(),
                  "na": na.detach(), "grads": {k: g.clone() for k, g in zip(names, grads)}}
    print("clip", draws["order"], float(clip_loss), float(na), [float(g) for g in grads[:6]])
    out_path = os.path.join(HERE, "range_augment_vit_fp32.pt")
    torch.save(fx, out_path)
    print(out_path, os.path.getsize(out_path), "bytes")


if __name__ == "__main__":
    main()

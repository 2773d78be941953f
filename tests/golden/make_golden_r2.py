"""Round-2 golden fixtures FROM THE REAL REFERENCE (apple/ml-cvnets @ /root/reference); see make_golden.py for the method.

  * ``lsa_cross`` / ``laffn_cross``: LinearSelfAttention / LinearAttnFFN cross-attention (linear_attention.py:163-207, transformer.py:254-260)
  * ``pw_bn_act`` / ``pw_bias`` / ``dw_bn_act`` / ``ln2d`` / ``ln`` / ``ln_fp32`` / ``linear`` / ``pool``: the stand-alone layers
  * ``model_b16``: MobileViTv2-1.0, batch 16 at 128x128, train mode -- a WELL-CONDITIONED end-to-end fixture (VERDICT r1: the batch-2
    fixtures let train-mode BatchNorm amplify bf16 rounding to ~10 %): logits, loss and every gradient tensor <= 64k elements.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_r2.py
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(HERE))
from golden_sample import sample_large  # noqa: E402
from make_golden import O, F, ConvLayer2d, LinearSelfAttention, LinearAttnFFN, get_model, load_seeded, make_opts, run_module, strip, torch  # noqa: E402

from cvnets.layers import GlobalPool, LinearLayer  # noqa: E402
from cvnets.layers.normalization.layer_norm import LayerNorm, LayerNorm2D_NCHW, LayerNormFP32  # noqa: E402


def run_cross(module, x, xp, gy_seed):
    module.train()
    x = x.clone().requires_grad_(True)
    xp = xp.clone().requires_grad_(True)
    y = module(x, xp)
    gy = O.seeded_input(tuple(y.shape), gy_seed)
    y.backward(gy)
    return {"x": x.detach().clone(), "x_prev": xp.detach().clone(), "y": y.detach().clone(), "gy": gy, "gx": x.grad.clone(), "gx_prev": xp.grad.clone(),
            "grads": {k: p.grad.clone() for k, p in module.named_parameters()}, "buffers": {}}


def main():
    torch.manual_seed(0)
    opts = make_opts(1.0)
    fx = {}
    P = {}
    O._conv_bn(P, "m.qkv_proj", 16, 33, 1, norm=False, bias=True)
    O._conv_bn(P, "m.out_proj", 16, 16, 1, norm=False, bias=True)
    m = LinearSelfAttention(opts, embed_dim=16, attn_dropout=0.0, bias=True)
    load_seeded(m, strip("m.", P), 34)
    fx["lsa_cross"] = dict(cfg=dict(d=16), seed=34, **run_cross(m, O.seeded_input((2, 16, 4, 9), 134), O.seeded_input((2, 16, 4, 12), 135), 234))
    P = {}
    O.linear_attn_ffn_shapes(P, "m", 16, 32)
    m = LinearAttnFFN(opts, embed_dim=16, ffn_latent_dim=32, attn_dropout=0.0, dropout=0.0, ffn_dropout=0.0)
    load_seeded(m, strip("m.", P), 35)
    fx["laffn_cross"] = dict(cfg=dict(d=16, ffn=32), seed=35, **run_cross(m, O.seeded_input((2, 16, 4, 9), 136), O.seeded_input((2, 16, 4, 12), 137), 235))

    # ---- stand-alone layers
    P = {}
    O._conv_bn(P, "m", 16, 24, 1)
    m = ConvLayer2d(opts, 16, 24, 1, use_norm=True, use_act=True)
    load_seeded(m, strip("m.", P), 36)
    fx["pw_bn_act"] = dict(cfg=dict(cin=16, cout=24), seed=36, **run_module(m, O.seeded_input((3, 16, 6, 5), 138), 238))
    P = {}
    O._conv_bn(P, "m", 16, 24, 1, norm=False, bias=True)
    m = ConvLayer2d(opts, 16, 24, 1, use_norm=False, use_act=False, bias=True)
    load_seeded(m, strip("m.", P), 37)
    fx["pw_bias"] = dict(cfg=dict(cin=16, cout=24), seed=37, **run_module(m, O.seeded_input((3, 16, 6, 5), 139), 239))
    P = {}
    O._conv_bn(P, "m", 16, 16, 3, groups=16)
    m = ConvLayer2d(opts, 16, 16, 3, stride=2, groups=16, use_norm=True, use_act=True)
    load_seeded(m, strip("m.", P), 38)
    fx["dw_bn_act"] = dict(cfg=dict(c=16, stride=2), seed=38, **run_module(m, O.seeded_input((3, 16, 8, 8), 140), 240))
    for name, cls, shape in (("ln2d", LayerNorm2D_NCHW, (3, 16, 4, 9)), ("ln", LayerNorm, (3, 7, 32)), ("ln_fp32", LayerNormFP32, (3, 7, 32))):
        C = shape[1] if name == "ln2d" else shape[-1]
        P = {}
        O._gn(P, "m", C)
        m = cls(C)
        O.seeded_fill_(P, 39)  # fill under the PREFIXED keys ("m.weight" is a norm gamma; a bare "weight" would be seeded like a bias)
        m.load_state_dict({k: v.clone() for k, v in strip("m.", P).items()}, strict=True)
        fx[name] = dict(cfg=dict(c=C), seed=39, **run_module(m, O.seeded_input(shape, 141), 241))
    P = {}
    O._linear(P, "m", 32, 40)
    m = LinearLayer(32, 40, bias=True)
    load_seeded(m, strip("m.", P), 40)
    fx["linear"] = dict(cfg=dict(cin=32, cout=40), seed=40, **run_module(m, O.seeded_input((3, 7, 32), 142), 242))
    m = GlobalPool(pool_type="mean", keep_dim=False)
    fx["pool"] = dict(cfg={}, seed=0, **run_module(m, O.seeded_input((3, 16, 5, 4), 143), 243))
    torch.save(fx, os.path.join(HERE, "standalone_fp32.pt"))

    # ---- well-conditioned model fixture
    width, res, seed, B = 1.0, 128, 41, 16
    model = get_model(make_opts(width))
    P = O.mobilevit_v2_shapes(width)
    load_seeded(model, P, seed)
    model.train()
    x = O.seeded_input((B, 3, res, res), 300 + seed)
    labels = (torch.arange(B) * 61) % 1000
    logits = model(x)
    loss = F.cross_entropy(logits, labels, label_smoothing=0.1)
    loss.backward()
    grads = {k: p.grad for k, p in model.named_parameters()}
    fixture = dict(width=width, res=res, seed=seed, x_seed=300 + seed, batch=B, labels=labels, logits=logits.detach().clone(), loss=loss.detach().clone(),
                   grad_norms={k: float(g.norm()) for k, g in grads.items()},
                   grads={k: sample_large(g.clone().half() if g.numel() > 4096 else g.clone(), limit=2048, n=2048) for k, g in grads.items()
                          if g.numel() <= 65536},
                   buffers_after={k: b.detach().clone() for k, b in model.named_buffers() if b.numel() <= 4096})
    torch.save(fixture, os.path.join(HERE, "mobilevit_v2_b16_fp32.pt"))
    # ---- VisionTransformer, "small" geometry (same code path as base: 12 layers, head_dim 64, S = 197), batch 2 @ 224
    opts = make_opts(1.0)
    for k, v in {"model.classification.name": "vit", "model.classification.vit.mode": "small", "model.classification.vit.norm_layer": "layer_norm_fp32",
                 "model.activation.name": "gelu", "model.classification.activation.name": "gelu", "model.classification.n_classes": 1000}.items():
        setattr(opts, k, v)
    model = get_model(opts)
    P = O.vit_shapes("small")
    load_seeded(model, P, 51)
    model.train()
    x = O.seeded_input((2, 3, 224, 224), 351)
    labels = torch.tensor([5, 701])
    logits = model(x)
    loss = F.cross_entropy(logits, labels, label_smoothing=0.1)
    loss.backward()
    grads = {k: p.grad for k, p in model.named_parameters()}
    vit_fx = dict(mode="small", seed=51, x_seed=351, labels=labels, logits=logits.detach().clone(), loss=loss.detach().clone(),
                  keys=[[k, list(v.shape)] for k, v in model.state_dict().items()],
                  grad_norms={k: float(g.norm()) for k, g in grads.items()},
                  grads={k: g.clone() for k, g in grads.items() if g.numel() <= 20000})
    torch.save(vit_fx, os.path.join(HERE, "vit_small_fp32.pt"))
    # ---- MobileViT v1 XXS (BASELINE.json configs[0]): eval forward at 1x3x256x256 + a train-mode fwd/bwd (dropouts 0) at 4x3x192x192
    opts = make_opts(1.0)
    for k, v in {"model.classification.name": "mobilevit", "model.classification.mit.mode": "xx_small", "model.classification.mit.dropout": 0.0,
                 "model.classification.mit.attn_dropout": 0.0, "model.classification.mit.ffn_dropout": 0.0,
                 "model.classification.classifier_dropout": 0.0, "model.classification.n_classes": 1000}.items():
        setattr(opts, k, v)
    model = get_model(opts)
    P = O.mobilevit_v1_shapes("xx_small")
    load_seeded(model, P, 61)
    model.eval()
    x1 = O.seeded_input((1, 3, 256, 256), 361)
    with torch.no_grad():
        eval_logits = model(x1).clone()
    model.train()
    x = O.seeded_input((4, 3, 192, 192), 362)  # (128x128 would give N == d = 64 at layer 3: the reference LayerNorm then takes its channel-first branch)
    labels = torch.tensor([5, 701, 33, 999])
    logits = model(x)
    loss = F.cross_entropy(logits, labels, label_smoothing=0.1)
    loss.backward()
    grads = {k: p.grad for k, p in model.named_parameters()}
    mit_fx = dict(mode="xx_small", seed=61, eval_x_seed=361, eval_logits=eval_logits, x_seed=362, labels=labels, logits=logits.detach().clone(),
                  loss=loss.detach().clone(), keys=[[k, list(v.shape)] for k, v in model.state_dict().items()],
                  grad_norms={k: float(g.norm()) for k, g in grads.items()}, grads={k: g.clone() for k, g in grads.items() if g.numel() <= 5000})
    torch.save(mit_fx, os.path.join(HERE, "mobilevit_v1_xxs_fp32.pt"))
    # ---- CLIP (BASELINE.json configs[4]) at a reduced geometry: ViT-small image tower, 4-layer / 256-wide causal text transformer, projection 128
    from loss_fn.multi_modal_img_text.contrastive_loss_clip import ContrastiveLossClip
    opts = make_opts(1.0)
    for k, v in {"dataset.category": "multi_modal_image_text", "model.multi_modal_image_text.name": "clip", "model.multi_modal_image_text.clip.projection_dim": 128,
                 "model.classification.name": "vit", "model.classification.vit.mode": "small", "model.classification.vit.norm_layer": "layer_norm_fp32",
                 "model.activation.name": "gelu", "model.classification.activation.name": "gelu", "model.image_projection_head.name": "simple_projection_nc2nc",
                 "model.text.name": "transformer", "model.text.transformer.model_dim": 256, "model.text.transformer.n_transformer_layers": 4,
                 "model.text.transformer.n_heads_per_layer": 4, "model.text.transformer.ffn_multiplier_per_layer": 4.0,
                 "model.text.transformer.causal_masking": True, "model.text.transformer.norm_layer": "layer_norm_fp32", "dataset.text_vocab_size": 1000,
                 "dataset.text_context_length": 16, "dataset.padding_index": None, "ddp.use_distributed": False, "ddp.rank": 0}.items():
        setattr(opts, k, v)
    model = get_model(opts)
    P = O.clip_shapes("small", proj=128, text_dim=256, text_layers=4, vocab=1000, ctx=16)
    load_seeded(model, P, 71)
    model.train()
    images = O.seeded_input((8, 3, 224, 224), 371)
    gen = torch.Generator().manual_seed(372)
    tokens = torch.randint(1, 999, (8, 16), generator=gen)
    tokens[torch.arange(8), torch.tensor([15, 7, 9, 12, 3, 15, 10, 5])] = 999  # the end-of-text token is the highest id
    out = model({"image": images, "text": tokens})
    crit = ContrastiveLossClip(opts)
    crit.train()
    img_f, txt_f = out["image"].detach().clone(), out["text"].detach().clone()
    loss = crit(input_sample=None, prediction=dict(out), target=None)["total_loss"]
    loss.backward()
    grads = {k: p.grad for k, p in model.named_parameters()}
    clip_fx = dict(seed=71, x_seed=371, tokens=tokens, image_features=img_f, text_features=txt_f, loss=loss.detach().clone(),
                   keys=[[k, list(v.shape)] for k, v in model.state_dict().items()], grad_norms={k: float(g.norm()) for k, g in grads.items()},
                   grads={k: g.clone() for k, g in grads.items() if g.numel() <= 20000})
    torch.save(clip_fx, os.path.join(HERE, "clip_small_fp32.pt"))
    for fn in ("standalone_fp32.pt", "mobilevit_v2_b16_fp32.pt", "vit_small_fp32.pt", "mobilevit_v1_xxs_fp32.pt", "clip_small_fp32.pt"):
        print(fn, os.path.getsize(os.path.join(HERE, fn)), "bytes")


if __name__ == "__main__":
    main()

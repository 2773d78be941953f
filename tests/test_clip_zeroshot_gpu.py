"""CLIP zero-shot evaluation on the GPU (-m gpu): the class-embedding and logits / top-k kernels (csrc/zeroshot.cu) against fp32 torch, the
causal-prefix, length-bucketed text encoding, and the model against the real reference (tests/golden/make_golden_clip_zeroshot.py) within
the bounds of the torch-autocast restatement, as test_clip_against_reference_fixture does for training."""
import os
import sys

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from clip_zeroshot_ref import image_features, zero_shot_table  # noqa: E402

pytestmark = pytest.mark.gpu

SMALL = dict(projection_dim=128, text_dim=256, text_layers=4, text_heads=4, vocab_size=1000, context_length=16)


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as m
    return m


@pytest.fixture(scope="module")
def fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "clip_zeroshot_fp32.pt"), weights_only=False)


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))


def small_clip(pkg, fx, **extra):
    from ml_cvnets_b200.models_clip import CLIP, default_clip_opts
    model = CLIP(default_clip_opts("small", **SMALL, **extra))
    shapes = O.clip_shapes("small", proj=128, text_dim=256, text_layers=4, vocab=1000, ctx=16)
    model.load_state_dict(O.seeded_fill_(shapes, fx["seed"]), strict=True)
    return model.cuda().eval(), shapes


# ---------------------------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("d", [128, 512])
@pytest.mark.parametrize("M", [1, 5, 78])
@pytest.mark.parametrize("Cl", [1, 12, 1000])
def test_zs_class_embed(pkg, Cl, M, d):
    from ml_cvnets_b200 import ops
    g = torch.Generator(device="cuda").manual_seed(Cl * 1000 + M * 10 + d)
    R = Cl * M + 3  # a few rows no class uses
    X = (torch.randn(R, d, device="cuda", generator=g) * 3.0).to(torch.bfloat16)
    perm = torch.randperm(R, device="cuda", generator=g)[:Cl * M].to(torch.int32)
    table = ops.zs_class_embed(X, perm, Cl, M)
    ref = F.normalize(F.normalize(X.float()[perm.long()].view(Cl, M, d), dim=-1).mean(1), dim=-1).t()
    assert table.shape == (d, Cl) and table.dtype == torch.float32
    torch.testing.assert_close(table, ref, rtol=1e-5, atol=2e-6)
    assert torch.equal(ops.zs_class_embed(X, perm, Cl, M), table)


@pytest.mark.parametrize("B", [1, 37, 256])
def test_zs_logits_topk(pkg, B):
    from ml_cvnets_b200 import ops
    Cl, d = 1000, 512
    g = torch.Generator(device="cuda").manual_seed(B)
    img = F.normalize(torch.randn(B, d, device="cuda", generator=g), dim=-1).to(torch.bfloat16)
    table = F.normalize(torch.randn(d, Cl, device="cuda", generator=g), dim=0).contiguous()
    ref = 100.0 * img.float() @ table
    order = ref.argsort(dim=1, descending=True)
    pick = torch.randint(0, 8, (B,), device="cuda", generator=g)  # targets ranked 0..7: hits and misses of both k
    targets = order[torch.arange(B, device="cuda"), pick].contiguous()
    targets[::5] = torch.randint(0, Cl, (targets[::5].numel(),), device="cuda", generator=g)
    hits = torch.zeros(2, device="cuda", dtype=torch.int64)
    logits = ops.zs_logits_topk(img, table, 100.0, targets, hits)
    torch.testing.assert_close(logits, ref, rtol=1e-5, atol=1e-4)
    top = logits.topk(6, dim=1).values
    assert bool((top[:, :-1] > top[:, 1:]).all()), "inputs must be tie-free near the top"
    pred = logits.topk(5, 1, True, True).indices
    hit = pred.eq(targets.view(-1, 1))
    want = [int(hit[:, :1].sum()), int(hit.sum())]
    assert hits.tolist() == want
    if B > 1:
        assert 0 < want[0] <= want[1] < B
    for _ in range(2):  # counts only, added into the same counters
        assert ops.zs_logits_topk(img, table, 100.0, targets, hits, want_logits=False) is None
    assert hits.tolist() == [3 * w for w in want]


# ---------------------------------------------------------------------------------------------------------------------------- model
def test_zero_shot_against_reference_fixture(pkg, fx):
    model, shapes = small_clip(pkg, fx)
    tokens, images = fx["tokens"].cuda(), O.seeded_input((8, 3, 224, 224), fx["x_seed"]).cuda()
    table = model.zero_shot_table(tokens)
    logits = model.zero_shot_logits(images, table)
    _, txt, _ = model(images, tokens)
    assert torch.equal(txt, table)
    assert torch.equal(model.zero_shot_logits(images, tokens), logits)
    Pa = O.clone_params(O.seeded_fill_(dict(shapes), fx["seed"]), device="cuda", requires_grad=False)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.bfloat16):
        ta = zero_shot_table(Pa, tokens, text_layers=4, text_heads=4).float()
        la = 100.0 * image_features(Pa, images).float() @ ta
    et, el = rel_l2(table, fx["table"]), rel_l2(logits, fx["zero_shot_image_logits"])
    eta, ela = rel_l2(ta, fx["table"]), rel_l2(la, fx["zero_shot_image_logits"])
    print(f"[zero-shot] rel-L2 vs the reference: table {et:.4g} (autocast {eta:.4g}), logits {el:.4g} (autocast {ela:.4g})")
    assert et <= max(2e-2, 1.5 * eta) and el <= max(2e-2, 1.5 * ela)
    ref = fx["zero_shot_image_logits"].cuda()
    s = ref.sort(dim=1, descending=True).values
    resolved = (s[:, 0] - s[:, 1]) > 2.0 * float((la - ref).abs().max())  # rows whose top-1 the same-precision comparator cannot flip
    assert torch.equal(logits.argmax(1)[resolved], ref.argmax(1)[resolved])
    hits = torch.zeros(2, device="cuda", dtype=torch.int64)
    labels = fx["labels"].cuda()
    model.zero_shot_logits(images, table, targets=labels, hits=hits)
    hit = logits.topk(5, 1, True, True).indices.eq(labels.view(-1, 1))
    assert hits.tolist() == [int(hit[:, :1].sum()), int(hit.sum())]
    acc = pkg.ZeroShotAccuracy(model, tokens)
    acc.update(images[:5], labels[:5])
    acc.update(images[5:], labels[5:])
    res = acc.compute()
    assert res == {"top1": 100.0 * hits[0].item() / 8, "top5": 100.0 * hits[1].item() / 8}
    print(f"[zero-shot] top-1 / top-5 {res['top1']} / {res['top5']} (reference {fx['top1']} / {fx['top5']}); {int(resolved.sum())} of 8 rows resolved")


def test_token_budget_does_not_change_the_table(pkg, fx):
    model, _ = small_clip(pkg, fx)
    tokens = fx["tokens"].cuda()
    t1 = model.zero_shot_table(tokens)
    model.text_encoder.zero_shot_token_budget = 16  # one or two rows per tower call
    t2 = model.zero_shot_table(tokens)
    assert torch.equal(t1, t2)


def _random_rows(n, L, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    rows = torch.randint(1, vocab - 1, (n, L), generator=g)
    rows[torch.arange(n), torch.randint(1, L, (n,), generator=g)] = vocab - 1  # the end-of-text token is the highest id
    return rows.cuda()


@pytest.mark.parametrize("geometry", ["small16", "base77"])
def test_truncated_encoding_matches_full_length(pkg, fx, geometry):
    """Each caption runs at its causal prefix: the projected end-of-text features must match a full-length encoding of the same rows."""
    from ml_cvnets_b200.models_clip import TextTransformer, default_clip_opts
    if geometry == "small16":
        enc = small_clip(pkg, fx)[0].text_encoder
        rows = fx["tokens"][0].reshape(-1, 16).cuda()
    else:
        torch.manual_seed(0)
        enc = TextTransformer(default_clip_opts(), projection_dim=512).cuda().eval()
        rows = _random_rows(300, 77, 49408, 5)
    with torch.no_grad():
        feats, where = enc._encode_rows(rows, None)
        full = enc._tower(rows, enc.positional_embedding.pos_embed.pos_embed, None)
    trunc = feats[where]
    e = rel_l2(trunc, full)
    print(f"[zero-shot] {geometry}: truncated vs full-length rel-L2 {e:.3g}, bitwise equal: {torch.equal(trunc, full)}")
    assert e <= 1e-3


def test_3d_batch(pkg, fx):
    model, _ = small_clip(pkg, fx)
    enc = model.text_encoder
    tok3 = fx["tokens_3d"].cuda()
    with torch.no_grad():
        out = enc(tok3)
        flat = enc(tok3.reshape(-1, 16)).view(3, 2, -1)
    assert out.shape == (3, 2, 128)
    e = rel_l2(out, flat)
    print(f"[zero-shot] 3-D vs 2-D of the flattened tokens: rel-L2 {e:.3g}, bitwise equal: {torch.equal(out, flat)}; "
          f"vs the reference {rel_l2(out, fx['text_3d']):.4g}")
    assert torch.equal(out, flat) and rel_l2(out, fx["text_3d"]) <= 2e-2
    model.train()
    grad_out = enc(tok3)  # with autograd: the 2-D path on the flattened tokens
    with torch.no_grad():
        flat_train = enc(tok3.reshape(-1, 16)).view(3, 2, -1)
    assert torch.equal(grad_out.detach(), flat_train) and grad_out.requires_grad


def test_4d_in_training_raises(pkg, fx):
    model, _ = small_clip(pkg, fx)
    model.train()
    tokens = fx["tokens"].cuda()
    with pytest.raises(NotImplementedError):
        model.text_encoder(tokens)
    with pytest.raises(NotImplementedError):
        model.zero_shot_logits(O.seeded_input((2, 3, 224, 224), 1).cuda(), tokens)


def test_zero_shot_cache(pkg, fx):
    tokens = fx["tokens"].cuda()
    other = tokens.flip(1).contiguous()  # the classes in reverse order: another table
    model, _ = small_clip(pkg, fx, **{"model.multi_modal_image_text.clip.cache_text_features_zero_shot": True})
    t1 = model.zero_shot_table(tokens)
    assert model.zero_shot_table(other) is t1  # cached, as the reference does
    model.clear_zero_shot_cache()
    t2 = model.zero_shot_table(other)
    assert torch.equal(t2, t1.flip(1))
    model.train()
    assert model.cached_text_features is None  # dropped on train(): the weights may change
    model.eval()
    assert torch.equal(model.zero_shot_table(tokens), t1)
    plain, _ = small_clip(pkg, fx)
    assert plain.zero_shot_table(tokens) is not plain.zero_shot_table(tokens) and plain.cached_text_features is None

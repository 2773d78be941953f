"""Kernel-level parity at the edges (-m gpu): the C-ABI entry points that the model and module tests reach at one shape only, called directly
at the shapes, layouts and boundary values where kernels go wrong, against fp32 / fp64 torch restatements on the same bf16-rounded inputs.
Pure data movement is compared bitwise; kernels that round once are held to one bf16 ulp; the others use close() of test_kernels_gpu."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernels_gpu import BF, _mha_ref, bf, close, rnd  # noqa: E402

pytestmark = pytest.mark.gpu

LN2 = math.log(2.0)


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ml_cvnets_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def lib(ops):
    from ml_cvnets_b200 import _lib as L
    return L.load()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def bf_ulp(r):
    """spacing of bf16 numbers at |r| (r already bf16-representable); the smallest normal spacing at 0"""
    r = r.float()
    _, e = torch.frexp(r)
    ulp = torch.ldexp(torch.ones_like(r), (e - 8).to(torch.int32))
    return torch.where(r == 0, torch.full_like(r, 2.0 ** -133), ulp)


def within_ulp(a, ref, what="", atol=0.0):
    """a (bf16) is within one bf16 ulp of the bf16 rounding of the high-precision value ref (plus an absolute floor for cancellation)"""
    r = ref.to(BF)
    err = (a.float() - r.float()).abs()
    bad = err > bf_ulp(r) + atol
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} outside 1 bf16 ulp, e.g. got {a.flatten()[bad.flatten()][:4].tolist()} " \
                          f"want {ref.flatten()[bad.flatten()][:4].tolist()}"


def same(a, b, what=""):
    assert a.shape == b.shape and a.dtype == b.dtype, f"{what}: {tuple(a.shape)} {a.dtype} vs {tuple(b.shape)} {b.dtype}"
    eq = (a == b) | (torch.isnan(a.float()) & torch.isnan(b.float())) if a.is_floating_point() else (a == b)
    assert bool(eq.all()), f"{what}: {int((~eq).sum())}/{eq.numel()} elements differ"


# ------------------------------------------------------------------------------------------- stand-alone GroupNorm(1, C) backward
# cgs * floor(256 / cgs) threads (cgs = C / 8) is not a multiple of 32 at C = 24, 40, 80, 96, 192: the per-sample sums must still be right.
# (3, 16384) makes more row chunks per sample than the grid cap at C >= 192 (and (8, 1024) at C = 2048): the chunks-over-cap branch.
@pytest.mark.parametrize("C", [8, 24, 40, 80, 96, 192, 256, 2048])
@pytest.mark.parametrize("B,rps", [(1, 1), (3, 7), (8, 1024), (3, 16384)])
def test_gn_bwd_standalone(ops, B, rps, C):
    M = B * rps
    X = bf(rnd(M, C, seed=501) * 1.3 + 0.4)
    gamma = 1 + 0.2 * rnd(C, seed=502)
    beta = 0.1 * rnd(C, seed=503)
    xs = X.double().view(B, -1)
    mean, var = xs.mean(1), xs.var(1, unbiased=False)
    gn = torch.stack([mean, (var + 1e-5).rsqrt()]).float()
    xh = ((X.double().view(B, rps, C) - gn[0].double()[:, None, None]) * gn[1].double()[:, None, None])
    # an upstream gradient with a per-sample mean and a component along xhat: the mean terms of dx are then of the size of dx itself, so a wrong
    # per-sample sum cannot hide under the element-wise bound
    V = bf(1 + 0.5 * xh.float().view(M, C) + 0.3 * rnd(M, C, seed=504))
    DR = bf(rnd(M, C, seed=505)) if rps % 2 else None

    def run():
        dg = torch.zeros(C, device="cuda", dtype=torch.float64)
        db = torch.zeros(C, device="cuda", dtype=torch.float64)
        ws = torch.zeros(2, B, device="cuda", dtype=torch.float64)
        DX = ops.gn_bwd(V, X, gn, gamma, rps * C, B, rps, dg, db, ws, DRES=DR)
        torch.cuda.synchronize()
        return DX, dg, db, ws

    DX, dg, db, ws = run()
    v = V.double().view(B, rps, C)
    g = v * gamma.double()
    # fp32 partial sums inside the kernel: a few 1e-6 of the sum of |terms|; one lane's share of a 256-thread CTA would be ~4e-3
    gx = g * xh
    for what, got, ref, scale in (("sum g", ws[0], g.view(B, -1).sum(1), g.abs().view(B, -1).sum(1)),
                                  ("sum g*xhat", ws[1], gx.view(B, -1).sum(1), gx.abs().view(B, -1).sum(1))):
        err = (got - ref).abs()
        assert bool((err <= 3e-5 * scale).all()), f"{what}: per-sample error {err.tolist()} vs sum|terms| {scale.tolist()}"
    vx = v * xh
    for what, got, ref, scale in (("dbeta", db, v.sum((0, 1)), v.abs().sum((0, 1))), ("dgamma", dg, vx.sum((0, 1)), vx.abs().sum((0, 1)))):
        err = (got - ref).abs()
        assert bool((err <= 3e-5 * scale + 1e-9).all()), f"{what}: max err {float(err.max()):.3g}"
    xv = X.float().view(B, rps, C).permute(0, 2, 1).contiguous().requires_grad_(True)
    out = F.group_norm(xv, 1, gamma, beta, 1e-5)
    out.backward(V.float().view(B, rps, C).permute(0, 2, 1))
    ref = xv.grad.permute(0, 2, 1).reshape(M, C) + (DR.float() if DR is not None else 0)
    close(DX, ref, what="gn dx")
    DX2, dg2, db2, ws2 = run()
    same(DX2, DX, "dx rerun")
    same(dg2, dg, "dgamma rerun")
    same(db2, db, "dbeta rerun")
    same(ws2, ws, "per-sample sums rerun")


# ------------------------------------------------------------------------------------------- attention head dims of MobileViT-v1
def _lse_ref(qkv, B, S, H, c, scale, amask, kpm):
    x = qkv.float().view(B, S, 3, H, c).permute(2, 0, 3, 1, 4)
    att = (x[0] * scale) @ x[1].transpose(-1, -2)
    if amask is not None:
        att = att + amask[:, None]
    if kpm is not None:
        att = att.masked_fill(kpm[:, None, None, :].bool(), float("-inf"))
    return torch.logsumexp(att, dim=-1) / LN2  # [B, H, S], base 2


def _masks(B, S, mask):
    amask = kpm = None
    if mask == "causal":
        amask = torch.full((S, S), float("-inf"), device="cuda").triu(1)[None].repeat(B, 1, 1).contiguous()
    if mask == "padding":
        kpm = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
        kpm[:, S - max(1, S // 5):] = 1
    return amask, kpm


def _check_mha(ops, qkv, B, S, H, c, mask, seed):
    C = H * c
    dO = bf(rnd(B * S, C, seed=seed))
    amask, kpm = _masks(B, S, mask)
    scale = c ** -0.5
    O, LSE = ops.mha_fwd(qkv, B, S, H, c, scale, attn_mask=amask, key_padding_mask=kpm)
    x = qkv.float().requires_grad_(True)
    ref = _mha_ref(x, B, S, H, c, scale, amask, kpm)
    close(O, ref.detach(), what="mha fwd")
    lse = _lse_ref(qkv, B, S, H, c, scale, amask, kpm)
    err = float((LSE - lse).abs().max())
    assert err <= 1e-4 * float(lse.abs().max()) + 1e-4, f"LSE: max err {err:.3g}"
    ref.backward(dO.float())
    DQKV = ops.mha_bwd(qkv, O, dO, LSE, B, S, H, c, scale, attn_mask=amask, key_padding_mask=kpm)
    close(DQKV[:, :3 * C], x.grad[:, :3 * C], rtol=3e-2, atol=2e-2 * float(x.grad.abs().max()) + 1e-6, what="mha bwd")


# XXS heads 16 / 20 / 24, XS 24 / 30 / 36, S 36 / 48 / 60 (4 heads); H = 3 where 3 * head_dim keeps the rows 16-byte aligned.  Head h starts at
# column h * head_dim: 8- but not 16-byte aligned for 20 / 36 / 60, 4-byte aligned for 30
@pytest.mark.parametrize("c,H", [(8, 4), (8, 3), (20, 4), (24, 4), (24, 3), (30, 4), (36, 4), (48, 3), (48, 4), (60, 4)])
@pytest.mark.parametrize("S", [16, 64, 144, 256])
@pytest.mark.parametrize("mask", ["none", "causal", "padding"])
def test_mha_mobilevit_v1_head_dims(ops, c, H, S, mask):
    B = 2
    qkv = bf(rnd(B * S, 3 * H * c, seed=511))
    _check_mha(ops, qkv, B, S, H, c, mask, seed=512)


@pytest.mark.parametrize("mask", ["none", "padding"])
def test_mha_strided_qkv_view(ops, mask):
    """QKV as a column slice of a wider projection (ldq = 3 H c + 8): the NaN-filled pad columns must never be read"""
    B, S, H, c = 2, 144, 4, 20
    big = torch.full((B * S, 3 * H * c + 8), float("nan"), device="cuda", dtype=BF)
    big[:, :3 * H * c] = bf(rnd(B * S, 3 * H * c, seed=513))
    qkv = big[:, :3 * H * c]
    assert qkv.stride(0) == 3 * H * c + 8
    _check_mha(ops, qkv, B, S, H, c, mask, seed=514)


# ------------------------------------------------------------------------------------------- cross-entropy, called directly
def _padded_logits(B, C, seed, scale=3.0):
    ld = (C + 7) // 8 * 8 + 8
    big = torch.full((B, ld), 1e4, device="cuda", dtype=BF)  # pad columns: large values that must not enter any sum
    big[:, :C] = bf(rnd(B, C, scale=scale, seed=seed))
    return big, ld


def _ce_run(ops, logits, C, target, ignore, smoothing, ldd, gout=None, gscale=None, mix=None, logit_scale=None, dlogit_scale=None):
    loss, lse, nv = ops.ce_fwd(logits, C, target, ignore, smoothing, mix=mix, logit_scale=logit_scale)
    d = ops.ce_bwd(logits, C, target, ignore, smoothing, lse, nv, gout, gscale, ldd, mix=mix, logit_scale=logit_scale, dlogit_scale=dlogit_scale)
    torch.cuda.synchronize()
    return loss, lse, nv, d


def _check_dlogits(d, ref, C, what):
    if d.shape[1] > C:
        assert float(d[:, C:].float().abs().max()) == 0.0, f"{what}: pad columns of dlogits are not zero"
    assert bool(torch.isfinite(d.float()).all()), f"{what}: non-finite dlogits"
    close(d[:, :C], ref, what=what)


# B > 32 rows: more rows than the forward kernel's 32 warps
@pytest.mark.parametrize("B", [1, 33, 1000, 4096])
@pytest.mark.parametrize("C", [2, 37, 1000])
@pytest.mark.parametrize("smoothing", [0.0, 0.1])
def test_ce_direct(ops, B, C, smoothing):
    ignore = -100
    logits, ld = _padded_logits(B, C, seed=521)
    target = torch.randint(0, C, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(522))
    if B > 1:
        target[::5] = ignore
    gout = torch.tensor([0.7], device="cuda")
    gscale = torch.tensor([1024.0], device="cuda")
    ldd = ld
    loss, lse, nv, d = _ce_run(ops, logits, C, target, ignore, smoothing, ldd, gout, gscale)
    lg = logits[:, :C].float().requires_grad_(True)
    ref = F.cross_entropy(lg, target, ignore_index=ignore, label_smoothing=smoothing)
    ref.backward()
    n_valid = int((target != ignore).sum())
    assert float(nv) == n_valid
    lse_ref = torch.logsumexp(lg.detach(), dim=1)
    assert float((lse - lse_ref).abs().max()) <= 1e-5 * float(lse_ref.abs().max()) + 1e-5
    assert abs(float(loss) - float(ref)) <= 3e-5 * abs(float(ref)) + 1e-6, (float(loss), float(ref))
    _check_dlogits(d, lg.grad * 0.7 * 1024.0, C, "dlogits")


def test_ce_all_rows_ignored(ops):
    B, C, ignore = 40, 37, 3
    logits, ld = _padded_logits(B, C, seed=523)
    target = torch.full((B,), ignore, device="cuda", dtype=torch.int64)
    for sm in (0.0, 0.1):
        loss, lse, nv, d = _ce_run(ops, logits, C, target, ignore, sm, ld)
        assert float(loss) == 0.0 and float(nv) == 0.0
        assert bool(torch.isfinite(lse).all())
        assert float(d.float().abs().max()) == 0.0 and not bool(torch.isnan(d.float()).any())


@pytest.mark.parametrize("B,C", [(1, 37), (33, 37), (1000, 1000)])
@pytest.mark.parametrize("smoothing", [0.0, 0.1])
def test_ce_mixed_targets(ops, B, C, smoothing):
    """mixup / cutmix targets lam * onehot(y) + (1 - lam) * onehot(y.roll(1)): row 0 pairs with row B - 1, B = 1 with itself"""
    lam = 0.3
    logits, ld = _padded_logits(B, C, seed=524)
    target = torch.randint(0, C, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(525))
    if B > 5:
        target[5] = target[4]  # t2 == t
    for mode in (1.0, 2.0):
        mix = torch.tensor([mode, lam, 0, 0, 0, 0], device="cuda")
        gout = torch.tensor([1.3], device="cuda")
        loss, lse, nv, d = _ce_run(ops, logits, C, target, -1, smoothing, ld, gout=gout, mix=mix)
        lg = logits[:, :C].float().requires_grad_(True)
        soft = lam * F.one_hot(target, C).float() + (1 - lam) * F.one_hot(target.roll(1), C).float()
        ref = F.cross_entropy(lg, soft, label_smoothing=smoothing)
        ref.backward()
        assert float(nv) == B
        assert abs(float(loss) - float(ref)) <= 3e-5 * abs(float(ref)) + 1e-6, (mode, float(loss), float(ref))
        _check_dlogits(d, lg.grad * 1.3, C, f"mixed dlogits (mode {mode})")


@pytest.mark.parametrize("BC", [33, 256])
@pytest.mark.parametrize("exp_s", [1 / 0.07, 99.0, 150.0])
def test_ce_logit_scale(ops, BC, exp_s):
    """CLIP's temperature: loss of clamp(exp(s), max=100) * raw similarities; d s is exactly 0 once the clamp is active"""
    raw = bf(torch.tanh(rnd(BC, BC, scale=2.0, seed=526)))
    raw[0, 0], raw[1, 1] = 1.0, -1.0  # scaled logits reach +-100
    labels = torch.arange(BC, device="cuda")
    s = torch.tensor([math.log(exp_s)], device="cuda")
    ds = torch.zeros(1, device="cuda")
    loss, lse, nv, d = _ce_run(ops, raw, BC, labels, -1, 0.0, BC, logit_scale=s, dlogit_scale=ds)
    rv = raw.float().requires_grad_(True)
    sv = s.clone().requires_grad_(True)
    ref = F.cross_entropy(torch.clamp(sv.exp(), max=100.0) * rv, labels)
    ref.backward()
    assert abs(float(loss) - float(ref)) <= 1e-5 * abs(float(ref)) + 1e-5, (float(loss), float(ref))
    _check_dlogits(d, rv.grad, BC, "d raw")
    if exp_s > 100:
        assert float(ds) == 0.0 and float(sv.grad) == 0.0
    else:
        assert abs(float(ds) - float(sv.grad)) <= 1e-3 * abs(float(sv.grad)) + 1e-4, (float(ds), float(sv.grad))


# ------------------------------------------------------------------------------------------- CLIP text-tower edges
@pytest.mark.parametrize("B,S,C,V,with_pos", [(256, 77, 512, 1000, True), (3, 5, 8, 4, True), (4, 16, 64, 50, False)])
def test_embedding(ops, B, S, C, V, with_pos):
    """B * S * C / 8 = 1.26M items at (256, 77, 512): the grid-stride loops run past the 16-per-SM grid cap"""
    g = torch.Generator(device="cuda").manual_seed(531)
    tokens = torch.randint(0, V, (B, S), device="cuda", generator=g)
    tokens[:, 0] = 0
    tokens[:, -1] = V - 1
    tokens[0, :] = tokens[0, 0]  # one id many times in a row
    table = rnd(V, C, seed=532)
    pos = rnd(S, C, seed=533) if with_pos else None
    out = ops.embedding_fwd(tokens, table, pos)
    ref = table[tokens] + (pos[None] if with_pos else 0)
    same(out, ref.to(BF), "embedding fwd")
    dout = bf(rnd(B, S, C, seed=534))
    dtable = torch.zeros(V, C, device="cuda")
    dpos = torch.zeros(S, C, device="cuda") if with_pos else None
    ops.embedding_bwd(dout, tokens, dtable, dpos)
    flat = dout.double().view(-1, C)
    idx = tokens.view(-1)
    ref_t = torch.zeros(V, C, device="cuda", dtype=torch.float64).index_add_(0, idx, flat)
    abs_t = torch.zeros(V, C, device="cuda", dtype=torch.float64).index_add_(0, idx, flat.abs())
    assert bool(((dtable.double() - ref_t).abs() <= 1e-5 * abs_t).all()), "dtable"
    if with_pos:
        d = dout.double()
        assert bool(((dpos.double() - d.sum(0)).abs() <= 1e-5 * d.abs().sum(0)).all()), "dpos"


@pytest.mark.parametrize("C", [8, 768, 1032])
def test_eot_gather(ops, C):
    """argmax of the token ids with the first maximum winning ties (torch.argmax), end-of-text at 0 and at S - 1; C = 1032 loops the row copy"""
    B, S = 6, 77
    g = torch.Generator(device="cuda").manual_seed(541)
    tokens = torch.randint(0, 1000, (B, S), device="cuda", generator=g)
    tokens[0, 0] = 5000                               # eot first
    tokens[1, S - 1] = 5000                           # eot last
    tokens[2, 10] = tokens[2, 40] = 5000              # tie: 10 wins
    tokens[3, :] = 7                                  # all equal: 0 wins
    tokens[4, 0] = tokens[4, S - 1] = 5000            # tie at both ends: 0 wins
    tokens[5, 30] = tokens[5, 31] = tokens[5, 76] = 4000
    X = bf(rnd(B, S, C, seed=542))
    out, idx = ops.eot_gather_fwd(X, tokens)
    first = torch.stack([(tokens[b] == tokens[b].max()).nonzero()[0, 0] for b in range(B)])
    assert first.tolist() == [0, S - 1, 10, 0, 0, 30]
    same(idx.long(), first, "eot index")
    same(out, X[torch.arange(B), first], "eot gather fwd")
    dout = bf(rnd(B, C, seed=543))
    dX = ops.eot_gather_bwd(dout, idx, B, S, C)
    ref = torch.zeros(B, S, C, device="cuda", dtype=BF)
    ref[torch.arange(B), first] = dout
    same(dX, ref, "eot gather bwd")


@pytest.mark.parametrize("M", [1, 13, 100])
@pytest.mark.parametrize("C", [8, 512, 520, 1024])
def test_l2norm(ops, M, C):
    """F.normalize(x, dim=-1): row norms from 1e-6 to 1e6, an all-zero row (output 0, gradient dy / eps, no NaN); M not a multiple of 8"""
    x = rnd(M, C, seed=551) * torch.logspace(-6, 6, M, device="cuda")[:, None]
    if M > 1:
        x[M // 2] = 0
    X = bf(x)
    Y, inv = ops.l2norm_fwd(X)
    xv = X.float().requires_grad_(True)
    y = F.normalize(xv, dim=-1)
    within_ulp(Y, y.detach(), "l2norm fwd")
    norm = X.double().norm(dim=1)
    inv_ref = 1.0 / norm.clamp_min(1e-12)
    assert bool(((inv.double() - inv_ref).abs() <= 1e-5 * inv_ref).all()), "inv_norm"
    dy = bf(rnd(M, C, seed=552))
    y.backward(dy.float())
    DX = ops.l2norm_bwd(dy, Y, inv)
    assert bool(torch.isfinite(DX.float()).all())
    # per-row relative error: the rows differ by twelve orders of magnitude.  The backward reads the bf16 output y and rounds dx: a row of 8
    # values can reach 5e-3, the root mean square over rows stays near bf16 rounding of an exact result
    err = (DX.double() - xv.grad.double()).norm(dim=1) / xv.grad.double().norm(dim=1)
    assert float(err.max()) <= 8e-3, f"l2norm bwd: per-row rel-L2 up to {float(err.max()):.3g}"
    assert float(err.square().mean().sqrt()) <= 4e-3, f"l2norm bwd: rms of the per-row rel-L2 {float(err.square().mean().sqrt()):.3g}"
    if M > 1:
        assert float(Y[M // 2].float().abs().max()) == 0.0


@pytest.mark.parametrize("R,C", [(1, 8), (77, 520), (33, 1000)])
def test_transpose_and_add(ops, R, C):
    X = bf(rnd(R, C, seed=561))
    same(ops.transpose_bf16(X), X.t().contiguous(), "transpose")
    Bf = rnd(R, C, seed=562)
    same(ops.add_bf16_f32(X, Bf), (X.float() + Bf).to(BF), "add")
    same(ops.add_bf16_f32(None, Bf), Bf.to(BF), "add, A = None")


@pytest.mark.parametrize("n", [1000, 4096 * 256 + 1000])
def test_add_bf16_f32_lengths(ops, n):
    """n not a multiple of the 256-thread CTA, and n > 4096 CTAs x 256 (the grid cap): the loop strides"""
    A = bf(rnd(n, seed=563))
    Bf = rnd(n, seed=564)
    same(ops.add_bf16_f32(A, Bf), (A.float() + Bf).to(BF), "add")


# ------------------------------------------------------------------------------------------- im2col / col2im
def _unfold_ref(x, k, s, p):
    """F.unfold in the kernel's column order (u, v, ci): [B * L, k * k * Cin]"""
    B, Cin = x.shape[:2]
    u = F.unfold(x, kernel_size=k, stride=s, padding=p)  # [B, Cin * k * k, L], rows (ci, u, v)
    L = u.shape[-1]
    return u.view(B, Cin, k * k, L).permute(0, 3, 2, 1).reshape(B * L, k * k * Cin)


CONV_GEOM = [(4, 4, 1, 16, 16), (2, 2, 0, 14, 10), (3, 1, 1, 9, 12), (3, 2, 1, 15, 13), (2, 2, 0, 7, 9)]


@pytest.mark.parametrize("k,s,p,H,W", CONV_GEOM)
@pytest.mark.parametrize("Cin", [8, 64])
def test_im2col_col2im_nhwc(ops, k, s, p, H, W, Cin):
    B = 3
    Xn = bf(rnd(B * H * W, Cin, seed=571))
    x = Xn.view(B, H, W, Cin).permute(0, 3, 1, 2)  # logical NCHW, channels-last memory: the 16-byte gather path
    A, Ho, Wo = ops.im2col(x, k, s, p)
    ref = _unfold_ref(x.float(), k, s, p)
    same(A, ref.to(BF), "im2col nhwc")
    # col2im: adjoint, gathered in fp32; fp64 fold as the truth.  dA as a view with lda = k k Cin + 8 (NaN pad, never read)
    kk = k * k * Cin
    big = torch.full((B * Ho * Wo, kk + 8), float("nan"), device="cuda", dtype=BF)
    big[:, :kk] = bf(rnd(B * Ho * Wo, kk, seed=572))
    dA = big[:, :kk]
    dX = ops.col2im(dA, B, Cin, H, W, k, s, p)
    cols = dA.double().view(B, Ho * Wo, k * k, Cin).permute(0, 3, 2, 1).reshape(B, Cin * k * k, Ho * Wo)
    fold = F.fold(cols, output_size=(H, W), kernel_size=k, stride=s, padding=p).permute(0, 2, 3, 1).reshape(B * H * W, Cin)
    within_ulp(dX, fold, "col2im")
    lhs = float((dX.double() * Xn.double()).sum())
    rhs = float((dA.double() * A.double()).sum())
    bound = 2.0 ** -8 * float((dX.double().abs() * Xn.double().abs()).sum())
    assert abs(lhs - rhs) <= bound, f"<col2im(dA), x> = {lhs} vs <dA, im2col(x)> = {rhs}"


@pytest.mark.parametrize("k,s,p,H,W", CONV_GEOM)
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
def test_im2col_generic(ops, k, s, p, H, W, layout):
    """3-channel fp32 images (the ViT / CLIP stem input) and lda > k k Cin: the element-wise gather, pad columns zero"""
    B, Cin = 2, 3
    x = rnd(B, Cin, H, W, seed=573)
    if layout == "channels_last":
        x = x.contiguous(memory_format=torch.channels_last)
    kk = k * k * Cin
    lda = (kk + 7) // 8 * 8 + 8
    A, Ho, Wo = ops.im2col(x, k, s, p, lda=lda)
    same(A[:, :kk], _unfold_ref(x, k, s, p).to(BF), "im2col generic")
    assert float(A[:, kk:].float().abs().max()) == 0.0


# ------------------------------------------------------------------------------------------- MobileViT-v1 unfolding / folding, concat
def _unfold_v1(fm, ph, pw):
    """mobilevit_block.py:186-230 (no resize branch): [B, C, H, W] -> [B * P, N, C]"""
    B, C, H, W = fm.shape
    nh, nw = H // ph, W // pw
    t = fm.reshape(B * C * nh, ph, nw, pw).transpose(1, 2).reshape(B, C, nh * nw, ph * pw).transpose(1, 3)
    return t.reshape(B * ph * pw, nh * nw, C)


def _fold_v1(patches, B, C, H, W, ph, pw):
    """mobilevit_block.py:232-267: [B * P, N, C] -> [B, C, H, W]"""
    nh, nw = H // ph, W // pw
    p = patches.contiguous().view(B, ph * pw, nh * nw, C).transpose(1, 3)
    return p.reshape(B * C * nh, nw, ph, pw).transpose(1, 2).reshape(B, C, H, W)


@pytest.mark.parametrize("B,H,W,ph,pw", [(2, 8, 12, 2, 2), (1, 16, 6, 2, 2), (3, 12, 8, 4, 2)])
@pytest.mark.parametrize("C", [8, 144])
def test_patch_permute(ops, B, H, W, ph, pw, C):
    X = bf(rnd(B * H * W, C, seed=581))
    fm = X.view(B, H, W, C).permute(0, 3, 1, 2)
    T = ops.patch_permute(X, B, H, W, ph, pw, inverse=False)
    ref = _unfold_v1(fm, ph, pw).reshape(-1, C)
    same(T, ref, "unfolding")
    back = ops.patch_permute(T, B, H, W, ph, pw, inverse=True)
    same(back, X, "folding(unfolding(x))")
    G = bf(rnd(B * H * W, C, seed=582))
    fold_ref = _fold_v1(G.view(B * ph * pw, -1, C), B, C, H, W, ph, pw).permute(0, 2, 3, 1).reshape(-1, C)
    same(ops.patch_permute(G, B, H, W, ph, pw, inverse=True), fold_ref, "folding")


@pytest.mark.parametrize("M", [1, 1000, 50000])
@pytest.mark.parametrize("C1,C2", [(8, 96), (96, 8)])
def test_concat2_split2(ops, M, C1, C2):
    """M = 50000 at 13 chunks per row exceeds the grid cap: the loops stride"""
    A, Bt = bf(rnd(M, C1, seed=591)), bf(rnd(M, C2, seed=592))
    out = ops.concat2(A, Bt)
    same(out, torch.cat([A, Bt], dim=1), "concat2")
    da, db = ops.split2(out, C1, C2)
    same(da, A, "split2 first")
    same(db, Bt, "split2 second")


# ------------------------------------------------------------------------------------------- stand-alone activations
ACTS = [(0, F.silu), (1, F.gelu), (2, F.relu), (3, F.hardswish), (4, F.hardsigmoid), (5, torch.sigmoid)]


@pytest.mark.parametrize("kind,fn", ACTS, ids=["silu", "gelu", "relu", "hardswish", "hardsigmoid", "sigmoid"])
def test_act_kinds(ops, kind, fn):
    """values at the kinks (-3, 0, 3) and out to |x| = 20; gradients follow torch's conventions at the kinks; 8M elements run the grid-stride
    loop past the 16-per-SM grid cap"""
    kinks = torch.tensor([-3.0, 0.0, 3.0, -20.0, 20.0, -2.984375, 2.984375, -3.015625, 3.015625], device="cuda")
    grid = torch.linspace(-20, 20, 4000, device="cuda")
    x = torch.cat([kinks, grid, rnd(8 * 2 ** 20 - kinks.numel() - grid.numel(), scale=4.0, seed=601)])
    X = bf(x)
    Y = ops.act_fwd(X, kind)
    xv = X.float().requires_grad_(True)
    y = fn(xv)
    # SiLU's sigmoid is tanh.approx.f32 (as in every fused SiLU of the library): ~1e-4 absolute, visible where silu' crosses zero
    atol = 1e-4 if kind == 0 else 1e-5
    within_ulp(Y, y.detach(), f"act {kind} fwd", atol=atol)
    DY = bf(1 + 0.5 * rnd(X.numel(), seed=602))
    DY[:kinks.numel()] = 1.0
    y.backward(DY.float())
    DX = ops.act_bwd(DY, X, kind)
    within_ulp(DX, xv.grad, f"act {kind} bwd", atol=atol)
    # the one-sided derivatives torch picks at the kinks -3, 0, 3, exactly (torch 2.x: hardswish' = 0 at -3 and 1 at 3, hardsigmoid' = 0 at +-3,
    # relu' = 0 at 0); bf16 inputs hit +-3 exactly about once per 800 values of N(0, 4^2)
    if kind in (2, 3, 4):
        same(DX[:3], xv.grad[:3].to(BF), f"act {kind} bwd at the kinks")


# ------------------------------------------------------------------------------------------- linear cross-attention
@pytest.mark.parametrize("Mp,N", [(16, 64), (64, 16)])
@pytest.mark.parametrize("d", [16, 128, 192])
def test_linattn_cross(ops, Mp, N, d):
    """LinearSelfAttention._forward_cross_attn (linear_attention.py:163-207): query + key from x_prev (Mp patches), value from x (N patches)"""
    B, P = 2, 4
    ld = 2 * d + 8
    QKP = bf(rnd(B * P * Mp, ld, seed=611))
    QKVX = bf(rnd(B * P * N, ld, seed=612))
    DO = bf(rnd(B * P * N, d, seed=613))

    def run():
        O, S, CTX = ops.linattn_cross_fwd(QKP, QKVX, B, P, Mp, N, d)
        db = torch.zeros(ld, device="cuda")
        DQKP, DQKVX = ops.linattn_cross_bwd(QKP, QKVX, DO, S, CTX, B, P, Mp, N, d, dbias=db)
        torch.cuda.synchronize()
        return O, S, CTX, DQKP, DQKVX, db

    O, S, CTX, DQKP, DQKVX, db = run()
    qk = QKP.float().view(B, P, Mp, ld)
    key = qk[..., :d].clone().requires_grad_(True)
    query = qk[..., 2 * d].clone().requires_grad_(True)
    value = QKVX.float().view(B, P, N, ld)[..., d:2 * d].clone().requires_grad_(True)
    s = torch.softmax(query, dim=-1)                         # over Mp
    ctx = (key * s[..., None]).sum(2)                        # [B, P, d]
    out = torch.relu(value) * ctx[:, :, None, :]             # [B, P, N, d]
    close(O, out.detach().reshape(-1, d), what="O")
    close(S, s.detach(), rtol=2e-3, atol=1e-5, what="scores")
    close(CTX, ctx.detach(), rtol=2e-3, atol=1e-4, what="ctx")
    out.backward(DO.float().view(B, P, N, d))
    close(DQKP[:, :d], key.grad.reshape(-1, d), what="dkey")
    dq = query.grad.reshape(-1)
    close(DQKP[:, 2 * d], dq, rtol=3e-2, atol=2e-2 * float(dq.abs().max()) + 1e-6, what="dquery")
    close(DQKVX[:, d:2 * d], value.grad.reshape(-1, d), what="dvalue")
    assert float(DQKP[:, d:2 * d].float().abs().max()) == 0.0, "value columns of dQK_prev"
    assert float(DQKP[:, 2 * d + 1:].float().abs().max()) == 0.0, "pad columns of dQK_prev"
    assert float(DQKVX[:, :d].float().abs().max()) == 0.0 and float(DQKVX[:, 2 * d:].float().abs().max()) == 0.0, "key / query columns of dV_x"
    sums = torch.cat([DQKP[:, :d].float().sum(0), DQKVX[:, d:2 * d].float().sum(0), DQKP[:, 2 * d:2 * d + 1].float().sum(0)])
    close(db[:2 * d + 1], sums, rtol=2e-3, atol=2e-3 * float(sums.abs().max()) + 1e-5, what="dbias")
    for a, b_, what in zip((O, S, CTX, DQKP, DQKVX, db), run(), ("O", "S", "CTX", "dQK_prev", "dV_x", "dbias")):
        same(b_, a, what + " rerun")


# ------------------------------------------------------------------------------------------- stem gather with batch mixing
@pytest.mark.parametrize("B,H,W", [(1, 16, 20), (4, 16, 20), (3, 10, 14)])
@pytest.mark.parametrize("layout", ["nchw", "channels_last"])
def test_stem_im2col_with_mix(ops, lib, B, H, W, layout):
    x = rnd(B, 3, H, W, seed=621)
    if layout == "channels_last":
        x = x.contiguous(memory_format=torch.channels_last)
    prev = x.roll(1, 0)

    def ref_cols(img):
        u = F.unfold(img, kernel_size=3, stride=2, padding=1)
        return u.permute(0, 2, 1).reshape(-1, 27)

    # mix = NULL, through the wrapper and directly, equals mode 0
    plain = ops.stem_im2col(x)
    A0 = torch.empty_like(plain)
    sn, sc, sh, sw = x.stride()
    lib.cvb_stem_im2col(x.data_ptr(), sn, sc, sh, sw, B, H, W, A0.data_ptr(), None, _stream())
    same(A0, plain, "cvb_stem_im2col")
    same(ops.stem_im2col(x, torch.tensor([0.0, 0.3, 1, 1, 5, 5], device="cuda")), plain, "mode 0")
    # mixup: fp32 blend, then one bf16 rounding
    lam = 0.3
    A = ops.stem_im2col(x, torch.tensor([1.0, lam, 0, 0, 0, 0], device="cuda"))
    within_ulp(A[:, :27], ref_cols(lam * x.double() + (1 - lam) * prev.double()), "mixup")
    assert float(A[:, 27:].float().abs().max()) == 0.0
    # cutmix: rows [y1, y2) x columns [x1, x2) from the predecessor; a box on the image border and an empty box
    for (x1, y1, x2, y2) in ((0, 3, 7, H), (W - 5, 0, W, 4), (4, 2, 4, 9)):
        A = ops.stem_im2col(x, torch.tensor([2.0, lam, x1, y1, x2, y2], device="cuda"))
        xm = x.clone()
        xm[:, :, y1:y2, x1:x2] = prev[:, :, y1:y2, x1:x2]
        same(A[:, :27], ref_cols(xm).to(BF), f"cutmix box {(x1, y1, x2, y2)}")
        assert float(A[:, 27:].float().abs().max()) == 0.0


# ------------------------------------------------------------------------------------------- batched fp64 -> fp32 cast
def test_cast_f64_f32_descriptor_table(ops, lib):
    """three descriptors in one launch, built the way StepWorkspace.scatter64 builds them; n = 70000 > 16 CTAs x 256: the capped grid strides"""
    from ml_cvnets_b200 import _lib as L
    sizes = (1, 4095, 70000)
    g = torch.Generator(device="cuda").manual_seed(631)
    srcs = [torch.randn(n, device="cuda", dtype=torch.float64, generator=g) * torch.logspace(-30, 30, n, device="cuda", dtype=torch.float64)
            for n in sizes]
    dsts = [torch.full((n + 8,), float("nan"), device="cuda") for n in sizes]  # 8 sentinels past the end of each destination
    descs = (L.cvb_cast_desc * len(sizes))()
    for i, (s, d) in enumerate(zip(srcs, dsts)):
        descs[i] = L.cvb_cast_desc(s.data_ptr(), d.data_ptr(), s.numel(), 0)
    table = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).to("cuda")
    lib.cvb_cast_f64_f32(table.data_ptr(), len(sizes), max(sizes), _stream())
    torch.cuda.synchronize()
    for s, d in zip(srcs, dsts):
        same(d[:s.numel()], s.float(), f"cast n={s.numel()}")
        assert bool(torch.isnan(d[s.numel():]).all()), "wrote past the end"

"""The transformer encoder's kernels at the recipes' training shapes (-m gpu): ViT-B/16 at 224² and at the sampler's 320² / 128² crops,
ViT-S/16, the CLIP ViT-H/16 image tower, the ViT-H/16 finetune crop and both CLIP text towers, each at its recipe's full batch
(tests/test_transformer_shapes_cpu.py derives the table).

Full-size shapes take paths the small kernel tests never reach: at K >= 768 the wgmma GEMM streams its weight panel through the A ring and each
persistent CTA walks 18 - 132 tiles, so the ring's stage index and parity cross tile boundaries; the large weight gradients run one pixel split
per CTA over ~790 ring stages in a multi-wave grid; every LayerNorm has rows_per_sample = 1, and LN2's statistics come from the per-row fp64
sums of the out_proj epilogue; attention runs 3072 - 5120 register-resident CTAs, or the streaming kernels at 401 tokens.

Kernel level: every kernel _encoder_forward / _encoder_backward (functional.py) issues, called through the same ops wrappers with the same
arguments, runs twice (torch.equal, except what test_reproducible_gpu.NONDETERMINISTIC lists) and is compared over the whole tensor with an
fp64 restatement on the same bf16-rounded inputs.  Negative controls show the bounds would catch a dropped ring stage.  A coverage guard runs a
real TransformerEncoder per geometry with every wrapper recorded, and fails naming any call the kernel-level table lacks.  Layer level: one
encoder forward / backward against the oracle in fp64 at the ViT-H/16 320² crop and the causal text tower."""
import inspect
import json
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from oracle import cvnets_oracle as O  # noqa: E402
from test_kernels_gpu import bf, close, close_stat, load_ref, rnd  # noqa: E402
from test_kernels_edges_gpu import LN2  # noqa: E402
from test_modules_gpu import rel_l2  # noqa: E402
from test_parity_gpu import _record  # noqa: E402
from test_reproducible_gpu import NONDETERMINISTIC, same, twice, zeros64  # noqa: E402
from test_transformer_shapes_cpu import attention_route, geometries, keep_normalised, wgrad_launch  # noqa: E402

pytestmark = pytest.mark.gpu

F64 = torch.float64
GEOMS = {g["id"]: g for g in geometries()}
IDS = list(GEOMS)
CHUNK = 8192  # rows per fp64 reference chunk: peak memory stays in the low GiB on a shared GPU
HD = 64


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ml_cvnets_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def sms(ops):
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.fixture(autouse=True)
def _release():
    yield
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- worst errors, per geometry and kind
_WORST = {}


def note(gid, kind, err):
    w = _WORST.setdefault(gid, {})
    w[kind] = max(w.get(kind, 0.0), err)
    _record("transformer_shapes_worst_rel_l2", _WORST)


# ------------------------------------------------------------------------------------------- fp64 references and whole-tensor checks
def tmm64(G, A):
    """fp64 G^T @ A summed over row chunks (the weight gradient's reduction) -> fp32"""
    acc = torch.zeros(G.shape[1], A.shape[1], device="cuda", dtype=F64)
    for i in range(0, G.shape[0], CHUNK):
        acc += G[i:i + CHUNK].double().t() @ A[i:i + CHUNK].double()
    return acc.float()


def colsum64(G):
    acc = torch.zeros(G.shape[1], device="cuda", dtype=F64)
    for i in range(0, G.shape[0], CHUNK):
        acc += G[i:i + CHUNK].double().sum(0)
    return acc


def mm64(A, W):
    """fp64 A @ W^T of two bf16 / fp32 operands (A's rows in chunks) -> fp32"""
    M = A.shape[0]
    Wt = W.double().t()
    out = torch.empty(M, W.shape[0], device="cuda")
    for i in range(0, M, CHUNK):
        out[i:i + CHUNK] = (A[i:i + CHUNK].double() @ Wt).float()
    return out


def check_out(out, ref, what, gid=None, kind=None, rtol=1.5e-2, rel=4e-3):
    """close() of test_kernels_gpu over the whole tensor, row chunk by row chunk: element-wise bound with the global absolute term, and the
    whole-tensor relative L2"""
    atol = 1e-2 * float(ref.abs().max()) + 1e-6
    num = den = 0.0
    for i in range(0, out.shape[0], CHUNK):
        a, b = out[i:i + CHUNK].double(), ref[i:i + CHUNK].double()
        close(a, b, rtol=rtol, atol=atol, what=f"{what} rows {i}+", rel_l2=None)
        num += float(((a - b) ** 2).sum())
        den += float((b ** 2).sum())
    r = (num / max(den, 1e-60)) ** 0.5
    assert r <= rel, f"{what}: rel-L2 {r:.4g} > {rel:.3g}"
    if gid is not None:
        note(gid, kind, r)
    return r


def check_wgrad(dW, ref, what, gid=None, kind="wgrad"):
    """the benched weight-gradient bounds: element-wise rtol 2e-3 with an absolute term of 2e-3 of the largest value, rel-L2 1e-3"""
    close(dW, ref, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) + 1e-5, what=what, rel_l2=1e-3)
    if gid is not None:
        note(gid, kind, rel_l2(dW, ref))


def rejects(check, refs):
    """negative controls: the bound that passed fails against each corrupted reference"""
    for name, ref in refs:
        with pytest.raises(AssertionError):
            check(ref)
        del ref


def gemm_controls(ref, A, W, what):
    """(a) the last 32-wide k-block missing from one 128-row tile (one dropped stage of the A / W ring), (b) one 64-row M stage missing"""
    M, K = A.shape[0], A.shape[1]
    t0 = (M // 128 - 1) * 128
    a = ref.clone()
    a[t0:t0 + 128] -= (A[t0:t0 + 128, K - 32:].double() @ W[:, K - 32:].double().t()).float()
    b = ref.clone()
    m0 = (M // 2) // 64 * 64
    b[m0:m0 + 64] -= (A[m0:m0 + 64].double() @ W.double().t()).float()
    return [(f"{what}: last k-block of one tile dropped", a), (f"{what}: one 64-row stage dropped", b)]


def wgrad_controls(ref, G, A, what):
    """dW = G^T A summed over M in 64-row ring stages: (a) the last 32 columns of the last full stage missing, (b) one 64-row stage missing"""
    M, K = A.shape[0], A.shape[1]
    s0 = (M // 64 - 1) * 64
    a = ref.clone()
    a[:, K - 32:] -= (G[s0:s0 + 64].double().t() @ A[s0:s0 + 64, K - 32:].double()).float()
    b = ref.clone()
    m0 = (M // 2) // 64 * 64
    b -= (G[m0:m0 + 64].double().t() @ A[m0:m0 + 64].double()).float()
    return [(f"{what}: last k-block of one stage dropped", a), (f"{what}: one 64-row stage dropped", b)]


def tokens(M, C, seed, offset_rows=False):
    """token rows with per-row offsets and scales, as residual streams have; ``offset_rows``: every 7th row at mean 64, std 0.5"""
    X = rnd(M, C, seed=seed) * (1 + rnd(M, 1, seed=seed + 1).abs()) + 0.5 * rnd(M, 1, seed=seed + 2)
    if offset_rows:
        X[::7] = 64 + 0.5 * rnd(X[::7].shape[0], C, seed=seed + 3)
    return bf(X)


def ln_ref64(X, gamma, beta, eps):
    """fp64 LayerNorm of X's rows (chunked) -> fp32"""
    out = torch.empty(X.shape, device="cuda")
    for i in range(0, X.shape[0], CHUNK):
        x = X[i:i + CHUNK].double()
        out[i:i + CHUNK] = F.layer_norm(x, (x.shape[1],), gamma.double(), beta.double(), eps).float()
    return out


def layer_params(N, K, seed):
    return bf(rnd(N, K, scale=K ** -0.5, seed=seed)), 0.1 * rnd(N, seed=seed + 1)


# ------------------------------------------------------------------------------------------- the kernel-level call table
def call_key(name, fn, *a, **kw):
    """what the coverage guard records of one ops call: the wrapper, the widths and modes, which optional operands are present -- not M"""
    from ml_cvnets_b200 import ops as o
    b = inspect.signature(fn).bind(*a, **kw)
    b.apply_defaults()
    v = b.arguments
    if name == "pw_gemm":
        return (name, v["N"], v["K"] or v["A"].shape[1], v["a_mode"], v["e_mode"], v["rows_per_sample"], v["bias"] is not None, v["R"] is not None,
                v["samp_stats"] is not None, v["col_stats"] is not None)
    if name == "pw_wgrad":
        return (name, v["N"], v["K"], v["g_mode"], v["a_mode"], v["rows_per_sample"], v["dbias"] is not None)
    if name == "apply_load_mode":
        return (name, v["K"], v["mode"], v["rows_per_sample"])
    if name in ("mha_fwd", "mha_bwd"):
        return (name, v["S"], v["H"], v["head_dim"], v["attn_mask"] is not None, v["key_padding_mask"] is not None)
    if name == "ln_stats":
        return (name, v["X"].shape[1])
    if name == "gn_finalize":
        return (name, int(v["count"]))
    if name in ("act_fwd", "act_bwd"):
        return (name, v["kind"])
    if name == "ln_bwd":
        return (name, v["V"].shape[1], v["DRES"] is not None, v["col_sum"] is not None)
    return (name,)


RECORDED = ("pw_gemm", "pw_wgrad", "apply_load_mode", "mha_fwd", "mha_bwd", "ln_stats", "gn_finalize", "act_fwd", "act_bwd", "ln_bwd",
            "dropout_fwd", "dropout_bwd")


@pytest.fixture
def recorder(ops, monkeypatch):
    """records every top-level call of the encoder's ops wrappers (a pre-pass issued inside pw_gemm / pw_wgrad is part of that call)"""
    calls, depth = [], [0]
    for name in RECORDED:
        real = getattr(ops, name)

        def wrapped(*a, _real=real, _name=name, **kw):
            if depth[0] == 0:
                calls.append(call_key(_name, _real, *a, **kw))
            depth[0] += 1
            try:
                return _real(*a, **kw)
            finally:
                depth[0] -= 1

        monkeypatch.setattr(ops, name, wrapped)
    return calls


def kernel_table(g):
    """the calls the kernel-level tests below make at geometry g on the model's LayerNorm route -> the tests that make them"""
    from ml_cvnets_b200 import ops as o
    C, ffn, S, H = g["C"], g["ffn"], g["S"], g["heads"]
    t = {}

    def add(group, *key):
        t.setdefault(key, set()).add(group)

    add("ln_stats", "ln_stats", C)
    add("attention", "mha_fwd", S, H, HD, g["causal"], False)
    add("attention", "mha_bwd", S, H, HD, g["causal"], False)
    add("out_proj_ln2", "pw_gemm", C, C, o.A_RAW, o.E_STORE, 1, True, True, True, False)
    add("out_proj_ln2", "gn_finalize", C)
    add("ffn2", "act_fwd", o.ACT_GELU)
    add("ffn2", "pw_gemm", C, ffn, o.A_RAW, o.E_STORE, 0, True, True, False, False)
    for N, K in ((ffn, C), (C, ffn), (C, C), (C, 3 * C)):  # input gradients of ffn.4, ffn.1, out_proj, qkv_proj
        add("dgrad", "pw_gemm", N, K, o.A_RAW, o.E_STORE, 0, False, False, False, False)
    add("dgrad", "act_bwd", o.ACT_GELU)
    add("wgrad", "pw_wgrad", C, ffn, o.A_RAW, o.A_RAW, 0, True)
    add("wgrad", "pw_wgrad", C, C, o.A_RAW, o.A_RAW, 0, False)
    add("ln_bwd", "ln_bwd", C, True, True)
    add("ln_bwd", "ln_bwd", C, True, False)
    for proj, N in (("qkv", 3 * C), ("ffn1", ffn)):
        group = f"ln_projection {proj}"
        if keep_normalised(g):
            add(group, "apply_load_mode", C, o.A_GN, 1)
            add(group, "pw_gemm", N, C, o.A_RAW, o.E_STORE, 0, True, False, False, False)
            add(group, "pw_wgrad", N, C, o.A_RAW, o.A_RAW, 0, True)
        else:
            add(group, "pw_gemm", N, C, o.A_GN, o.E_STORE, 1, True, False, False, False)
            add(group, "pw_wgrad", N, C, o.A_RAW, o.A_GN, 1, True)
    return t


def covers(g, group, calls):
    """the calls one kernel-level test made are exactly its entries of the table"""
    want = {k for k, v in kernel_table(g).items() if group in v}
    assert set(calls) == want, f"{g['id']} {group}: calls {sorted(set(calls) - want)} are not in the table, {sorted(want - set(calls))} not made"


# ------------------------------------------------------------------------------------------- LayerNorm statistics and the normalised operand
@pytest.mark.parametrize("gid", IDS)
def test_ln_stats(ops, recorder, gid):
    """ln_stats over every token (one fp32 pass), rows at mean 64 / std 0.5 among them; the LayerNorm load mode's operand from it against the
    fp64 LayerNorm.  The rstd of the offset rows is not bounded on its own: its one-pass error (~1e-3 at |mean| / std = 128) is below the
    bf16 resolution of the normalised output, which is what the GEMMs read."""
    g = GEOMS[gid]
    M, C = g["B"] * g["S"], g["C"]
    X = tokens(M, C, 2001, offset_rows=True)
    gamma, beta = 1 + 0.2 * rnd(C, seed=2005), 0.1 * rnd(C, seed=2006)
    (ln,) = twice(lambda: [ops.ln_stats(X, g["eps"])], ("ln stats",))
    covers(g, "ln_stats", recorder)
    mean = torch.empty(M, device="cuda", dtype=F64)
    var = torch.empty(M, device="cuda", dtype=F64)
    for i in range(0, M, CHUNK):
        x = X[i:i + CHUNK].double()
        mean[i:i + CHUNK], var[i:i + CHUNK] = x.mean(1), x.var(1, unbiased=False)
    err = (ln[0].double() - mean).abs()
    assert float((err - 4e-6 * mean.abs()).max()) <= 1e-4, f"mean: max err {float(err.max()):.3g}"
    rstd = (var + g["eps"]).rsqrt()
    plain = torch.ones(M, dtype=torch.bool, device="cuda")
    plain[::7] = False
    rel = ((ln[1].double() - rstd) / rstd).abs()
    assert float(rel[plain].max()) < 1e-3, f"rstd: max rel err {float(rel[plain].max()):.3g}"
    xn = twice(lambda: [ops.apply_load_mode(X, ops.A_GN, C, a_p=(gamma, beta), row_stats=(ln[0], ln[1]), rows_per_sample=1)], ("xn",))[0]
    check_out(xn, ln_ref64(X, gamma, beta, g["eps"]), "LayerNorm operand", gid, "layernorm")


# ------------------------------------------------------------------------------------------- the LayerNorm-fused projections
def _ln_proj_routes():
    return [pytest.param(gid, proj, route, id=f"{gid}-{proj}-{route}") for gid in IDS for proj in ("qkv", "ffn1")
            for route in (("model", "in-kernel") if gid in ("vitb224", "vith224") else ("model",))]


@pytest.mark.parametrize("gid,proj,route", _ln_proj_routes())
def test_ln_projection(ops, recorder, monkeypatch, gid, proj, route):
    """qkv_proj / ffn.1: LayerNorm(X) @ W^T + b and its weight gradient with the bias gradient, as ln_proj / ln_wgrad issue them -- the kept
    normalised tokens of the pre-pass, or (ops.WIDE_K raised) the LayerNorm load mode inside the GEMM and the weight-gradient kernel"""
    g = GEOMS[gid]
    M, C = g["B"] * g["S"], g["C"]
    N = 3 * C if proj == "qkv" else g["ffn"]
    if route == "in-kernel":
        monkeypatch.setattr(ops, "WIDE_K", 1 << 30)
    keep = keep_normalised(g)
    assert keep == (route == "model" and gid != "vits224")
    X = tokens(M, C, 2101)
    ln = ops.ln_stats(X, g["eps"])
    recorder.clear()
    gamma, beta = 1 + 0.2 * rnd(C, seed=2102), 0.1 * rnd(C, seed=2103)
    W, bias = layer_params(N, C, 2104)
    G = bf(rnd(M, N, seed=2106))
    kw = dict(a_p=(gamma, beta), row_stats=(ln[0], ln[1]), rows_per_sample=1)

    def run():
        if keep:
            xn = ops.apply_load_mode(X, ops.A_GN, C, **kw)
            out = ops.pw_gemm(xn, W, N, bias=bias)
            db = torch.zeros(N, device="cuda")
            dW = ops.pw_wgrad(G, xn, N, C, dbias=db)
        else:
            out = ops.pw_gemm(X, W, N, a_mode=ops.A_GN, bias=bias, **kw)
            db = torch.zeros(N, device="cuda")
            dW = ops.pw_wgrad(G, X, N, C, a_mode=ops.A_GN, dbias=db, **kw)
        return out, dW, db

    out, dW, db = twice(run, ("out", "dW", "dbias"))
    if route == "model":
        covers(g, f"ln_projection {proj}", recorder)
    Xn = load_ref(ops.A_GN, X, (gamma, beta), row=(ln[0], ln[1]), rps=1)  # the bf16 operand both routes multiply
    check_out(out, mm64(Xn, W) + bias, f"{proj} {route}", gid, "gemm")
    check_wgrad(dW, tmm64(G, Xn), f"{proj} {route} dW", gid)
    dbr = colsum64(G).float()
    close(db, dbr, rtol=2e-3, atol=2e-3 * float(dbr.abs().max()) + 1e-4, what=f"{proj} dbias", rel_l2=1e-3)


# ------------------------------------------------------------------------------------------- attention
def _mha64(qkv, dO, b0, b1, S, H, scale, causal):
    """fp64 softmax attention of samples [b0, b1) on the packed projection: O, LSE (base 2) and dQKV"""
    x = qkv[b0 * S:b1 * S].double().view(b1 - b0, S, 3, H, HD).permute(2, 0, 3, 1, 4)  # [3, b, H, S, c]
    q, k, v = x[0], x[1], x[2]
    s = (q @ k.transpose(-1, -2)) * scale
    if causal:
        s = s.masked_fill(torch.ones(S, S, dtype=torch.bool, device="cuda").triu(1), float("-inf"))
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    o = p @ v
    do = dO[b0 * S:b1 * S].double().view(b1 - b0, S, H, HD).transpose(1, 2)
    dv = p.transpose(-1, -2) @ do
    dp = do @ v.transpose(-1, -2)
    ds = p * (dp - (dp * p).sum(-1, keepdim=True))
    dq, dk = (ds @ k) * scale, (ds.transpose(-1, -2) @ q) * scale
    dqkv = torch.stack([dq, dk, dv]).permute(1, 3, 0, 2, 4).reshape((b1 - b0) * S, 3 * H * HD)
    return o.transpose(1, 2).reshape((b1 - b0) * S, H * HD), lse / LN2, dqkv


@pytest.mark.parametrize("gid", IDS)
def test_attention(ops, recorder, gid):
    """mha_fwd / mha_bwd over the whole recipe batch (B * H CTAs of the register-resident kernels, or the streaming kernels at 401 tokens):
    O, LSE and dQKV against fp64 softmax attention, sample chunk by sample chunk"""
    g = GEOMS[gid]
    B, S, H, C = g["B"], g["S"], g["heads"], g["C"]
    qkv, dO = bf(rnd(B * S, 3 * C, seed=2201)), bf(rnd(B * S, C, seed=2202))
    amask = torch.full((S, S), float("-inf"), device="cuda").triu(1)[None].repeat(B, 1, 1).contiguous() if g["causal"] else None
    scale = HD ** -0.5
    O_, LSE = twice(lambda: ops.mha_fwd(qkv, B, S, H, HD, scale, amask), ("O", "LSE"))

    def bwd():
        return [ops.mha_bwd(qkv, O_, dO, LSE, B, S, H, HD, scale, amask)]

    if attention_route(g) == "register":
        # NONDETERMINISTIC["cvb_mha_bwd"]: the register-resident kernel sums dQ with shared-memory float atomics; dK and dV have one writer
        assert "cvb_mha_bwd" in NONDETERMINISTIC
        D1 = bwd()[0].clone()
        D2 = bwd()[0]
        same(D2[:, C:], D1[:, C:], "dK, dV: second run")
        D = D1
    else:
        (D,) = twice(bwd, ("dQKV",))
    covers(g, "attention", recorder)
    bc = max(1, (1 << 25) // (H * S * S))
    refO = torch.empty(B * S, C, device="cuda")
    refD = torch.empty(B * S, 3 * C, device="cuda")
    lse_err, lse_max = 0.0, 0.0
    for b0 in range(0, B, bc):
        b1 = min(B, b0 + bc)
        o, lse, d = _mha64(qkv, dO, b0, b1, S, H, scale, g["causal"])
        refO[b0 * S:b1 * S], refD[b0 * S:b1 * S] = o.float(), d.float()
        lse_err = max(lse_err, float((LSE[b0:b1].double() - lse).abs().max()))
        lse_max = max(lse_max, float(lse.abs().max()))
    check_out(O_, refO, "O", gid, "attention")
    assert lse_err <= 1e-4 * lse_max + 1e-4, f"LSE: max err {lse_err:.3g}"
    check_out(D, refD, "dQKV", gid, "attention", rtol=3e-2)


# ------------------------------------------------------------------------------------------- out_proj + residual + LN2 statistics
@pytest.mark.parametrize("gid", IDS)
def test_out_proj_ln2(ops, recorder, gid):
    """X1 = O @ Wo^T + bo + x with the per-row fp64 sums of the epilogue (rows_per_sample = 1: one sample per token, from C / 128 N tiles),
    and gn_finalize(count = C) turning them into LN2's statistics; all bitwise run to run"""
    g = GEOMS[gid]
    M, C = g["B"] * g["S"], g["C"]
    Oa, x2 = bf(rnd(M, C, seed=2301)), tokens(M, C, 2302)
    W, bo = layer_params(C, C, 2305)

    def run():
        samp = zeros64(2, M)
        X1 = ops.pw_gemm(Oa, W, C, bias=bo, R=x2, samp_stats=samp, rows_per_sample=1)
        return X1, samp, ops.gn_finalize(samp, C, g["eps"])

    X1, samp, ln2 = twice(run, ("X1", "samp_stats", "LN2 statistics"))
    covers(g, "out_proj_ln2", recorder)
    check_out(X1, mm64(Oa, W) + bo + x2.float(), "out_proj + residual", gid, "gemm")
    x = X1.double()
    s, q = x.sum(1), (x * x).sum(1)
    close_stat(samp[0], s, "per-row sum")
    close_stat(samp[1], q, "per-row sum of squares")
    mean, var = s / C, (x - (s / C)[:, None]).pow(2).mean(1)
    assert float((ln2[0].double() - mean).abs().max()) <= 1e-5 * float(mean.abs().max()) + 1e-6
    rstd = (var + g["eps"]).rsqrt()
    r = float(((ln2[1].double() - rstd) / rstd).abs().max())
    assert r <= 1e-4, f"LN2 rstd: max rel err {r:.3g}"
    note(gid, "layernorm", r)


# ------------------------------------------------------------------------------------------- FFN down projection (K = 4C)
@pytest.mark.parametrize("gid", IDS)
def test_ffn2(ops, recorder, gid):
    """ha = GELU(h); X2 = ha @ W2^T + b2 + X1: K = 3072 / 5120 streams the weight k-blocks through the A ring across 18 - 31 tiles per CTA"""
    g = GEOMS[gid]
    M, C, ffn = g["B"] * g["S"], g["C"], g["ffn"]
    h, X1 = bf(rnd(M, ffn, seed=2401) * 1.5), tokens(M, C, 2402)
    W, b2 = layer_params(C, ffn, 2405)
    def run():
        ha = ops.act_fwd(h, ops.ACT_GELU)
        return ha, ops.pw_gemm(ha, W, C, bias=b2, R=X1)

    ha, X2 = twice(run, ("GELU", "X2"))
    covers(g, "ffn2", recorder)
    har = torch.empty(M, ffn, device="cuda")
    for i in range(0, M, CHUNK):
        har[i:i + CHUNK] = F.gelu(h[i:i + CHUNK].double()).float()
    check_out(ha, har, "GELU", gid, "elementwise")
    del har
    ref = mm64(ha, W) + b2 + X1.float()
    check_out(X2, ref, "ffn2 + residual", gid, "gemm")
    check = lambda r: check_out(X2, r, "ffn2 + residual")  # noqa: E731
    rejects(check, gemm_controls(ref, ha, W, "ffn2"))


# ------------------------------------------------------------------------------------------- input-gradient GEMMs
@pytest.mark.parametrize("gid", IDS)
def test_dgrad(ops, recorder, gid):
    """the four input-gradient GEMMs on the transposed weights: dha = dY @ W2 (then GELU'), vF = dh @ W1 (K = ffn), dO = dA @ Wo,
    vA = dqkv @ Wqkv (K = 3C)"""
    g = GEOMS[gid]
    M, C, ffn = g["B"] * g["S"], g["C"], g["ffn"]
    dY, dh, dA, dq = bf(rnd(M, C, seed=2501)), bf(rnd(M, ffn, seed=2502)), bf(rnd(M, C, seed=2503)), bf(rnd(M, 3 * C, seed=2504))
    h = bf(rnd(M, ffn, seed=2505) * 1.5)
    W2t, W1t = layer_params(ffn, C, 2506)[0], layer_params(C, ffn, 2507)[0]
    Wot, Wqt = layer_params(C, C, 2508)[0], layer_params(C, 3 * C, 2509)[0]

    def run():
        dha = ops.pw_gemm(dY, W2t, ffn, K=C)
        return (dha, ops.act_bwd(dha, h, ops.ACT_GELU), ops.pw_gemm(dh, W1t, C, K=ffn), ops.pw_gemm(dA, Wot, C, K=C),
                ops.pw_gemm(dq, Wqt, C, K=3 * C))

    dha, dhr, vF, dO, vA = twice(run, ("dha", "GELU backward", "vF", "dO", "vA"))
    covers(g, "dgrad", recorder)
    check_out(dha, mm64(dY, W2t), "ffn2 dgrad", gid, "gemm")
    ref = torch.empty(M, ffn, device="cuda")
    for i in range(0, M, CHUNK):
        z = h[i:i + CHUNK].double().requires_grad_(True)
        F.gelu(z).backward(dha[i:i + CHUNK].double())
        ref[i:i + CHUNK] = z.grad.float()
    check_out(dhr, ref, "GELU backward", gid, "elementwise")
    del ref
    for out, A, W, what in ((vF, dh, W1t, "ffn1 dgrad"), (dO, dA, Wot, "out_proj dgrad"), (vA, dq, Wqt, "qkv dgrad")):
        ref = mm64(A, W)
        check_out(out, ref, what, gid, "gemm")
        check = lambda r, out=out, what=what: check_out(out, r, what)  # noqa: E731
        if what == "ffn1 dgrad":
            rejects(check, gemm_controls(ref, A, W, what))


# ------------------------------------------------------------------------------------------- weight gradients of the un-normalised operands
@pytest.mark.parametrize("gid", IDS)
def test_wgrad(ops, recorder, sms, gid):
    """ffn.4: dW2 = dY^T GELU(h) with the bias gradient (one pixel split per CTA in a multi-wave grid at C >= 768); out_proj: dWo = dA^T O,
    its bias gradient coming from ln_bwd's column sums"""
    g = GEOMS[gid]
    M, C, ffn = g["B"] * g["S"], g["C"], g["ffn"]
    dY, ha, dA, Oa = bf(rnd(M, C, seed=2601)), bf(rnd(M, ffn, seed=2602)), bf(rnd(M, C, seed=2603)), bf(rnd(M, C, seed=2604))

    def run():
        db = torch.zeros(C, device="cuda")
        return ops.pw_wgrad(dY, ha, C, ffn, dbias=db), db, ops.pw_wgrad(dA, Oa, C, C)

    dW2, db2, dWo = twice(run, ("dW2", "db2", "dWo"))
    covers(g, "wgrad", recorder)
    ref = tmm64(dY, ha)
    check_wgrad(dW2, ref, "ffn2 dW", gid)
    check = lambda r: check_wgrad(dW2, r, "ffn2 dW")  # noqa: E731
    if C >= 768:
        assert wgrad_launch(M, C, ffn, sms)["splits"] == 1
        rejects(check, wgrad_controls(ref, dY, ha, "ffn2 dW"))
    dbr = colsum64(dY).float()
    close(db2, dbr, rtol=2e-3, atol=2e-3 * float(dbr.abs().max()) + 1e-4, what="ffn2 dbias", rel_l2=1e-3)
    check_wgrad(dWo, tmm64(dA, Oa), "out_proj dW", gid)


# ------------------------------------------------------------------------------------------- LayerNorm backward
@pytest.mark.parametrize("gid", IDS)
def test_ln_bwd(ops, recorder, gid):
    """dX1 = LN2 backward of vF + dY with the column sums (= d(out_proj bias)), and dx = LN1 backward of vA + dX1; dgamma / dbeta in fp64"""
    g = GEOMS[gid]
    M, C = g["B"] * g["S"], g["C"]
    V, X, R = bf(rnd(M, C, seed=2701)), tokens(M, C, 2702), bf(rnd(M, C, seed=2703))
    gamma = 1 + 0.2 * rnd(C, seed=2704)
    ln = ops.ln_stats(X, g["eps"])
    recorder.clear()

    def run():
        col, cs, col1 = zeros64(2, C), zeros64(C), zeros64(2, C)
        DX = ops.ln_bwd(V, X, ln, gamma, col, DRES=R, col_sum=cs)
        DX1 = ops.ln_bwd(V, X, ln, gamma, col1, DRES=DX)
        return DX, col, cs, DX1, col1

    DX, col, cs, DX1, col1 = twice(run, ("dx", "dbeta / dgamma", "column sums", "dx (no column sums)", "dbeta / dgamma (second)"))
    covers(g, "ln_bwd", recorder)
    ref = torch.empty(M, C, device="cuda")
    dg, dbt = zeros64(C), zeros64(C)
    for i in range(0, M, CHUNK):
        v, x = V[i:i + CHUNK].double(), X[i:i + CHUNK].double()
        mu, rs = ln[0][i:i + CHUNK].double()[:, None], ln[1][i:i + CHUNK].double()[:, None]
        xh = (x - mu) * rs
        gv = v * gamma.double()
        ref[i:i + CHUNK] = (rs * (gv - gv.mean(1, keepdim=True) - xh * (gv * xh).mean(1, keepdim=True)) + R[i:i + CHUNK].double()).float()
        dg += (v * xh).sum(0)
        dbt += v.sum(0)
    check_out(DX, ref, "ln_bwd dx", gid, "layernorm")
    close_stat(col[0], dbt, "dbeta", rtol=5e-3)
    close_stat(col[1], dg, "dgamma", rtol=5e-3)
    close_stat(cs, DX.double().sum(0), "column sums of dx", rtol=5e-3)
    ref1 = ref - R.float() + DX.float()
    check_out(DX1, ref1, "ln_bwd dx (residual = dx)")
    close_stat(col1[0], dbt, "dbeta (second)", rtol=5e-3)


# ------------------------------------------------------------------------------------------- patch embedding and token assembly
IMAGE = [gid for gid in IDS if GEOMS[gid]["n_patch"] is not None]


@pytest.mark.parametrize("gid", IMAGE)
def test_patch_embedding(ops, gid):
    """patch_emb.2 (2x2 stride 2 conv with bias on the gathered patch matrix, K = 4 * stem width): forward GEMM, input-gradient GEMM and the
    weight gradient with its bias gradient"""
    g = GEOMS[gid]
    M, C, K = g["B"] * g["n_patch"], g["C"], g["stem_k"]
    x2, dout = bf(rnd(M, K, seed=2801)), bf(rnd(M, C, seed=2802))
    W, bias = layer_params(C, K, 2803)
    Wt = bf(rnd(K, C, scale=C ** -0.5, seed=2805))

    def run():
        db = torch.zeros(C, device="cuda")
        return ops.pw_gemm(x2, W, C, bias=bias), ops.pw_gemm(dout, Wt, K, K=C), ops.pw_wgrad(dout, x2, C, K, dbias=db), db

    y, dA, dW, db = twice(run, ("patch tokens", "dpatch", "dW", "dbias"))
    check_out(y, mm64(x2, W) + bias, "patch embedding", gid, "gemm")
    check_out(dA, mm64(dout, Wt), "patch embedding dgrad", gid, "gemm")
    check_wgrad(dW, tmm64(dout, x2), "patch embedding dW", gid)
    dbr = colsum64(dout).float()
    close(db, dbr, rtol=2e-3, atol=2e-3 * float(dbr.abs().max()) + 1e-4, what="patch dbias", rel_l2=1e-3)


@pytest.mark.parametrize("gid", [gid for gid in IMAGE if GEOMS[gid]["n_patch"] != GEOMS[gid]["n_pos"]])
def test_tokens_interp(ops, gid):
    """cat(cls, patch + the 196-entry table resampled to the crop's patch count) and its adjoint, at the sampler's batch"""
    g = GEOMS[gid]
    B, N, C, n_pos = g["B"], g["n_patch"], g["C"], g["n_pos"]
    pos, cls = rnd(1, 1, n_pos, C, seed=2901), rnd(1, 1, C, seed=2902)
    patch, dout = bf(rnd(B * N, C, seed=2903)), bf(rnd(B, N + 1, C, seed=2904))

    def run():
        dpos, dcls = torch.zeros(n_pos, C, device="cuda"), torch.zeros(C, device="cuda")
        return ops.vit_tokens_interp_fwd(patch, pos, cls, B, N, C), ops.vit_tokens_interp_bwd(dout, dpos, dcls, B, N, C), dpos, dcls

    out, dpatch, dpos, dcls = twice(run, ("tokens", "dpatch", "dpos", "dcls"))
    p64 = pos.double().requires_grad_(True)
    table = F.interpolate(p64, size=(N, C), mode="bilinear").reshape(N, C)
    ref = patch.double().view(B, N, C) + table.detach()
    err = (out[:, 1:].double() - ref).abs() - ref.abs() * 2.0 ** -8
    assert float(err.max()) <= 1e-4, f"tokens: max err beyond bf16 rounding {float(err.max()):.3g}"
    same(out[:, 0], cls.view(1, C).to(torch.bfloat16).expand(B, C), "cls rows")
    same(dpatch.view(B, N, C), dout[:, 1:], "dpatch")
    table.backward(dout[:, 1:].double().sum(0))
    close(dpos, p64.grad.view(n_pos, C), rtol=1e-4, atol=1e-4 * float(p64.grad.abs().max()) + 1e-6, what="dpos", rel_l2=1e-5)
    close(dcls, dout[:, 0].double().sum(0), rtol=1e-5, atol=1e-6, what="dcls", rel_l2=1e-6)


# ------------------------------------------------------------------------------------------- coverage guard
def _encoder(pkg, g, seed):
    opts = pkg.default_opts(**{"model.activation.name": g["act"]})
    shapes = {}
    O.transformer_encoder_shapes(shapes, "m", g["C"], g["ffn"])
    m = pkg.TransformerEncoder(opts, g["C"], g["ffn"], num_heads=g["heads"])
    P = O.seeded_fill_(shapes, seed)
    m.load_state_dict({k[2:]: v for k, v in P.items()}, strict=True)
    for mod in m.modules():
        if isinstance(mod, torch.nn.LayerNorm):
            mod.eps = g["eps"]
    return m.cuda().train(), shapes


@pytest.mark.parametrize("gid", IDS)
def test_kernel_table_covers_the_encoder(ops, recorder, gid):
    """one real TransformerEncoder forward / backward at batch 2 with every ops wrapper recorded: each call (modulo M) must be one the
    kernel-level tests above make at this geometry"""
    import ml_cvnets_b200 as pkg
    g = GEOMS[gid]
    m, _ = _encoder(pkg, g, 3001)
    B, S = 2, g["S"]
    x = torch.randn(B, S, g["C"], device="cuda").bfloat16().float().requires_grad_(True)
    mask = torch.full((S, S), float("-inf"), device="cuda").triu(1)[None].repeat(B, 1, 1) if g["causal"] else None
    y = m(x, attn_mask=mask)
    y.backward(torch.randn_like(y))
    torch.cuda.synchronize()
    table = kernel_table(g)
    missing = sorted(set(recorder) - set(table))
    assert not missing, f"{gid}: the encoder issues calls the kernel-level table does not test: {missing}"
    assert len(set(recorder)) >= 16 and x.grad is not None


# ------------------------------------------------------------------------------------------- layer level
@pytest.mark.parametrize("gid,B", [("vith320", 31), ("text512", 64)])
def test_encoder_layer_against_fp64_oracle(gid, B):
    """one drop-in TransformerEncoder forward / backward against oracle.transformer_encoder in fp64 on the GPU (the streaming attention at
    401 tokens; the causal text tower): the bounds of test_modules_gpu.test_transformer_encoder_vit_base_shape, and no further from fp64 than
    1.15x the oracle under torch bf16 autocast plus 2e-3, the widths suite's margin (the layer's output is stored in bf16, the comparator's
    residual sum stays fp32)"""
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as pkg
    g = GEOMS[gid]
    S, C, H = g["S"], g["C"], g["heads"]
    m, shapes = _encoder(pkg, g, 3101)
    gen = torch.Generator(device="cuda").manual_seed(3102)
    x = torch.randn(B, S, C, device="cuda", generator=gen).bfloat16().float()
    gy = torch.randn(B, S, C, device="cuda", generator=gen).bfloat16().float()
    mask = torch.full((S, S), float("-inf"), device="cuda").triu(1)[None].repeat(B, 1, 1) if g["causal"] else None

    def oracle(dtype, autocast):
        P = O.clone_params(O.seeded_fill_(dict(shapes), 3101), device="cuda", dtype=dtype)
        xo = x.to(dtype).clone().requires_grad_(True)
        with torch.autocast("cuda", dtype=torch.bfloat16, enabled=autocast):
            yo = O.transformer_encoder(P, "m", xo, H, act=g["act"], eps=g["eps"], attn_mask=None if mask is None else mask.to(dtype))
        yo.backward(gy.to(yo.dtype))
        return yo.detach().double(), xo.grad.double(), {k[2:]: p.grad.double() for k, p in P.items() if p.requires_grad}

    y64, gx64, gp64 = oracle(F64, False)
    ya, gxa, gpa = oracle(torch.float32, True)
    xg = x.clone().requires_grad_(True)
    y = m(xg, attn_mask=mask)
    y.backward(gy.to(y.dtype))
    torch.cuda.synchronize()
    named = dict(m.named_parameters())
    flat = lambda d: torch.cat([d[k].flatten() for k in sorted(gp64)])  # noqa: E731
    rec = {"y": rel_l2(y, y64), "y_autocast": rel_l2(ya, y64), "gx": rel_l2(xg.grad, gx64), "gx_autocast": rel_l2(gxa, gx64),
           "grads": rel_l2(flat({k: named[k].grad for k in gp64}), flat(gp64)), "grads_autocast": rel_l2(flat(gpa), flat(gp64))}
    rec["per_param"] = {k: rel_l2(named[k].grad, gp64[k]) for k in gp64}
    print(f"\n[{gid} B={B}] " + json.dumps(rec))
    _record(f"transformer_layer_{gid}_B{B}", rec)
    assert rec["y"] <= 2e-2 and rec["gx"] <= 5e-2, rec
    for k, e in rec["per_param"].items():
        assert e <= 6e-2, f"{k}: {e:.4g}"
    for k in ("y", "gx", "grads"):
        assert rec[k] <= 1.15 * rec[f"{k}_autocast"] + 2e-3, (k, rec)

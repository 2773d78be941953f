"""MobileViT-v1 XS and S, the recipes' own models (-m gpu): the kernels at the recipe's training shapes, and the model end to end.

Every other MobileViT-v1 test runs XXS at batch 1 - 8.  At XS / S, 256x256 and batch 128 the blocks reach paths those never do: 512 attention
sequences per call at head dims 24 - 60 (30 takes the 4-byte-chunk load, 60 is the widest non-64 head), dense 3x3 convs whose input-gradient
GEMMs write up to 2880 columns with a ragged last tile and whose weight gradients split between the two kernels by K % 64 at M = 131 072,
narrow GEMMs on the mma.sync kernel's resident weight panel at K up to 1440, LayerNorm at 96 - 240 channels, and expand-4 inverted residuals.

Kernel level (tests/test_mobilevit_v1_modes_cpu.py derives the table): each kernel call the model makes, through the same ops wrappers with
the model's arguments, runs twice (torch.equal) and is compared over the whole tensor with an fp64 restatement on the same bf16 inputs, in
row chunks.  Negative controls show the bounds catch one corrupted output tile, one dropped
k-block, a skipped ragged N tile and a mishandled last head-dim chunk.  A coverage guard records a real MobileViTBlock's calls per mode and
fails naming any call the table does not test.  Model level: the reference's fixtures, stage-wise parity at batch 128, a train step at batch 16
against the fp32 oracle bounded by its bf16-autocast counterpart, three bitwise MobileViT-S TrainStep steps with the recipe's dropouts, and
the refusal at the crop where a block's token count equals its width."""
import inspect
import json
import os
import sys
from types import SimpleNamespace

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_reproducible_gpu as R  # noqa: E402
import test_transformer_shapes_gpu as T  # noqa: E402
from oracle import cvnets_oracle as O  # noqa: E402
from test_kernels_edges_gpu import LN2, _fold_v1, _unfold_v1  # noqa: E402
from test_kernels_gpu import bf, close, close_stat, dsilu, load_ref, rnd, silu  # noqa: E402
from test_mobilevit_v1_modes_cpu import MODES, attn_blocks, colliding_crops, head_load_chunk, load_mit_fixture, table  # noqa: E402
from test_parity_gpu import _record, stagewise_record, train_parity_record  # noqa: E402
from test_reproducible_gpu import same, twice, zeros64  # noqa: E402
from test_standalone_gpu import check_mobilevit_v1_against_fixture  # noqa: E402
from test_transformer_shapes_gpu import CHUNK, check_wgrad, colsum64, gemm_controls, layer_params, ln_ref64, mm64, rejects, tmm64, tokens, wgrad_controls  # noqa: E402,E501

pytestmark = pytest.mark.gpu

F64 = torch.float64
TABLE = table()
EPS = 1e-5          # nn.LayerNorm's default, which every MobileViT-v1 LayerNorm keeps
P_DROP = 0.1        # the recipes' mit.dropout (attention / FFN branch outputs)


def ids(kind):
    return [uid for uid, (k, _) in TABLE.items() if k == kind]


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ml_cvnets_b200 import ops as o
    return o


@pytest.fixture(scope="module")
def pkg(ops):
    import ml_cvnets_b200 as m
    return m


@pytest.fixture(autouse=True)
def _release():
    yield
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------- worst errors, per mode and kind
_WORST = {}


def note(g, kind, err):
    w = _WORST.setdefault(g["mode"], {})
    w[kind] = max(w.get(kind, 0.0), err)
    _record("mobilevit_v1_modes_worst_rel_l2", _WORST)


def check(out, ref, what, g=None, kind=None, **kw):
    """test_transformer_shapes_gpu.check_out (element-wise bound and whole-tensor rel-L2, row chunk by row chunk), noted per mode"""
    r = T.check_out(out, ref, what, **kw)
    if g is not None:
        note(g, kind, r)
    return r


def check_dw(dW, ref, what, g):
    check_wgrad(dW, ref, what)
    note(g, "wgrad", float((dW.double() - ref.double()).norm() / ref.double().norm()))


def bias_check(db, G, what):
    dbr = colsum64(G).float()
    close(db, dbr, rtol=2e-3, atol=2e-3 * float(dbr.abs().max()) + 1e-4, what=what, rel_l2=1e-3)


def col_stats_check(st, Y, what, Y2=None):
    """the epilogue's fp64 column sums of Y and of Y * Y2 (Y2 = None: sums of squares) against fp64 sums of the stored bf16 Y.  Full tiles
    of the wgmma kernel sum the fp32 values before their rounding (gemm_tc.cu), so the bound is close_stat's plus six standard deviations
    of the sum of the M rounding errors (each uniform within one bf16 ulp <= 2^-7 |y|)"""
    sq = Y2 is None
    s, q, vs, vq = (torch.zeros(Y.shape[1], device="cuda", dtype=F64) for _ in range(4))
    for i in range(0, Y.shape[0], CHUNK):
        y = Y[i:i + CHUNK].double()
        p = y * (y if sq else Y2[i:i + CHUNK].double())
        s += y.sum(0)
        q += p.sum(0)
        vs += (y * y).sum(0)
        vq += ((2 if sq else 1) * p).pow(2).sum(0)
    sig = 2.0 ** -7 / 12 ** 0.5
    for got, ref, var, name in ((st[0], s, vs, "column sums"), (st[1], q, vq, "column sums of products")):
        err = (got.double() - ref).abs()
        bound = 2e-3 * float(ref.abs().max()) + 6 * sig * var.sqrt() + 1e-6
        bad = err > bound
        assert not bool(bad.any()), f"{what} {name}: {int(bad.sum())} channels off, worst err {float(err.max()):.4g} (scale {float(ref.abs().max()):.4g})"


def chunked(fn, M, N):
    """an fp32 [M, N] reference computed by fn(row slice) in fp64, chunk by chunk"""
    out = torch.empty(M, N, device="cuda")
    for i in range(0, M, CHUNK):
        out[i:i + CHUNK] = fn(slice(i, min(M, i + CHUNK))).float()
    return out


def bn_params(C, seed):
    """a BatchNorm forward record [4, C] (mean, rstd, scale, shift) and backward coefficients [3, C]"""
    bn = torch.stack([0.1 * rnd(C, seed=seed), 1 + 0.1 * rnd(C, seed=seed + 1).abs(), 1 + 0.2 * rnd(C, seed=seed + 2), 0.3 * rnd(C, seed=seed + 3)])
    coef = torch.stack([1 + 0.2 * rnd(C, seed=seed + 4), 0.1 * rnd(C, seed=seed + 5), 0.1 * rnd(C, seed=seed + 6)])
    return bn, coef


# ------------------------------------------------------------------------------------------- the call table and the coverage guard
def call_key(name, fn, *a, **kw):
    """what the coverage guard records of one ops call: the wrapper, its widths, modes and which optional operands are present -- not M"""
    b = inspect.signature(fn).bind(*a, **kw)
    b.apply_defaults()
    v = b.arguments
    if name == "im2col":
        return (name, v["x"].shape[1], v["k"], v["stride"], v["pad"])
    if name == "col2im":
        return (name, v["Cin"], v["k"], v["stride"], v["pad"])
    if name == "patch_permute":
        return (name, v["X"].shape[1], bool(v["inverse"]))
    if name == "concat2":
        return (name, v["A"].shape[1], v["Bt"].shape[1])
    if name == "split2":
        return (name, v["C1"], v["C2"])
    if name == "bn_apply":
        return (name, v["Y"].shape[1], bool(v["act"]), v["R"] is not None)
    if name == "bn_bwd_reduce":
        return (name, v["Y"].shape[1], bool(v["act"]), bool(v["store_dz"]))
    if name == "dropout_fwd":
        return (name, v["V"].shape[1], v["p"], v["p_row"], v["R"] is not None)
    if name == "dropout_bwd":
        return (name, v["DY"].shape[1], v["p"], v["p_row"])
    return T.call_key(name, fn, *a, **kw)


# the per-channel kernels that have no token dimension are not recorded: bn_finalize / bn_bwd_finalize (C-long vectors, test_kernels_gpu),
# unprep_grad (a weight-gradient layout copy) and rng_next (one mask key)
RECORDED = T.RECORDED + ("im2col", "col2im", "patch_permute", "concat2", "split2", "bn_apply", "bn_bwd_reduce")


@pytest.fixture
def recorder(ops, monkeypatch):
    """records every top-level call of the recorded ops wrappers (a pre-pass issued inside pw_gemm / pw_wgrad is part of that call)"""
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


def block_table(g):
    """the calls the kernel-level tests below make for one MobileViTBlock (dropout 0 and the recipe's 0.1) -> the tests that make them"""
    from ml_cvnets_b200 import ops as o
    c, d, ffn, S = g["c"], g["d"], g["ffn"], g["S"]
    t = {}

    def add(group, *key):
        t.setdefault(key, set()).add(group)

    for which, cin in (("local_rep.conv_3x3", c), ("fusion", 2 * c)):
        grp = f"conv {which}"
        add(grp, "im2col", cin, 3, 1, 1)
        add(grp, "pw_gemm", c, 9 * cin, o.A_RAW, o.E_STORE, 0, False, False, False, True)
        add(grp, "bn_apply", c, True, False)
        add(grp, "bn_bwd_reduce", c, True, True)
        add(grp, "pw_gemm", 9 * cin, c, o.A_BNB, o.E_STORE, 0, False, False, False, False)
        add(grp, "pw_wgrad", c, 9 * cin, o.A_BNB, o.A_RAW, 0, False)
        add(grp, "col2im", cin, 3, 1, 1)
    add("block_1x1", "pw_gemm", d, c, o.A_RAW, o.E_STORE, 0, False, False, False, False)      # conv_1x1
    add("block_1x1", "pw_gemm", c, d, o.A_RAW, o.E_STORE, 0, False, False, False, False)      # its input gradient
    add("block_1x1", "pw_wgrad", d, c, o.A_RAW, o.A_RAW, 0, False)
    add("block_1x1", "pw_gemm", c, d, o.A_RAW, o.E_STORE, 0, False, False, False, True)       # conv_proj
    add("block_1x1", "bn_apply", c, True, False)
    add("block_1x1", "bn_bwd_reduce", c, True, True)
    add("block_1x1", "pw_gemm", d, c, o.A_BNB, o.E_STORE, 0, False, False, False, False)
    add("block_1x1", "pw_wgrad", c, d, o.A_BNB, o.A_RAW, 0, False)
    for inverse in (False, True):
        add("tokens", "patch_permute", d, inverse)
    add("tokens", "concat2", c, c)
    add("tokens", "split2", c, c)
    add("layernorm", "ln_stats", d)
    add("layernorm", "apply_load_mode", d, o.A_GN, 1)
    add("layernorm", "ln_bwd", d, False, False)
    add("attention", "mha_fwd", S, g["heads"], g["hd"], False, False)
    add("attention", "mha_bwd", S, g["heads"], g["hd"], False, False)
    for proj, N in (("qkv", 3 * d), ("ffn1", ffn)):
        add(f"ln_projection {proj}", "pw_gemm", N, d, o.A_GN, o.E_STORE, 1, True, False, False, False)
        add(f"ln_projection {proj}", "pw_wgrad", N, d, o.A_RAW, o.A_GN, 1, True)
    add("residuals", "pw_gemm", d, d, o.A_RAW, o.E_STORE, 1, True, True, True, False)      # out_proj + x with LN2's per-row sums
    add("residuals", "gn_finalize", d)
    add("residuals", "pw_gemm", d, ffn, o.A_SILU, o.E_STORE, 0, True, True, False, False)  # ffn2 on SiLU(h) + X1
    add("residuals dropout", "ln_stats", d)
    add("residuals dropout", "pw_gemm", d, d, o.A_RAW, o.E_STORE, 0, True, False, False, False)
    add("residuals dropout", "dropout_fwd", d, P_DROP, 0.0, True)
    add("residuals dropout", "act_fwd", o.ACT_SILU)
    add("residuals dropout", "pw_gemm", d, ffn, o.A_RAW, o.E_STORE, 0, True, False, False, False)
    for N, K in ((d, ffn), (d, d), (d, 3 * d)):  # input gradients of ffn.1, out_proj, qkv_proj
        add("dgrad shared", "pw_gemm", N, K, o.A_RAW, o.E_STORE, 0, False, False, False, False)
    add("dgrad", "pw_gemm", ffn, d, o.A_RAW, o.E_SILU_BWD, 0, False, False, False, False)   # ffn.4's with SiLU' in the epilogue
    add("dgrad dropout", "dropout_bwd", d, P_DROP, 0.0)
    add("dgrad dropout", "pw_gemm", ffn, d, o.A_RAW, o.E_STORE, 0, False, False, False, False)
    add("dgrad dropout", "act_bwd", o.ACT_SILU)
    add("wgrad", "pw_wgrad", d, ffn, o.A_RAW, o.A_SILU, 0, True)
    add("wgrad", "pw_wgrad", d, d, o.A_RAW, o.A_RAW, 0, False)
    add("wgrad dropout", "pw_wgrad", d, ffn, o.A_RAW, o.A_RAW, 0, True)
    add("wgrad dropout", "pw_wgrad", d, d, o.A_RAW, o.A_RAW, 0, True)
    add("ln_bwd", "ln_bwd", d, True, True)
    add("ln_bwd", "ln_bwd", d, True, False)
    return t


def covers(g, group, calls):
    """the calls one kernel-level test made are exactly the table's entries of its group (or groups, a tuple)"""
    groups = group if isinstance(group, tuple) else (group,)
    want = {k for k, v in block_table(g).items() if v & set(groups)}
    assert want, group
    assert set(calls) == want, f"{group}: calls {sorted(set(calls) - want)} are not in the table, {sorted(want - set(calls))} not made"


def _block(pkg, mode, li, dropout):
    """the real MobileViTBlock layer_<li>.1 of the mode, seeded, train mode"""
    opts = pkg.default_mit_opts(mode, **{"model.classification.mit.dropout": dropout})
    model = pkg.MobileViT(opts)
    model.load_state_dict(O.seeded_fill_(O.mobilevit_v1_shapes(mode), 4001), strict=True)
    return getattr(model, f"layer_{li}")[1].cuda().train()


GUARD = [pytest.param(mode, g["layer"], p, id=f"{mode}-layer_{g['layer']}.1-dropout{p}")
         for mode in MODES for g in attn_blocks(mode) for p in (0.0, P_DROP)]


@pytest.mark.parametrize("mode,li,dropout", GUARD)
def test_kernel_table_covers_the_block(pkg, ops, recorder, mode, li, dropout):
    """one real MobileViTBlock forward / backward at batch 2, 256x256, with every recorded ops wrapper recorded: each call (modulo M) must be
    one the kernel-level tests make for this block"""
    g = next(b for b in attn_blocks(mode) if b["layer"] == li)
    blk = _block(pkg, mode, li, dropout)
    x = torch.randn(2, g["c"], g["H"], g["H"], device="cuda").requires_grad_(True)
    y = blk(x)
    y.backward(torch.randn_like(y))
    torch.cuda.synchronize()
    table_ = block_table(g)
    missing = sorted(set(recorder) - set(table_))
    assert not missing, f"{mode} layer_{li}.1: the block issues calls the kernel-level table does not test: {missing}"
    assert x.grad is not None and len(set(recorder)) >= 25


# ------------------------------------------------------------------------------------------- attention
def _mha64(qkv, dO, s0, s1, S, H, hd, scale):
    """fp64 softmax attention of sequences [s0, s1) on the packed projection: O, LSE (base 2) and dQKV"""
    n = s1 - s0
    x = qkv[s0 * S:s1 * S].double().view(n, S, 3, H, hd).permute(2, 0, 3, 1, 4)
    q, k, v = x[0], x[1], x[2]
    s = (q @ k.transpose(-1, -2)) * scale
    lse = torch.logsumexp(s, -1)
    p = torch.exp(s - lse[..., None])
    o = p @ v
    do = dO[s0 * S:s1 * S].double().view(n, S, H, hd).transpose(1, 2)
    dv = p.transpose(-1, -2) @ do
    dp = do @ v.transpose(-1, -2)
    ds = p * (dp - (dp * p).sum(-1, keepdim=True))
    dq, dk = (ds @ k) * scale, (ds.transpose(-1, -2) @ q) * scale
    dqkv = torch.stack([dq, dk, dv]).permute(1, 3, 0, 2, 4).reshape(n * S, 3 * H * hd)
    return o.transpose(1, 2).reshape(n * S, H * hd), lse / LN2, dqkv


@pytest.mark.parametrize("uid", ids("attention"))
def test_attention(ops, recorder, uid):
    """mha_fwd / mha_bwd over the 512 sequences of a batch-128 block (the mma.sync kernels, one CTA per sequence and head): O, LSE and dQKV
    against fp64 softmax attention.  Negative control: the last load chunk of every head (2 channels at head_dim 30) left out of O."""
    g = TABLE[uid][1]
    n, S, H, hd = g["seqs"], g["S"], g["heads"], g["hd"]
    C = H * hd
    qkv, dO = bf(rnd(n * S, 3 * C, seed=3201)), bf(rnd(n * S, C, seed=3202))
    scale = hd ** -0.5
    O_, LSE = twice(lambda: ops.mha_fwd(qkv, n, S, H, hd, scale), ("O", "LSE"))
    (D,) = twice(lambda: [ops.mha_bwd(qkv, O_, dO, LSE, n, S, H, hd, scale)], ("dQKV",))  # one writer per element (mha.cu)
    covers(g, "attention", recorder)
    bc = max(1, (1 << 25) // (H * S * S))
    refO, refD = torch.empty(n * S, C, device="cuda"), torch.empty(n * S, 3 * C, device="cuda")
    lse_err, lse_max = 0.0, 0.0
    for s0 in range(0, n, bc):
        s1 = min(n, s0 + bc)
        o, lse, dd = _mha64(qkv, dO, s0, s1, S, H, hd, scale)
        refO[s0 * S:s1 * S], refD[s0 * S:s1 * S] = o.float(), dd.float()
        lse_err = max(lse_err, float((LSE[s0:s1].double() - lse).abs().max()))
        lse_max = max(lse_max, float(lse.abs().max()))
    check(O_, refO, "O", g, "attention")
    assert lse_err <= 1e-4 * lse_max + 1e-4, f"LSE: max err {lse_err:.3g}"
    check(D, refD, "dQKV", g, "attention", rtol=3e-2)
    w = head_load_chunk(hd) // 2
    bad = refO.clone()
    for h in range(H):
        bad[:, h * hd + hd - w:(h + 1) * hd] = 0
    rejects(lambda r: T.check_out(O_, r, "O"), [(f"last {w}-channel chunk of every head dropped", bad)])


# ------------------------------------------------------------------------------------------- dense 3x3 convs: im2col + GEMM + BatchNorm
def _patch_ref(x, sl_samples):
    """F.unfold of the samples in the kernel's column order (u, v, ci), bf16-exact"""
    xs = x[sl_samples].double()
    Bc, Cin = xs.shape[:2]
    u = F.unfold(xs, kernel_size=3, padding=1)
    return u.view(Bc, Cin, 9, -1).permute(0, 3, 2, 1).reshape(-1, 9 * Cin)


def ragged_tile_control(ref, what):
    """the last (ragged) 128-channel N tile of the output left unwritten"""
    N = ref.shape[1]
    n0 = (N - 1) // 128 * 128
    bad = ref.clone()
    bad[:, n0:] = 0
    return [(f"{what}: last N tile (columns {n0}..{N - 1}) skipped", bad)]


def tile_control(ref, what):
    """one 128 x 128 output tile in the middle of the tensor off by 5 % of the largest value"""
    m0 = (ref.shape[0] // 2) // 128 * 128
    bad = ref.clone()
    bad[m0:m0 + 128, :128] += 0.05 * float(ref.abs().max())
    return [(f"{what}: one output tile corrupted", bad)]


@pytest.mark.parametrize("uid", ids("conv3x3"))
def test_dense_conv(ops, recorder, uid):
    """local_rep.conv_3x3 (c -> c) / fusion (2c -> c) at batch 128, as PointwiseConvFn issues them.  Forward: the gathered patch matrix, the
    GEMM with the BatchNorm column statistics, BatchNorm + SiLU.  Backward: dz through SiLU' with the BatchNorm-backward sums, the input
    gradient GEMM on the BatchNorm-backward load mode (N = 9 Cin columns, up to 2880) and its col2im, and the weight gradient on whichever
    kernel K = 9 Cin % 64 selects"""
    g = TABLE[uid][1]
    Bn, H, c = g["B"], g["H"], g["c"]
    cin = 2 * c if g["conv"] == "fusion" else c
    K, M = 9 * cin, Bn * H * H
    X2 = bf(rnd(M, cin, seed=3301))
    x = X2.view(Bn, H, H, cin).permute(0, 3, 1, 2)       # logical NCHW, channels-last memory: what the block hands the conv
    W = bf(rnd(c, K, scale=K ** -0.5, seed=3302))
    Wt = bf(rnd(K, c, scale=c ** -0.5, seed=3303))
    bn, coef = bn_params(c, 3304)
    dout, y = bf(rnd(M, c, seed=3311)), bf(rnd(M, c, seed=3312) * 1.3)

    def fwd():
        A, _, _ = ops.im2col(x, 3, 1, 1)
        st = zeros64(2, c)
        Y = ops.pw_gemm(A, W, c, col_stats=st)
        return A, Y, st, ops.bn_apply(Y, bn, act=True)

    def bwd():
        sums = zeros64(2, c)
        dz = ops.bn_bwd_reduce(dout, y, sums, bn, act=True, store_dz=True)
        dA = ops.pw_gemm(dz, Wt, K, K=c, a_mode=ops.A_BNB, A2=y, a_p=coef)
        dW = ops.pw_wgrad(dz, A, c, K, g_mode=ops.A_BNB, G2=y, g_p=coef)
        return dz, sums, dA, dW, ops.col2im(dA, Bn, cin, H, H, 3, 1, 1)

    A, Y, st, out = twice(fwd, ("patch matrix", "Y", "BatchNorm statistics", "BatchNorm + SiLU"))
    dz, sums, dA, dW, dX = twice(bwd, ("dz", "BatchNorm-backward sums", "dA", "dW", "dx"))
    covers(g, f"conv {g['conv']}", recorder)
    bc = max(1, CHUNK // (H * H))
    for b0 in range(0, Bn, bc):
        b1 = min(Bn, b0 + bc)
        same(A[b0 * H * H:b1 * H * H], _patch_ref(x, slice(b0, b1)).to(torch.bfloat16), f"patch matrix, samples {b0}+")
    ref = mm64(A, W)
    check(Y, ref, "conv GEMM", g, "gemm")
    rejects(lambda r: T.check_out(Y, r, "conv GEMM"), gemm_controls(ref, A, W, "conv GEMM") + tile_control(ref, "conv GEMM"))
    del ref
    col_stats_check(st, Y, "conv GEMM")
    check(out, chunked(lambda s: silu(Y[s].double() * bn[2].double() + bn[3].double()), M, c), "BatchNorm + SiLU", g, "elementwise")
    dzr = chunked(lambda s: dout[s].double() * dsilu(y[s].double() * bn[2].double() + bn[3].double()), M, c)
    check(dz, dzr, "dz", g, "elementwise")
    col_stats_check(sums, dz, "dz", Y2=y)
    G = load_ref(ops.A_BNB, dz, coef, y)                    # the bf16 operand both GEMMs read
    ref = mm64(G, Wt)
    check(dA, ref, "dgrad GEMM", g, "gemm")
    rejects(lambda r: T.check_out(dA, r, "dgrad GEMM"), gemm_controls(ref, G, Wt, "dgrad GEMM") + ragged_tile_control(ref, "dgrad GEMM"))
    del ref
    ref = tmm64(G, A)
    check_dw(dW, ref, "conv dW", g)
    rejects(lambda r: check_wgrad(dW, r, "conv dW"), wgrad_controls(ref, G, A, "conv dW"))
    del ref, G
    fold = torch.empty(M, cin, device="cuda")
    for b0 in range(0, Bn, bc):
        b1 = min(Bn, b0 + bc)
        cols = dA[b0 * H * H:b1 * H * H].double().view(b1 - b0, H * H, 9, cin).permute(0, 3, 2, 1).reshape(b1 - b0, cin * 9, H * H)
        fold[b0 * H * H:b1 * H * H] = F.fold(cols, output_size=(H, H), kernel_size=3, padding=1).permute(0, 2, 3, 1).reshape(-1, cin).float()
    check(dX, fold, "col2im", g, "elementwise")


# ------------------------------------------------------------------------------------------- the block's 1x1 convs
@pytest.mark.parametrize("uid", ids("block_1x1"))
def test_block_pointwise(ops, recorder, uid):
    """local_rep.conv_1x1 (c -> d, no norm, no activation) and conv_proj (d -> c, BatchNorm + SiLU): forward GEMMs, input gradients (conv_proj's
    on the BatchNorm-backward load mode) and weight gradients"""
    g = TABLE[uid][1]
    M, c, d = g["B"] * g["H"] ** 2, g["c"], g["d"]
    Xc, Xd = bf(rnd(M, c, seed=3401)), bf(rnd(M, d, seed=3402))
    W1, W1t = bf(rnd(d, c, scale=c ** -0.5, seed=3403)), bf(rnd(c, d, scale=d ** -0.5, seed=3404))
    Wp, Wpt = bf(rnd(c, d, scale=d ** -0.5, seed=3405)), bf(rnd(d, c, scale=c ** -0.5, seed=3406))
    Gd, Gc, yc = bf(rnd(M, d, seed=3407)), bf(rnd(M, c, seed=3408)), bf(rnd(M, c, seed=3409))
    bn, coef = bn_params(c, 3410)

    def run():
        st, sums = zeros64(2, c), zeros64(2, c)
        t1 = ops.pw_gemm(Xc, W1, d)
        dA1 = ops.pw_gemm(Gd, W1t, c, K=d)
        dW1 = ops.pw_wgrad(Gd, Xc, d, c)
        yp = ops.pw_gemm(Xd, Wp, c, col_stats=st)
        op = ops.bn_apply(yp, bn, act=True)
        dz = ops.bn_bwd_reduce(Gc, yc, sums, bn, act=True, store_dz=True)
        dAp = ops.pw_gemm(dz, Wpt, d, K=c, a_mode=ops.A_BNB, A2=yc, a_p=coef)
        dWp = ops.pw_wgrad(dz, Xd, c, d, g_mode=ops.A_BNB, G2=yc, g_p=coef)
        return t1, dA1, dW1, yp, st, op, dz, sums, dAp, dWp

    t1, dA1, dW1, yp, st, op, dz, sums, dAp, dWp = twice(run, ("conv_1x1", "conv_1x1 dgrad", "conv_1x1 dW", "conv_proj", "conv_proj statistics",
                                                              "conv_proj BatchNorm + SiLU", "dz", "sums", "conv_proj dgrad", "conv_proj dW"))
    covers(g, "block_1x1", recorder)
    check(t1, mm64(Xc, W1), "conv_1x1", g, "gemm")
    check(dA1, mm64(Gd, W1t), "conv_1x1 dgrad", g, "gemm")
    check_dw(dW1, tmm64(Gd, Xc), "conv_1x1 dW", g)
    ref = mm64(Xd, Wp)
    check(yp, ref, "conv_proj", g, "gemm")
    rejects(lambda r: T.check_out(yp, r, "conv_proj"), tile_control(ref, "conv_proj"))
    col_stats_check(st, yp, "conv_proj")
    check(op, chunked(lambda s: silu(yp[s].double() * bn[2].double() + bn[3].double()), M, c), "conv_proj BatchNorm + SiLU", g, "elementwise")
    check(dz, chunked(lambda s: Gc[s].double() * dsilu(yc[s].double() * bn[2].double() + bn[3].double()), M, c), "dz", g, "elementwise")
    col_stats_check(sums, dz, "dz", Y2=yc)
    G = load_ref(ops.A_BNB, dz, coef, yc)
    check(dAp, mm64(G, Wpt), "conv_proj dgrad", g, "gemm")
    check_dw(dWp, tmm64(G, Xd), "conv_proj dW", g)


# ------------------------------------------------------------------------------------------- unfold / fold / concat
@pytest.mark.parametrize("uid", ids("tokens"))
def test_unfold_fold_concat(ops, recorder, uid):
    """patch_permute both ways at the full batch against the reference's unfolding / folding, concat2 / split2 of (x, conv_proj output): exact"""
    g = TABLE[uid][1]
    Bn, H, c, d = g["B"], g["H"], g["c"], g["d"]
    M = Bn * H * H
    X, Gt, A, Bt = bf(rnd(M, d, seed=3501)), bf(rnd(M, d, seed=3502)), bf(rnd(M, c, seed=3503)), bf(rnd(M, c, seed=3504))

    def run():
        cat = ops.concat2(A, Bt)
        da, db = ops.split2(cat, c, c)
        return ops.patch_permute(X, Bn, H, H, 2, 2, False), ops.patch_permute(Gt, Bn, H, H, 2, 2, True), cat, da, db

    T_, Fo, cat, da, db = twice(run, ("unfolding", "folding", "concat2", "split2 first", "split2 second"))
    covers(g, "tokens", recorder)
    same(T_, _unfold_v1(X.view(Bn, H, H, d).permute(0, 3, 1, 2), 2, 2).reshape(-1, d), "unfolding")
    same(Fo, _fold_v1(Gt.view(Bn * 4, -1, d), Bn, d, H, H, 2, 2).permute(0, 2, 3, 1).reshape(-1, d), "folding")
    same(cat, torch.cat([A, Bt], dim=1), "concat2")
    same(da, A, "split2 first")
    same(db, Bt, "split2 second")


# ------------------------------------------------------------------------------------------- LayerNorm
@pytest.mark.parametrize("uid", ids("layernorm"))
def test_layernorm(ops, recorder, uid):
    """the block's closing LayerNorm (global_rep[-1], LayerNormFn): ln_stats over every token, rows at mean 64 / std 0.5 among them, the
    normalised tokens materialised by the load-mode pass (the route the encoder takes for wide layers), and ln_bwd without a residual"""
    g = TABLE[uid][1]
    M, d = g["B"] * g["H"] ** 2, g["d"]
    X = tokens(M, d, 3601, offset_rows=True)
    V = bf(rnd(M, d, seed=3602))
    gamma, beta = 1 + 0.2 * rnd(d, seed=3603), 0.1 * rnd(d, seed=3604)

    def fwd():
        ln = ops.ln_stats(X, EPS)
        return ln, ops.apply_load_mode(X, ops.A_GN, d, a_p=(gamma, beta, None), row_stats=(ln[0], ln[1]), rows_per_sample=1)

    ln, xn = twice(fwd, ("statistics", "normalised tokens"))

    def bwd():
        col = zeros64(2, d)
        return ops.ln_bwd(V, X, ln, gamma, col), col

    DX, col = twice(bwd, ("ln_bwd dx", "dbeta / dgamma"))
    covers(g, "layernorm", recorder)
    mean = torch.empty(M, device="cuda", dtype=F64)
    var = torch.empty(M, device="cuda", dtype=F64)
    for i in range(0, M, CHUNK):
        x = X[i:i + CHUNK].double()
        mean[i:i + CHUNK], var[i:i + CHUNK] = x.mean(1), x.var(1, unbiased=False)
    err = (ln[0].double() - mean).abs()
    assert float((err - 4e-6 * mean.abs()).max()) <= 1e-4, f"mean: max err {float(err.max()):.3g}"
    plain = torch.ones(M, dtype=torch.bool, device="cuda")
    plain[::7] = False
    rstd = (var + EPS).rsqrt()
    rel = ((ln[1].double() - rstd) / rstd).abs()
    assert float(rel[plain].max()) < 1e-3, f"rstd: max rel err {float(rel[plain].max()):.3g}"
    check(xn, ln_ref64(X, gamma, beta, EPS), "LayerNorm", g, "layernorm")
    ref = torch.empty(M, d, device="cuda")
    dg, dbt = zeros64(d), zeros64(d)
    for i in range(0, M, CHUNK):
        v, x = V[i:i + CHUNK].double(), X[i:i + CHUNK].double()
        xh = (x - ln[0][i:i + CHUNK].double()[:, None]) * ln[1][i:i + CHUNK].double()[:, None]
        gv = v * gamma.double()
        ref[i:i + CHUNK] = (ln[1][i:i + CHUNK].double()[:, None] * (gv - gv.mean(1, keepdim=True) - xh * (gv * xh).mean(1, keepdim=True))).float()
        dg += (v * xh).sum(0)
        dbt += v.sum(0)
    check(DX, ref, "ln_bwd dx", g, "layernorm")
    close_stat(col[0], dbt, "dbeta", rtol=5e-3)
    close_stat(col[1], dg, "dgamma", rtol=5e-3)


# ------------------------------------------------------------------------------------------- the encoders' GEMMs
def _mask(ops, seed, M, C, S, skip=0):
    """the keep mask (1 kept / 0 dropped) of the key drawn after ``skip`` others from a generator seeded with ``seed``, as the hashed-mask
    kernel applies it to an [M, C] branch with S rows per sample; its values must be exactly 0 or the bf16 1 / (1 - p)"""
    ops.rng_seed(seed)
    for _ in range(skip):
        ops.rng_next("cuda")
    m = ops.dropout_fwd(torch.ones(M, C, device="cuda", dtype=torch.bfloat16), None, P_DROP, ops.rng_next("cuda"), rows_per_sample=S).float()
    scale = float(torch.tensor(1 / (1 - P_DROP)).to(torch.bfloat16))
    assert bool(((m == 0) | ((m - scale).abs() < 1e-6)).all())
    return (m != 0).float()


def _enc(uid):
    g = TABLE[uid][1]
    return g, g["B"] * g["H"] ** 2, g["d"], g["ffn"]


@pytest.mark.parametrize("route", ["model", "pre-pass"])
@pytest.mark.parametrize("proj", ["qkv", "ffn1"])
@pytest.mark.parametrize("uid", ids("encoder"))
def test_ln_projection(ops, recorder, uid, proj, route):
    """qkv_proj / ffn.1: LayerNorm(X) @ W^T + b and its weight gradient with the bias gradient, on the encoder's two LayerNorm routes: the
    load mode inside the GEMM and the weight-gradient kernel (what these widths take), and the normalised tokens kept from one pre-pass
    (what the wide ViT layers take; functional._encoder_forward ln_proj / ln_wgrad)"""
    g, M, C, ffn = _enc(uid)
    N = 3 * C if proj == "qkv" else ffn
    X = tokens(M, C, 3701)
    ln = ops.ln_stats(X, EPS)
    recorder.clear()
    gamma, beta = 1 + 0.2 * rnd(C, seed=3702), 0.1 * rnd(C, seed=3703)
    W, bias = layer_params(N, C, 3704)
    G = bf(rnd(M, N, seed=3706))
    kw = dict(a_p=(gamma, beta), row_stats=(ln[0], ln[1]), rows_per_sample=1)

    def run():
        db = torch.zeros(N, device="cuda")
        if route == "pre-pass":
            xn = ops.apply_load_mode(X, ops.A_GN, C, **kw)
            return ops.pw_gemm(xn, W, N, bias=bias), ops.pw_wgrad(G, xn, N, C, dbias=db), db
        return ops.pw_gemm(X, W, N, a_mode=ops.A_GN, bias=bias, **kw), ops.pw_wgrad(G, X, N, C, a_mode=ops.A_GN, dbias=db, **kw), db

    out, dW, db = twice(run, ("out", "dW", "dbias"))
    if route == "model":
        covers(g, f"ln_projection {proj}", recorder)
    Xn = load_ref(ops.A_GN, X, (gamma, beta), row=(ln[0], ln[1]), rps=1)
    ref = mm64(Xn, W) + bias
    check(out, ref, f"{proj} {route}", g, "gemm")
    rejects(lambda r: T.check_out(out, r, proj), tile_control(ref, proj))
    check_dw(dW, tmm64(G, Xn), f"{proj} {route} dW", g)
    bias_check(db, G, f"{proj} dbias")


@pytest.mark.parametrize("drop", [False, True], ids=["dropout0", "recipe-dropout"])
@pytest.mark.parametrize("uid", ids("encoder"))
def test_residual_branches(ops, recorder, uid, drop):
    """the attention and FFN branches with their residual adds.  Dropout 0: X1 = O Wo^T + bo + x with LN2's per-row sums in the epilogue and
    gn_finalize turning them into statistics, X2 = SiLU(h) W2^T + b2 + X1 with SiLU as the load mode.  The recipe's dropout 0.1: the GEMMs
    store the branch, the hashed-mask kernel adds it to the residual, LN2 from ln_stats, SiLU as its own pass"""
    g, M, C, ffn = _enc(uid)
    S = g["S"]
    Oa, x2, h = bf(rnd(M, C, seed=3801)), tokens(M, C, 3802), bf(rnd(M, ffn, seed=3803) * 1.5)
    Wo, bo = layer_params(C, C, 3804)
    W2, b2 = layer_params(C, ffn, 3806)
    X1in = tokens(M, C, 3808)
    ops.rng_seed(11)
    k1, k2 = ops.rng_next("cuda"), ops.rng_next("cuda")

    def run():
        if not drop:
            samp = zeros64(2, M)
            X1 = ops.pw_gemm(Oa, Wo, C, bias=bo, R=x2, samp_stats=samp, rows_per_sample=1)
            return X1, samp, ops.gn_finalize(samp, C, EPS), ops.pw_gemm(h, W2, C, a_mode=ops.A_SILU, bias=b2, R=X1in)
        A = ops.pw_gemm(Oa, Wo, C, bias=bo)
        X1 = ops.dropout_fwd(A, x2, P_DROP, k1, rows_per_sample=S)
        ha = ops.act_fwd(h, ops.ACT_SILU)
        Fo = ops.pw_gemm(ha, W2, C, bias=b2)
        return A, X1, ops.ln_stats(X1, EPS), ha, Fo, ops.dropout_fwd(Fo, X1in, P_DROP, k2, rows_per_sample=S)

    if not drop:
        X1, samp, ln2, X2 = twice(run, ("X1", "per-row sums", "LN2 statistics", "X2"))
        covers(g, "residuals", recorder)
        check(X1, mm64(Oa, Wo) + bo + x2.float(), "out_proj + residual", g, "gemm")
        x = X1.double()
        s, q = x.sum(1), (x * x).sum(1)
        close_stat(samp[0], s, "per-row sum")
        close_stat(samp[1], q, "per-row sum of squares")
        mean, var = s / C, (x - (s / C)[:, None]).pow(2).mean(1)
        assert float((ln2[0].double() - mean).abs().max()) <= 1e-5 * float(mean.abs().max()) + 1e-6
        rstd = (var + EPS).rsqrt()
        r = float(((ln2[1].double() - rstd) / rstd).abs().max())
        assert r <= 1e-4, f"LN2 rstd: max rel err {r:.3g}"
        ref = mm64(load_ref(ops.A_SILU, h), W2) + b2 + X1in.float()
        check(X2, ref, "ffn2 + residual", g, "gemm")
        rejects(lambda r_: T.check_out(X2, r_, "ffn2"), gemm_controls(ref, load_ref(ops.A_SILU, h), W2, "ffn2"))
        return
    A, X1, ln2, ha, Fo, X2 = twice(run, ("out_proj", "X1", "LN2 statistics", "SiLU", "ffn2", "X2"))
    covers(g, "residuals dropout", recorder)
    check(A, mm64(Oa, Wo) + bo, "out_proj", g, "gemm")
    check(ha, chunked(lambda s_: silu(h[s_].double()), M, ffn), "SiLU", g, "elementwise")
    check(Fo, mm64(ha, W2) + b2, "ffn2", g, "gemm")
    for seed_k, br, res, Y, what in ((0, A, x2, X1, "attention branch"), (1, Fo, X1in, X2, "FFN branch")):
        keep = _mask(ops, 11, M, C, S, skip=seed_k)
        rate = float(keep.mean())
        assert abs(rate - (1 - P_DROP)) <= 5e-3, f"{what}: keep rate {rate:.4f}"
        check(Y, res.float() + br.float() * keep / (1 - P_DROP), f"{what} + residual", g, "elementwise")
    x = X1.double()
    assert float((ln2[0].double() - x.mean(1)).abs().max()) <= 1e-4 * float(x.abs().max()) + 1e-5
    rstd = (x.var(1, unbiased=False) + EPS).rsqrt()
    assert float(((ln2[1].double() - rstd) / rstd).abs().max()) <= 1e-3


@pytest.mark.parametrize("drop", [False, True], ids=["dropout0", "recipe-dropout"])
@pytest.mark.parametrize("uid", ids("encoder"))
def test_encoder_dgrad(ops, recorder, uid, drop):
    """the input-gradient GEMMs on the transposed weights: dh = (dY W2) * SiLU'(h) in the epilogue (dropout 0) or through the regenerated mask
    and act_bwd (dropout 0.1), vF = dh W1 (K = ffn), dO = dA Wo, vA = dqkv Wqkv (K = 3C)"""
    g, M, C, ffn = _enc(uid)
    S = g["S"]
    dY, dh, dA, dq = bf(rnd(M, C, seed=3901)), bf(rnd(M, ffn, seed=3902)), bf(rnd(M, C, seed=3903)), bf(rnd(M, 3 * C, seed=3904))
    h = bf(rnd(M, ffn, seed=3905) * 1.5)
    W2t, W1t = layer_params(ffn, C, 3906)[0], layer_params(C, ffn, 3907)[0]
    Wot, Wqt = layer_params(C, C, 3908)[0], layer_params(C, 3 * C, 3909)[0]
    ops.rng_seed(12)
    k2 = ops.rng_next("cuda")

    def run():
        rest = (ops.pw_gemm(dh, W1t, C, K=ffn), ops.pw_gemm(dA, Wot, C, K=C), ops.pw_gemm(dq, Wqt, C, K=3 * C))
        if not drop:
            return (ops.pw_gemm(dY, W2t, ffn, K=C, e_mode=ops.E_SILU_BWD, Y=h),) + rest
        dF = ops.dropout_bwd(dY, P_DROP, k2, rows_per_sample=S)
        dha = ops.pw_gemm(dF, W2t, ffn, K=C)
        return (dF, dha, ops.act_bwd(dha, h, ops.ACT_SILU)) + rest

    if drop:
        dF, dha, dhr, vF, dO, vA = twice(run, ("dF", "dha", "SiLU backward", "vF", "dO", "vA"))
        covers(g, ("dgrad dropout", "dgrad shared"), recorder)
        keep = _mask(ops, 12, M, C, S)
        check(dF, dY.float() * keep / (1 - P_DROP), "dropout backward (the forward's mask)", g, "elementwise")
        check(dha, mm64(dF, W2t), "ffn2 dgrad", g, "gemm")
        check(dhr, chunked(lambda s: dha[s].double() * dsilu(h[s].double()), M, ffn), "SiLU backward", g, "elementwise")
    else:
        dhr, vF, dO, vA = twice(run, ("dh", "vF", "dO", "vA"))
        covers(g, ("dgrad", "dgrad shared"), recorder)
        check(dhr, chunked(lambda s: (dY[s].double() @ W2t.double().t()) * dsilu(h[s].double()), M, ffn), "ffn2 dgrad * SiLU'", g, "gemm")
    for out, A, W, what in ((vF, dh, W1t, "ffn1 dgrad"), (dO, dA, Wot, "out_proj dgrad"), (vA, dq, Wqt, "qkv dgrad")):
        ref = mm64(A, W)
        check(out, ref, what, g, "gemm")
        if what == "ffn1 dgrad":
            rejects(lambda r, out=out, what=what: T.check_out(out, r, what), gemm_controls(ref, A, W, what))


@pytest.mark.parametrize("drop", [False, True], ids=["dropout0", "recipe-dropout"])
@pytest.mark.parametrize("uid", ids("encoder"))
def test_encoder_wgrad(ops, recorder, uid, drop):
    """ffn.4: dW2 = dY^T SiLU(h) (SiLU as the load mode; with dropout on the stored SiLU output) with its bias gradient; out_proj:
    dWo = dA^T O (its bias gradient from ln_bwd's column sums, or with dropout from the weight-gradient kernel)"""
    g, M, C, ffn = _enc(uid)
    dY, h, dA, Oa = bf(rnd(M, C, seed=4001)), bf(rnd(M, ffn, seed=4002)), bf(rnd(M, C, seed=4003)), bf(rnd(M, C, seed=4004))

    def run():
        db2, dbo = torch.zeros(C, device="cuda"), torch.zeros(C, device="cuda")
        if drop:
            return ops.pw_wgrad(dY, h, C, ffn, dbias=db2), db2, ops.pw_wgrad(dA, Oa, C, C, dbias=dbo), dbo
        return ops.pw_wgrad(dY, h, C, ffn, a_mode=ops.A_SILU, dbias=db2), db2, ops.pw_wgrad(dA, Oa, C, C), dbo

    dW2, db2, dWo, dbo = twice(run, ("dW2", "db2", "dWo", "dbo"))
    covers(g, "wgrad dropout" if drop else "wgrad", recorder)
    Ha = h.float() if drop else load_ref(ops.A_SILU, h)
    ref = tmm64(dY, Ha)
    check_dw(dW2, ref, "ffn2 dW", g)
    rejects(lambda r: check_wgrad(dW2, r, "ffn2 dW"), wgrad_controls(ref, dY, Ha, "ffn2 dW"))
    bias_check(db2, dY, "ffn2 dbias")
    check_dw(dWo, tmm64(dA, Oa), "out_proj dW", g)
    if drop:
        bias_check(dbo, dA, "out_proj dbias")


@pytest.mark.parametrize("uid", ids("encoder"))
def test_encoder_ln_bwd(ops, recorder, uid):
    """dX1 = LN2 backward of vF + dY with the column sums (= d(out_proj bias)), and dx = LN1 backward of vA + dX1"""
    g, M, C, _ = _enc(uid)
    V, X, Rr = bf(rnd(M, C, seed=4101)), tokens(M, C, 4102), bf(rnd(M, C, seed=4103))
    gamma = 1 + 0.2 * rnd(C, seed=4104)
    ln = ops.ln_stats(X, EPS)
    recorder.clear()

    def run():
        col, cs, col1 = zeros64(2, C), zeros64(C), zeros64(2, C)
        DX = ops.ln_bwd(V, X, ln, gamma, col, DRES=Rr, col_sum=cs)
        return DX, col, cs, ops.ln_bwd(V, X, ln, gamma, col1, DRES=DX), col1

    DX, col, cs, DX1, col1 = twice(run, ("dx", "dbeta / dgamma", "column sums", "dx (residual = dx)", "dbeta / dgamma (second)"))
    covers(g, "ln_bwd", recorder)
    ref = torch.empty(M, C, device="cuda")
    dg, dbt = zeros64(C), zeros64(C)
    for i in range(0, M, CHUNK):
        v, x = V[i:i + CHUNK].double(), X[i:i + CHUNK].double()
        mu, rs = ln[0][i:i + CHUNK].double()[:, None], ln[1][i:i + CHUNK].double()[:, None]
        xh = (x - mu) * rs
        gv = v * gamma.double()
        ref[i:i + CHUNK] = (rs * (gv - gv.mean(1, keepdim=True) - xh * (gv * xh).mean(1, keepdim=True)) + Rr[i:i + CHUNK].double()).float()
        dg += (v * xh).sum(0)
        dbt += v.sum(0)
    check(DX, ref, "ln_bwd dx", g, "layernorm")
    close_stat(col[0], dbt, "dbeta", rtol=5e-3)
    close_stat(col[1], dg, "dgamma", rtol=5e-3)
    close_stat(cs, DX.double().sum(0), "column sums of dx", rtol=5e-3)
    check(DX1, ref - Rr.float() + DX.float(), "ln_bwd dx (residual = dx)")
    close_stat(col1[0], dbt, "dbeta (second)", rtol=5e-3)


# ------------------------------------------------------------------------------------------- expand-4 inverted residuals
@pytest.mark.parametrize("uid", ids("ir"))
def test_inverted_residual_gemms(ops, uid):
    """the GEMMs InvertedResidualFn issues at batch 128: exp_1x1 with BatchNorm statistics, red_1x1 on the expansion's BatchNorm + SiLU load
    mode, the output BatchNorm (+ the residual), red_1x1's input gradient on the BatchNorm-backward load mode with SiLU' and the sums in the
    epilogue, exp_1x1's (+ the residual's gradient), both weight gradients and the output BatchNorm-backward sums"""
    g = TABLE[uid][1]
    Bn, H, cin, hid, cout, s = g["B"], g["H"], g["cin"], g["hid"], g["cout"], g["stride"]
    M, M2 = Bn * H * H, Bn * ((H - 1) // s + 1) ** 2
    residual = s == 1 and cin == cout
    x2, y2 = bf(rnd(M, cin, seed=4201)), bf(rnd(M2, hid, seed=4202))
    W1, W3 = bf(rnd(hid, cin, scale=cin ** -0.5, seed=4203)), bf(rnd(cout, hid, scale=hid ** -0.5, seed=4204))
    W3t, W1t = bf(rnd(hid, cout, scale=cout ** -0.5, seed=4205)), bf(rnd(cin, hid, scale=hid ** -0.5, seed=4206))
    bn2, _ = bn_params(hid, 4207)
    bn3, c3 = bn_params(cout, 4211)
    _, c1 = bn_params(hid, 4215)
    y3, dout, dz1, y1 = bf(rnd(M2, cout, seed=4221)), bf(rnd(M2, cout, seed=4222)), bf(rnd(M, hid, seed=4223)), bf(rnd(M, hid, seed=4224))
    xres = bf(rnd(M2, cout, seed=4225)) if residual else None
    ap2 = (bn2[2], bn2[3])

    def run():
        st1, st3, sd3, sd2 = zeros64(2, hid), zeros64(2, cout), zeros64(2, cout), zeros64(2, hid)
        a = ops.pw_gemm(x2, W1, hid, col_stats=st1)
        b = ops.pw_gemm(y2, W3, cout, a_mode=ops.A_AFF_SILU, a_p=ap2, col_stats=st3)
        o = ops.bn_apply(y3, bn3, act=False, R=xres)
        ops.bn_bwd_reduce(dout, y3, sd3, bn3, act=False, store_dz=False)
        dz2 = ops.pw_gemm(dout, W3t, hid, K=cout, a_mode=ops.A_BNB, A2=y3, a_p=c3, e_mode=ops.E_SILU_BWD, Y=y2, e_p=ap2, col_stats=sd2)
        dW3 = ops.pw_wgrad(dout, y2, cout, hid, g_mode=ops.A_BNB, G2=y3, g_p=c3, a_mode=ops.A_AFF_SILU, a_p=ap2)
        dx = ops.pw_gemm(dz1, W1t, cin, K=hid, a_mode=ops.A_BNB, A2=y1, a_p=c1, R=dout if residual else None)
        dW1 = ops.pw_wgrad(dz1, x2, hid, cin, g_mode=ops.A_BNB, G2=y1, g_p=c1)
        return a, st1, b, st3, o, sd3, dz2, sd2, dW3, dx, dW1

    a, st1, b, st3, o, sd3, dz2, sd2, dW3, dx, dW1 = twice(run, ("exp_1x1", "exp statistics", "red_1x1", "red statistics", "output BatchNorm",
                                                                "output BatchNorm-backward sums", "red_1x1 dgrad", "its sums", "red_1x1 dW",
                                                                "exp_1x1 dgrad", "exp_1x1 dW"))
    ref = mm64(x2, W1)
    check(a, ref, "exp_1x1", g, "gemm")
    rejects(lambda r: T.check_out(a, r, "exp_1x1"), tile_control(ref, "exp_1x1"))
    del ref
    col_stats_check(st1, a, "exp_1x1")
    Y2a = load_ref(ops.A_AFF_SILU, y2, ap2 + (None,))
    check(b, mm64(Y2a, W3), "red_1x1", g, "gemm")
    col_stats_check(st3, b, "red_1x1")
    check(o, chunked(lambda s_: y3[s_].double() * bn3[2].double() + bn3[3].double() + (xres[s_].double() if residual else 0), M2, cout),
          "output BatchNorm", g, "elementwise")
    col_stats_check(sd3, dout, "output dz", Y2=y3)
    G3 = load_ref(ops.A_BNB, dout, c3, y3)
    check(dz2, chunked(lambda s_: (G3[s_].double() @ W3t.double().t()) * dsilu(y2[s_].double() * bn2[2].double() + bn2[3].double()), M2, hid),
          "red_1x1 dgrad", g, "gemm")
    col_stats_check(sd2, dz2, "red_1x1 dgrad", Y2=y2)
    check_dw(dW3, tmm64(G3, Y2a), "red_1x1 dW", g)
    del G3, Y2a
    G1 = load_ref(ops.A_BNB, dz1, c1, y1)
    check(dx, mm64(G1, W1t) + (dout.float() if residual else 0), "exp_1x1 dgrad", g, "gemm")
    check_dw(dW1, tmm64(G1, x2), "exp_1x1 dW", g)


def _dw_layers():
    seen = {(H, C, s) for H, C, s in R.DW_LAYERS}
    out = []
    for uid in ids("ir"):
        g = TABLE[uid][1]
        key = (g["H"], g["hid"], g["stride"])
        if key not in seen:
            seen.add(key)
            out.append(pytest.param(*key, id=f"{uid}-H{key[0]}-C{key[1]}-s{key[2]}"))
    return out


@pytest.mark.parametrize("H,C,s", _dw_layers())
def test_inverted_residual_depthwise(ops, H, C, s):
    """the expand-4 hidden widths' depthwise 3x3 forward (input: the expansion's BatchNorm + SiLU) and backward (BatchNorm-backward load mode),
    at a batch that makes every CTA's image loop run unevenly (test_reproducible_gpu's grid restatement)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    R._check_dw_fwd(ops, R.dw_batch(R.dw_fwd_grid(H, H, C, s, sms)), H, C, s, 1, 2, seed=4300 + H + C)
    R._check_dw_bwd(ops, R.dw_batch(R.dw_bwd_grid(H, H, C, s, sms)), H, C, s, 1, 5, 2, seed=4400 + H + C)


# ------------------------------------------------------------------------------------------- conv_1x1_exp and the classifier
@pytest.mark.parametrize("uid", ids("head"))
def test_head(ops, uid):
    """conv_1x1_exp (96 -> 384 / 160 -> 640 on the 8x8 maps, BatchNorm + SiLU) forward, input and weight gradients; global pooling; the
    1000-way classifier (LinearFn) forward, input gradient, weight and bias gradients; the pooling's adjoint"""
    g = TABLE[uid][1]
    Bn, cin, ex, ncls, HW = g["B"], g["cin"], g["exp"], g["ncls"], g["HW"]
    M = Bn * HW
    x2, W, Wt = bf(rnd(M, cin, seed=4501)), bf(rnd(ex, cin, scale=cin ** -0.5, seed=4502)), bf(rnd(cin, ex, scale=ex ** -0.5, seed=4503))
    dz, y = bf(rnd(M, ex, seed=4504)), bf(rnd(M, ex, seed=4505))
    bn, coef = bn_params(ex, 4506)
    feat = bf(rnd(M, ex, seed=4507) + 0.3)
    Wc, bc = layer_params(ncls, ex, 4508)
    Wct = bf(rnd(ex, ncls, scale=ncls ** -0.5, seed=4510))
    gl = bf(rnd(Bn, ncls, seed=4511))

    def run():
        st = zeros64(2, ex)
        yk = ops.pw_gemm(x2, W, ex, col_stats=st)
        dA = ops.pw_gemm(dz, Wt, cin, K=ex, a_mode=ops.A_BNB, A2=y, a_p=coef)
        dW = ops.pw_wgrad(dz, x2, ex, cin, g_mode=ops.A_BNB, G2=y, g_p=coef)
        pooled = ops.global_pool_fwd(feat, Bn, HW)
        logits = ops.pw_gemm(pooled, Wc, ncls, bias=bc)
        db = torch.zeros(ncls, device="cuda")
        dWc = ops.pw_wgrad(gl, pooled, ncls, ex, dbias=db)
        dp = ops.pw_gemm(gl, Wct, ex, K=ncls)
        return yk, st, dA, dW, pooled, logits, dWc, db, dp, ops.global_pool_bwd(dp, Bn, HW)

    yk, st, dA, dW, pooled, logits, dWc, db, dp, dfeat = twice(run, ("conv_1x1_exp", "statistics", "dgrad", "dW", "pooled", "logits",
                                                                    "classifier dW", "classifier dbias", "dpooled", "dfeatures"))
    check(yk, mm64(x2, W), "conv_1x1_exp", g, "gemm")
    col_stats_check(st, yk, "conv_1x1_exp")
    G = load_ref(ops.A_BNB, dz, coef, y)
    check(dA, mm64(G, Wt), "conv_1x1_exp dgrad", g, "gemm")
    check_dw(dW, tmm64(G, x2), "conv_1x1_exp dW", g)
    check(pooled, feat.double().view(Bn, HW, ex).mean(1).float(), "global pool", g, "elementwise")
    check(logits, mm64(pooled, Wc) + bc, "classifier", g, "gemm")
    check_dw(dWc, tmm64(gl, pooled), "classifier dW", g)
    bias_check(db, gl, "classifier dbias")
    check(dp, mm64(gl, Wct), "classifier dgrad", g, "gemm")
    check(dfeat, (dp.double() / HW).repeat_interleave(HW, 0).float(), "global pool adjoint", g, "elementwise")


# ------------------------------------------------------------------------------------------- model level
def mobilevit_v1_arch(mode):
    """test_parity_gpu's model-family record for MobileViT-v1 in one mode, every dropout 0 (the oracle has none)"""
    return SimpleNamespace(
        build=lambda pkg: pkg.MobileViT(pkg.default_mit_opts(mode, **{"model.classification.mit.dropout": 0.0,
                                                                     "model.classification.classifier_dropout": 0.0})),
        shapes=lambda: O.mobilevit_v1_shapes(mode), forward=lambda P, x, **kw: O.mobilevit_v1_forward(P, x, mode=mode, **kw),
        layout=lambda: O.mobilevit_v1_layout(mode))


@pytest.mark.parametrize("mode", MODES)
def test_model_against_reference_fixture(pkg, golden_dir, mode):
    """the state_dict keys, eval logits at 1x3x256x256 and a train step at 2x3x256x256 against the real reference's fp32 record, bounded by
    the oracle under bf16 autocast"""
    fx = load_mit_fixture(golden_dir, mode)
    e, et = check_mobilevit_v1_against_fixture(pkg, fx, (fx["batch"], 3, fx["res"], fx["res"]))
    _record(f"mit_{mode}_fixture", {"eval_logits_rel_l2": e, "train_logits_rel_l2": et})


@pytest.mark.parametrize("mode", MODES)
def test_stagewise_parity(pkg, mode):
    """every module fed the fp32 oracle's input of its stage, batch 128 at 256x256, train mode: rel-L2 <= 1.5e-2 per stage"""
    rec = stagewise_record(pkg, B=128, arch=mobilevit_v1_arch(mode))
    torch.cuda.empty_cache()
    print(f"\n[stage-wise parity {mode} B=128 train] " + json.dumps(rec))
    _record(f"stagewise_mit_{mode}_B128", rec)
    assert len(rec) == len(O.mobilevit_v1_layout(mode)) + 1
    for k, e in rec.items():
        assert e <= 1.5e-2, (k, e, rec)


@pytest.mark.parametrize("mode", MODES)
def test_train_step_parity(pkg, mode):
    """batch 16 at 256x256: logits, loss and gradients against the fp32 oracle, no further from it than torch bf16 autocast"""
    rec, sig = train_parity_record(pkg, 16, arch=mobilevit_v1_arch(mode))
    torch.cuda.empty_cache()
    print(f"\n[parity {mode} B=16 train] " + json.dumps(rec))
    _record(f"train_mit_{mode}_B16", rec)
    assert rec["logits_rel_l2"] <= 1.15 * rec["autocast_logits_rel_l2"] + 2e-3, rec
    assert abs(rec["loss"] - rec["loss_fp32"]) <= max(2e-3 * abs(rec["loss_fp32"]), 1.5 * abs(rec["loss_autocast"] - rec["loss_fp32"])), rec
    assert rec["grad_rel_l2_all"] <= 1.15 * rec["autocast_grad_rel_l2_all"] + 2e-3, rec
    assert rec["grad_cosine_all"] >= rec["autocast_grad_cosine_all"] - 2e-3, rec
    for t in sig:
        assert t[4] <= 1.5 * t[5] + 2e-2, t


def test_train_step_bitwise_small_with_recipe_dropouts(pkg, ops):
    """MobileViT-S with the recipe's dropouts (mit.dropout 0.1, classifier_dropout 0.1), batch 16 at 256x256, three AdamW steps: eager twice,
    without programmatic dependent launch, with the weight gradients on the main stream and replayed from a captured graph all end in the
    same bits -- the dropout masks come from the device-side generator, rewound to the same state for every run"""
    Bt = 16

    def build():
        m = pkg.MobileViT(pkg.default_mit_opts("small"))
        m.load_state_dict(O.seeded_fill_(O.mobilevit_v1_shapes("small"), 17), strict=True)
        return m.cuda().train()

    xs = [O.seeded_input((Bt, 3, 256, 256), 270 + i).cuda() for i in range(3)]
    ys = [(torch.arange(Bt, device="cuda") * (13 + i)) % 1000 for i in range(3)]
    ref_l, ref_s = R._train(pkg, ops, xs, ys, build=build)
    for what, kw in (("eager rerun", {}), ("PDL off", {"pdl": False}), ("side stream off", {"side": False}), ("graph replay", {"graph": True})):
        losses, st = R._train(pkg, ops, xs, ys, build=build, **kw)
        for i, (a, b) in enumerate(zip(losses, ref_l)):
            same(a, b, f"{what}: loss of step {i}")
        assert st.keys() == ref_s.keys()
        bad = [k for k in ref_s if not torch.equal(st[k], ref_s[k])]
        assert not bad, f"{what}: {len(bad)} of {len(ref_s)} state tensors differ from the first eager run, e.g. {bad[:6]}"
    assert float(ref_s["step"]) == 3.0


@pytest.mark.parametrize("mode,crop,layer,d", [(m, *c) for m in MODES for c in colliding_crops(m)])
def test_refuses_where_tokens_equal_width(pkg, ops, monkeypatch, mode, crop, layer, d):
    """at a recipe crop where a block has as many tokens as channels (MobileViT-S at 192x192: 144 tokens of width 144 in layer 3) the
    reference's LayerNorm would normalise over the token axis; the model raises NotImplementedError before that block's encoders issue
    any kernel"""
    model = pkg.MobileViT(pkg.default_mit_opts(mode)).cuda().train()
    launched = []
    real = ops.mha_fwd
    monkeypatch.setattr(ops, "mha_fwd", lambda *a, **k: launched.append(a[2]) or real(*a, **k))
    x = torch.randn(2, 3, crop, crop, device="cuda")
    with pytest.raises(NotImplementedError, match="S == C"):
        model(x)
    assert not launched, f"attention ran at {launched} tokens before the refusal"

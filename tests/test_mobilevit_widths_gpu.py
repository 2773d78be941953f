"""MobileViTv2 at the published widths 0.75 - 2.0 (-m gpu): the kernels at every shape these widths give them, and the model end to end.

The other suites run MobileViTv2 at widths 0.5 and 1.0 only.  The other widths reach paths those never do: attention dims d from 96 to 512
(at d = 336 / 448 one row's 8-channel groups span three warps, and linattn_bwd sums three warp pieces of ds), ragged last wgmma N tiles
(qkv N = 2d + 8), GroupNorm row blocks whose thread count is not a multiple of 32, and the wide-layer pre-pass (ops.WIDE_K / WIDE_N /
WIDE_N_WGRAD), which no MobileViTv2-1.0 layer triggers.

Kernel level: every shape comes from oracle.mobilevit_v2_config at batch 128 and 256x256, minus the shapes width 1.0 already covers.  Each
call runs twice (torch.equal) and is compared with an fp64 restatement on the same bf16-rounded inputs.  Model level: the real reference's
fixtures (mobilevit_v2_w<width>_fp32.pt), stage-wise parity at batch 128, an end-to-end train step at batch 16 against the fp32 oracle and its
bf16-autocast counterpart, and the MobileViTv2-2.0 TrainStep bitwise across launch paths."""
import json
import os
import sys

import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import test_reproducible_gpu as R  # noqa: E402
from oracle import cvnets_oracle as O  # noqa: E402
from test_kernels_gpu import bf, close, close_stat, dsilu, load_ref, rnd  # noqa: E402
from test_mobilevit_widths_cpu import load_width_fixture  # noqa: E402
from test_modules_gpu import check_model_against_fixture  # noqa: E402
from test_parity_gpu import _record, stagewise_record, train_parity_record  # noqa: E402
from test_reproducible_gpu import same, twice, zeros64  # noqa: E402

pytestmark = pytest.mark.gpu

WIDTHS = [0.75, 1.25, 1.5, 1.75, 2.0]
B, RES = 128, 256


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


@pytest.fixture(scope="module")
def sms(ops):
    return torch.cuda.get_device_properties(0).multi_processor_count


# ------------------------------------------------------------------------------------------- shapes from the configuration
def attn_stages(width):
    """(layer, H, d, ffn, C) of the three MobileViTv2 blocks at 256x256 input: layer 3 at 32^2, 4 at 16^2, 5 at 8^2"""
    cfg, shapes = O.mobilevit_v2_config(width), O.mobilevit_v2_shapes(width)
    out = []
    for li in (3, 4, 5):
        c = cfg[f"layer{li}"]
        ffn = shapes[f"layer_{li}.1.global_rep.0.pre_norm_ffn.1.block.conv.weight"].shape[0]
        out.append((li, RES >> li, c["attn_unit_dim"], ffn, c["out_channels"]))
    return out


_COVERED = set(attn_stages(1.0))
ATTN = [pytest.param(w, *st, id=f"w{w}-layer{st[0]}-d{st[2]}") for w in WIDTHS for st in attn_stages(w) if st not in _COVERED]


def inverted_residuals(width):
    """(prefix, H_in, Cin, hid, Cout, stride, input mode) of every InvertedResidual at 256x256 input.  The input mode is the load mode the
    model applies to the block's input: a producer without a residual hands its output over before its BatchNorm (models.py), unless this
    block adds its input back."""
    from ml_cvnets_b200.ops import A_AFF, A_AFF_SILU, A_RAW
    cfg = O.mobilevit_v2_config(width)
    shapes = O.mobilevit_v2_shapes(width)
    out, H, cin, prev = [], RES // 2, cfg["layer0"]["out_channels"], "stem"
    for kind, pre, kw in O.mobilevit_v2_layout(width):
        if kind == "ir":
            hid, cout = shapes[pre + ".block.exp_1x1.block.conv.weight"].shape[0], shapes[pre + ".block.red_1x1.block.conv.weight"].shape[0]
            residual = kw["stride"] == 1 and cin == cout
            mode = A_RAW if residual or prev == "ir_res" else (A_AFF_SILU if prev == "stem" else A_AFF)
            out.append((pre, H, cin, hid, cout, kw["stride"], mode))
            H, cin, prev = (H - 1) // kw["stride"] + 1, cout, "ir_res" if residual else "ir"
        elif kind == "mvit":
            prev = "mvit"
    return out


def wide_gemms(width):
    """Every pointwise GEMM / weight gradient of the model with a load-mode prologue, as (name, kind, M, N, K, a_mode, rows_per_sample)."""
    from ml_cvnets_b200.ops import A_AFF_SILU, A_BNB, A_GN, A_SILU
    out = []
    for pre, H, cin, hid, cout, s, mode in inverted_residuals(width):
        M, M2 = B * H * H, B * (((H - 1) // s + 1) ** 2)
        out += [(f"{pre} exp_1x1", "fwd", M, hid, cin, mode, 0), (f"{pre} red_1x1", "fwd", M2, cout, hid, A_AFF_SILU, 0),
                (f"{pre} red_1x1 dgrad", "fwd", M2, hid, cout, A_BNB, 0), (f"{pre} exp_1x1 dgrad", "fwd", M, cin, hid, A_BNB, 0),
                (f"{pre} red_1x1 wgrad", "wgrad", M2, cout, hid, A_AFF_SILU, 0), (f"{pre} exp_1x1 wgrad", "wgrad", M, hid, cin, mode, 0)]
    for li, H, d, ffn, C in attn_stages(width):
        M, pre = B * H * H, f"layer_{li}.1"
        out += [(f"{pre} local 1x1", "fwd", M, d, C, A_AFF_SILU, 0), (f"{pre} qkv", "fwd", M, 2 * d + 8, d, A_GN, H * H),
                (f"{pre} ffn1", "fwd", M, ffn, d, A_GN, H * H), (f"{pre} ffn2", "fwd", M, d, ffn, A_SILU, 0),
                (f"{pre} conv_proj", "fwd", M, C, d, A_GN, H * H), (f"{pre} conv_proj dgrad", "fwd", M, d, C, A_BNB, 0),
                (f"{pre} local 1x1 wgrad", "wgrad", M, d, C, A_AFF_SILU, 0), (f"{pre} qkv wgrad", "wgrad", M, 2 * d + 8, d, A_GN, H * H),
                (f"{pre} ffn1 wgrad", "wgrad", M, ffn, d, A_GN, H * H), (f"{pre} ffn2 wgrad", "wgrad", M, d, ffn, A_SILU, 0),
                (f"{pre} conv_proj wgrad", "wgrad", M, C, d, A_GN, H * H)]
    return out


def prepass_layers(width):
    """The GEMMs for which ops.pw_gemm / ops.pw_wgrad materialise the prologue first (the WIDE_K / WIDE_N / WIDE_N_WGRAD policy)."""
    from ml_cvnets_b200 import ops as o
    return [g for g in wide_gemms(width)
            if g[5] != o.A_RAW and g[4] >= o.WIDE_K and g[3] >= (o.WIDE_N if g[1] == "fwd" else o.WIDE_N_WGRAD)]


def _gn_rows(M, rps, seed):
    nb = M // rps
    return 0.2 * rnd(nb, seed=seed), 1 + 0.3 * rnd(nb, seed=seed + 1).abs()


# ------------------------------------------------------------------------------------------- linear attention
@pytest.mark.parametrize("width,li,H,d,ffn,C", ATTN)
def test_linattn_at_width(ops, width, li, H, d, ffn, C):
    """linattn_fwd / linattn_bwd at batch 128 against the fp64 unfold / fold restatement: O, S, CTX, dQKV, zero pad columns, dbias"""
    R.test_linattn_bitwise(ops, H, d)


def test_three_warp_rows_are_reached():
    """the configuration does contain attention dims whose rows span three warps in linattn_bwd (256-thread CTAs, d / 8 threads per row)"""
    def pieces(d):
        cgs = d // 8
        return max((g * cgs + cgs - 1) // 32 - (g * cgs) // 32 + 1 for g in range(256 // cgs))
    ds = {st[2] for w in WIDTHS for st in attn_stages(w)}
    assert {d for d in ds if pieces(d) == 3} == {336, 448}
    assert max(pieces(d) for _, _, d, _, _ in attn_stages(1.0)) <= 2


# ------------------------------------------------------------------------------------------- GroupNorm statistics and backward
@pytest.mark.parametrize("width,li,H,d,ffn,C", ATTN)
def test_gn_stats_and_bwd_apply_at_width(ops, width, li, H, d, ffn, C):
    """GroupNorm(1, d) over the H*H rows of each of 128 samples: statistics, and the input gradient with a residual and column sums"""
    rps = H * H
    M = B * rps
    X, G, DR = bf(rnd(M, d, seed=1501) + 0.5), bf(rnd(M, d, seed=1502)), bf(rnd(M, d, seed=1503))
    xs = X.double().view(B, -1)
    gn = torch.stack([xs.mean(1), (xs.var(1, unbiased=False) + 1e-5).rsqrt()]).float()
    xh = (xs - gn[0].double()[:, None]) * gn[1].double()[:, None]
    g = G.double().view(B, -1)
    ss = torch.stack([g.sum(1), (g * xh).sum(1)])

    def run():
        st, cs = zeros64(2, B), zeros64(d)
        ops.gn_stats(X, B, rps, st)
        DX = ops.gn_bwd_apply(G, X, gn, ss, rps * d, B, rps, DRES=DR, col_sum=cs)
        return st, DX, cs

    st, DX, cs = twice(run, ("gn stats", "dX", "col_sum"))
    close_stat(st[0], xs.sum(1), "gn sum")
    close_stat(st[1], (xs * xs).sum(1), "gn sq")
    n = rps * d
    ref = (gn[1].double()[:, None] * (g - ss[0][:, None] / n - xh * ss[1][:, None] / n)).view(M, d) + DR.double()
    close(DX, ref, what="gn dx")
    close_stat(cs, ref.sum(0), "col sum of dx", rtol=5e-3)


# ------------------------------------------------------------------------------------------- attention-unit GEMMs
UNIT_GEMMS = ["qkv", "ffn1", "ffn2", "conv_proj", "gn_bwd_qkv", "gn_bwd_ffn", "gn_bwd_proj", "silu_bwd", "wgrad_qkv", "wgrad_ffn1", "wgrad_proj"]


def _gn_bwd_check(ops, A, W, N, K, X, rps, seed, **kw):
    """E_GN_BWD with the per-sample workspace: g = gamma * (load(A) @ W^T), dgamma / dbeta column sums and the per-sample sums"""
    M = A.shape[0]
    gamma = 1 + 0.2 * rnd(N, seed=seed)
    row = _gn_rows(M, rps, seed + 1)
    nb = M // rps

    def run():
        col, samp = zeros64(2, N), zeros64(2, nb)
        out = ops.pw_gemm(A, W, N, K=K, e_mode=ops.E_GN_BWD, Y=X, e_p=(gamma, None), row_stats=row, rows_per_sample=rps, col_stats=col,
                          samp_stats=samp, gn_ws=zeros64(2, nb, N), **kw)
        return out, col, samp

    out, col, samp = twice(run, ("g", "col_stats", "samp_stats"))
    Af = load_ref(kw.get("a_mode", 0), A, kw.get("a_p", (None, None, None)), kw.get("A2")).double()
    v = Af @ W.double().t()
    xh = (X.double() - row[0].double().repeat_interleave(rps)[:, None]) * row[1].double().repeat_interleave(rps)[:, None]
    close(out, v * gamma.double(), what="g")
    close_stat(col[0], v.sum(0), "dbeta", rtol=5e-3)
    close_stat(col[1], (v * xh).sum(0), "dgamma", rtol=5e-3)
    o = out.double()
    close_stat(samp[0], o.view(nb, -1).sum(1), "sum g", rtol=5e-3)
    close_stat(samp[1], (o * xh).view(nb, -1).sum(1), "sum g*xh", rtol=5e-3)


def _wgrad_check(ops, G, A, N, K, rps, seed, g_mode=0, G2=None, gp=(None, None, None)):
    """dW = load(G)^T @ GN(A), dbias = column sums of load(G)"""
    ap = (1 + 0.2 * rnd(K, seed=seed), 0.3 * rnd(K, seed=seed + 1))
    row = _gn_rows(A.shape[0], rps, seed + 2)

    def run():
        db = torch.zeros(N, device="cuda")
        dW = ops.pw_wgrad(G, A, N, K, g_mode=g_mode, G2=G2, g_p=gp, a_mode=ops.A_GN, a_p=ap, row_stats=row, rows_per_sample=rps, dbias=db)
        return dW, db

    dW, db = twice(run, ("dW", "dbias"))
    Gr = load_ref(g_mode, G, gp, G2).double()
    Ar = load_ref(ops.A_GN, A, ap + (None,), None, row, rps).double()
    ref = Gr.t() @ Ar
    close(dW, ref, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) + 1e-5, what="dW", rel_l2=1e-3)
    close(db, Gr.sum(0), rtol=2e-3, atol=2e-3 * float(Gr.sum(0).abs().max()) + 1e-4, what="dbias", rel_l2=1e-3)


@pytest.mark.parametrize("kind", UNIT_GEMMS)
@pytest.mark.parametrize("width,li,H,d,ffn,C", ATTN)
def test_attention_unit_gemm(ops, width, li, H, d, ffn, C, kind):
    """The pointwise GEMMs of one MobileViTBlockv2 at this width's shapes, with the load modes and epilogues the model gives them."""
    rps = H * H
    M = B * rps
    nq = 2 * d + 8
    X = bf(rnd(M, d, seed=1601) * 1.3 + 0.2)
    if kind in ("qkv", "ffn1", "conv_proj"):
        N = {"qkv": nq, "ffn1": ffn, "conv_proj": C}[kind]
        W = bf(rnd(N, d, scale=d ** -0.5, seed=1602))
        bias = rnd(N, seed=1603) if kind != "conv_proj" else None
        p = (1 + 0.2 * rnd(d, seed=1604), 0.3 * rnd(d, seed=1605), None)
        row = _gn_rows(M, rps, 1606)

        def run():
            col, samp = zeros64(2, N), zeros64(2, B)
            out = ops.pw_gemm(X, W, N, a_mode=ops.A_GN, a_p=p, row_stats=row, rows_per_sample=rps, bias=bias,
                              col_stats=col if kind == "conv_proj" else None, samp_stats=samp if kind == "conv_proj" else None)
            return out, col, samp

        out, col, samp = twice(run, ("out", "col_stats", "samp_stats"))
        ref = load_ref(ops.A_GN, X, p, None, row, rps).double() @ W.double().t() + (bias.double() if bias is not None else 0)
        close(out, ref, what=kind)
        if kind == "conv_proj":
            o = out.double()
            close_stat(col[0], o.sum(0), "col_sum")
            close_stat(col[1], (o * o).sum(0), "col_sq")
    elif kind == "ffn2":
        h = bf(rnd(M, ffn, seed=1611))
        W = bf(rnd(d, ffn, scale=ffn ** -0.5, seed=1612))
        bias = rnd(d, seed=1613)

        def run():
            samp = zeros64(2, B)
            return ops.pw_gemm(h, W, d, a_mode=ops.A_SILU, bias=bias, R=X, samp_stats=samp, rows_per_sample=rps), samp

        out, samp = twice(run, ("out", "samp_stats"))
        ref = load_ref(ops.A_SILU, h).double() @ W.double().t() + bias.double() + X.double()
        close(out, ref, what="ffn2")
        o = out.double()
        close_stat(samp[0], o.view(B, -1).sum(1), "samp_sum")
        close_stat(samp[1], (o * o).view(B, -1).sum(1), "samp_sq")
    elif kind == "gn_bwd_qkv":
        _gn_bwd_check(ops, bf(rnd(M, nq, seed=1621)), bf(rnd(d, nq, scale=nq ** -0.5, seed=1622)), d, nq, X, rps, 1623)
    elif kind == "gn_bwd_ffn":
        _gn_bwd_check(ops, bf(rnd(M, ffn, seed=1631)), bf(rnd(d, ffn, scale=ffn ** -0.5, seed=1632)), d, ffn, X, rps, 1633)
    elif kind == "gn_bwd_proj":
        # conv_proj's input gradient: the BatchNorm backward of its output is the A_BNB load mode of dout
        c = (1 + 0.2 * rnd(C, seed=1641), 0.1 * rnd(C, seed=1642), 0.1 * rnd(C, seed=1643))
        _gn_bwd_check(ops, bf(rnd(M, C, seed=1644)), bf(rnd(d, C, scale=C ** -0.5, seed=1645)), d, C, X, rps, 1646,
                      a_mode=ops.A_BNB, A2=bf(rnd(M, C, seed=1647)), a_p=c)
    elif kind == "silu_bwd":
        dX = bf(rnd(M, d, seed=1651))
        W = bf(rnd(ffn, d, scale=d ** -0.5, seed=1652))
        h = bf(rnd(M, ffn, seed=1653))

        def run():
            col = zeros64(2, ffn)
            return ops.pw_gemm(dX, W, ffn, K=d, e_mode=ops.E_SILU_BWD, Y=h, col_stats=col), col

        out, col = twice(run, ("dh", "col_stats"))
        ref = (dX.double() @ W.double().t()) * dsilu(h.double())
        close(out, ref, what="silu_bwd")
        o = out.double()
        close_stat(col[0], o.sum(0), "sum dh")
        close_stat(col[1], (o * h.double()).sum(0), "sum dh*h")
    elif kind == "wgrad_qkv":
        _wgrad_check(ops, bf(rnd(M, nq, seed=1661)), X, nq, d, rps, 1662)
    elif kind == "wgrad_ffn1":
        _wgrad_check(ops, bf(rnd(M, ffn, seed=1671)), X, ffn, d, rps, 1672)
    elif kind == "wgrad_proj":
        gp = (1 + 0.2 * rnd(C, seed=1681), 0.1 * rnd(C, seed=1682), 0.1 * rnd(C, seed=1683))
        _wgrad_check(ops, bf(rnd(M, C, seed=1684)), X, C, d, rps, 1685, g_mode=ops.A_BNB, G2=bf(rnd(M, C, seed=1686)), gp=gp)


# ------------------------------------------------------------------------------------------- wide-layer pre-pass
PREPASS = [pytest.param(w, g, id=f"w{w}-{g[0].replace(' ', '-')}") for w in WIDTHS for g in prepass_layers(w)]


def test_prepass_fires_at_width_2():
    names = {g[0] for g in prepass_layers(2.0)}
    assert names and {"layer_5.0 exp_1x1", "layer_5.0 exp_1x1 wgrad", "layer_5.1 qkv", "layer_5.1 ffn1", "layer_5.1 conv_proj"} <= names, names
    assert not prepass_layers(1.0)


@pytest.mark.parametrize("width,gemm", PREPASS)
def test_wide_prepass(ops, monkeypatch, width, gemm):
    """Each layer where the policy applies the prologue once by a pre-pass: the pre-pass must run (counted through a wrapper of
    ops.apply_load_mode), and both it and the in-kernel prologue (policy constants raised) must match the fp64 restatement."""
    name, kind, M, N, K, a_mode, rps = gemm
    A, A2 = bf(rnd(M, K, seed=1701)), bf(rnd(M, K, seed=1702))
    p = (1 + 0.2 * rnd(K, seed=1703), 0.3 * rnd(K, seed=1704), 0.1 * rnd(K, seed=1705))
    row = _gn_rows(M, rps, 1706) if a_mode == ops.A_GN else None
    calls = []
    real = ops.apply_load_mode

    def counted(*a, **k):
        calls.append(1)
        return real(*a, **k)

    monkeypatch.setattr(ops, "apply_load_mode", counted)
    if kind == "fwd":
        W = bf(rnd(N, K, scale=K ** -0.5, seed=1707))
        bias = rnd(N, seed=1708)

        def run():
            col = zeros64(2, N)
            out = ops.pw_gemm(A, W, N, a_mode=a_mode, A2=A2 if a_mode == ops.A_BNB else None, a_p=p, row_stats=row, rows_per_sample=rps,
                              bias=bias, col_stats=col)
            return out, col

        ref = load_ref(a_mode, A, p, A2, row, rps).double() @ W.double().t() + bias.double()
    else:
        G = bf(rnd(M, N, seed=1709))

        def run():
            db = torch.zeros(N, device="cuda")
            return ops.pw_wgrad(G, A, N, K, a_mode=a_mode, a_p=p[:2], row_stats=row, rows_per_sample=rps, dbias=db), db

        ref = G.double().t() @ load_ref(a_mode, A, p[:2] + (None,), None, row, rps).double()

    def check(res, what):
        if kind == "fwd":
            close(res[0], ref, what=f"{name} {what}")
            close_stat(res[1][0], res[0].double().sum(0), f"{name} {what} col_sum")
        else:
            close(res[0], ref, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) + 1e-5, what=f"{name} {what} dW", rel_l2=1e-3)
            close(res[1], G.double().sum(0), rtol=2e-3, atol=2e-3 * float(G.double().sum(0).abs().max()) + 1e-4, what=f"{name} dbias", rel_l2=1e-3)

    pre = twice(run, ("out", "stats"))
    ran, err = len(calls), None
    try:
        check(pre, "pre-pass")
    except AssertionError as e:
        err = str(e)
    assert ran == 2 and err is None, f"{name}: the pre-pass ran {ran} times in two calls (want 2); against the reference: {err or 'ok'}"
    monkeypatch.setattr(ops, "WIDE_K", 1 << 30)
    inkernel = twice(run, ("out", "stats"))
    assert len(calls) == 2, f"{name}: the pre-pass ran with the policy off"
    check(inkernel, "in-kernel prologue")


# ------------------------------------------------------------------------------------------- depthwise 3x3
def _dw_layers():
    seen = {(H, C, s) for H, C, s in R.DW_LAYERS}
    out = []
    for w in WIDTHS:
        for pre, H, cin, hid, cout, s, mode in inverted_residuals(w):
            if (H, hid, s) not in seen:
                seen.add((H, hid, s))
                out.append(pytest.param(H, hid, s, 2, id=f"w{w}-{pre}-H{H}-C{hid}-s{s}"))  # input: the expansion's BatchNorm + SiLU, loaded lazily
        for li, H, d, ffn, C in attn_stages(w):
            if (H, C, 1) not in seen:
                seen.add((H, C, 1))
                out.append(pytest.param(H, C, 1, 1, id=f"w{w}-layer_{li}.1-H{H}-C{C}-s1"))  # local_rep: the previous block's BatchNorm, no activation
    return out


DW = _dw_layers()


@pytest.mark.parametrize("H,C,s,x_mode", DW)
def test_dw_fwd_at_width(ops, sms, H, C, s, x_mode):
    B_ = R.dw_batch(R.dw_fwd_grid(H, H, C, s, sms))
    R._check_dw_fwd(ops, B_, H, C, s, 1, x_mode, seed=1800 + H + C)


@pytest.mark.parametrize("H,C,s,x_mode", DW)
def test_dw_bwd_at_width(ops, sms, H, C, s, x_mode):
    B_ = R.dw_batch(R.dw_bwd_grid(H, H, C, s, sms))
    R._check_dw_bwd(ops, B_, H, C, s, 1, 5, x_mode, seed=1900 + H + C)


# ------------------------------------------------------------------------------------------- model level
@pytest.mark.parametrize("width", [str(w) for w in WIDTHS])
def test_model_against_reference_fixture(pkg, golden_dir, width):
    """batch 2 at 128x128, train mode, against the real reference's fp32 record, bounded by the oracle under bf16 autocast"""
    check_model_against_fixture(pkg, load_width_fixture(golden_dir, width))


@pytest.mark.parametrize("width", WIDTHS)
def test_stagewise_parity(pkg, width):
    """every module fed the fp32 oracle's input of its stage, batch 128 at 256x256, train mode: rel-L2 <= 1.5e-2 per stage"""
    rec = stagewise_record(pkg, width)
    torch.cuda.empty_cache()
    print(f"\n[stage-wise parity width {width} B=128 train] " + json.dumps(rec))
    _record(f"stagewise_w{width}_B128", rec)
    assert len(rec) == len(O.mobilevit_v2_layout(width)) + 1
    for k, e in rec.items():
        assert e <= 1.5e-2, (k, e, rec)


@pytest.mark.parametrize("width", WIDTHS)
def test_train_step_parity(pkg, width):
    """batch 16 at 256x256: logits, loss and gradients against the fp32 oracle, no further from it than torch bf16 autocast"""
    rec, sig = train_parity_record(pkg, 16, width)
    torch.cuda.empty_cache()
    print(f"\n[parity width {width} B=16 train] " + json.dumps(rec))
    _record(f"train_w{width}_B16", rec)
    assert rec["logits_rel_l2"] <= 1.15 * rec["autocast_logits_rel_l2"] + 2e-3, rec
    assert abs(rec["loss"] - rec["loss_fp32"]) <= max(2e-3 * abs(rec["loss_fp32"]), 1.5 * abs(rec["loss_autocast"] - rec["loss_fp32"])), rec
    assert rec["grad_rel_l2_all"] <= 1.15 * rec["autocast_grad_rel_l2_all"] + 2e-3, rec
    assert rec["grad_cosine_all"] >= rec["autocast_grad_cosine_all"] - 2e-3, rec
    for t in sig:
        assert t[4] <= 1.5 * t[5] + 2e-2, t


def test_train_step_bitwise_width_2(pkg, ops):
    """MobileViTv2-2.0, batch 16 at 256x256, three AdamW steps: eager twice, without programmatic dependent launch, with the weight
    gradients on the main stream and replayed from a captured graph all end in the same bits.  At this width the wide-layer pre-pass runs
    inside the step, on the side stream and inside the graph."""
    Bt = 16
    xs = [O.seeded_input((Bt, 3, RES, RES), 260 + i).cuda() for i in range(3)]
    ys = [(torch.arange(Bt, device="cuda") * (11 + i)) % 1000 for i in range(3)]
    ref_l, ref_s = R._train(pkg, ops, xs, ys, width=2.0)
    for what, kw in (("eager rerun", {}), ("PDL off", {"pdl": False}), ("side stream off", {"side": False}), ("graph replay", {"graph": True})):
        losses, st = R._train(pkg, ops, xs, ys, width=2.0, **kw)
        for i, (a, b) in enumerate(zip(losses, ref_l)):
            same(a, b, f"{what}: loss of step {i}")
        assert st.keys() == ref_s.keys()
        bad = [k for k in ref_s if not torch.equal(st[k], ref_s[k])]
        assert not bad, f"{what}: {len(bad)} of {len(ref_s)} state tensors differ from the first eager run, e.g. {bad[:6]}"
    assert float(ref_s["step"]) == 3.0

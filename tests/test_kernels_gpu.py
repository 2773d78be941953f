"""Kernel-level parity (-m gpu): C-ABI entry points against a plain PyTorch fp32 restatement of the same op on the
same (bf16-rounded) inputs.  Tolerances are bf16 output rounding (2^-8 relative) plus fp32 accumulation-order noise.
test_kernels_edges_gpu.py covers the remaining entry points and the edge shapes / values; test_kernel_coverage_cpu.py checks that
every export of include/cvnets_b200.h is called by some GPU test."""
import pytest
import torch

pytestmark = pytest.mark.gpu

BF = torch.bfloat16


@pytest.fixture(scope="module")
def ops():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ml_cvnets_b200 import ops as o
    return o


def rnd(*shape, scale=1.0, seed=None):
    g = torch.Generator(device="cuda")
    g.manual_seed(seed if seed is not None else (hash(shape) % 100000))
    return torch.randn(*shape, device="cuda", generator=g) * scale


def bf(x):
    return x.to(BF)


def silu(z):
    return z * torch.sigmoid(z)


def dsilu(z):
    s = torch.sigmoid(z)
    return s * (1 + z * (1 - s))


def load_ref(mode, x, p=(None, None, None), x2=None, row=None, rps=0):
    """fp32 restatement of the operand load modes, including the bf16 rounding of the transformed operand."""
    from ml_cvnets_b200.ops import A_AFF, A_AFF_SILU, A_BNB, A_GN, A_RAW, A_SILU
    x = x.float()
    if mode == A_RAW:
        return x
    if mode == A_AFF:
        y = x * p[0] + p[1]
    elif mode == A_AFF_SILU:
        y = silu(x * p[0] + p[1])
    elif mode == A_SILU:
        y = silu(x)
    elif mode == A_GN:
        mu = row[0].repeat_interleave(rps)[: x.shape[0], None]
        rs = row[1].repeat_interleave(rps)[: x.shape[0], None]
        y = (x - mu) * rs * p[0] + p[1]
    elif mode == A_BNB:
        y = p[0] * x + p[1] * x2.float() + p[2]
    return y.to(BF).float()


def close(a, b, rtol=1.5e-2, atol=None, what="", rel_l2=4e-3):
    """Element-wise bound (bf16 output rounding + accumulation-order noise; the absolute term covers cancellation near zero) AND a
    whole-tensor relative-L2 bound: bf16 rounding of an exact result gives ~1.7e-3, so 4e-3 leaves no room for a systematically wrong
    element class (VERDICT r1: the element-wise clause alone lets values at 10 % of the max be 10 % off)."""
    a, b = a.float(), b.float()
    if atol is None:
        atol = 1e-2 * float(b.abs().max()) + 1e-6
    err = (a - b).abs()
    bad = err > atol + rtol * b.abs()
    assert not bad.any(), f"{what}: {int(bad.sum())}/{bad.numel()} mismatches, max abs err {float(err.max()):.4g}, ref max {float(b.abs().max()):.4g}"
    if rel_l2 is not None and b.numel() > 1:
        r = float((a - b).double().norm() / (b.double().norm() + 1e-30))
        assert r <= rel_l2, f"{what}: rel-L2 {r:.4g} > {rel_l2:.3g}"


def close_stat(a, b, what="", rtol=2e-3):
    a, b = a.double(), b.double()
    scale = float(b.abs().max()) + 1e-12
    err = float((a - b).abs().max())
    assert err <= rtol * scale + 1e-6, f"{what}: max err {err:.4g} vs scale {scale:.4g}"


# ------------------------------------------------------------------------------------------------------------- GEMM fwd
@pytest.mark.parametrize("M,N,K", [(256, 64, 32), (300, 32, 64), (1000, 128, 128), (513, 264, 40), (130, 72, 264), (2048, 384, 192)])
@pytest.mark.parametrize("a_mode", [0, 1, 2, 3, 4, 5])
def test_pw_gemm_modes(ops, M, N, K, a_mode):
    rps = 50
    nb = (M + rps - 1) // rps
    A, A2 = bf(rnd(M, K, seed=1)), bf(rnd(M, K, seed=2))
    W = bf(rnd(N, K, scale=K ** -0.5, seed=3))
    bias = rnd(N, seed=4)
    p = (1 + 0.2 * rnd(K, seed=5), 0.3 * rnd(K, seed=6), 0.1 * rnd(K, seed=7))
    row = (0.2 * rnd(nb, seed=8), 1 + 0.3 * rnd(nb, seed=9).abs())
    R = bf(rnd(M, N, seed=10))
    col = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    samp = torch.zeros(2, nb, device="cuda", dtype=torch.float64)
    out = ops.pw_gemm(A, W, N, a_mode=a_mode, A2=A2 if a_mode == 5 else None, a_p=p, row_stats=row if a_mode == 4 else None,
                      rows_per_sample=rps, bias=bias, R=R, col_stats=col, samp_stats=samp)
    Ar = load_ref(a_mode, A, p, A2, row, rps)
    ref = Ar @ W.float().t() + bias + R.float()
    close(out, ref, what="out")
    o = out.float()
    close_stat(col[0], o.sum(0), "col_sum")
    close_stat(col[1], (o * o).sum(0), "col_sq")
    sid = torch.arange(M, device="cuda") // rps
    ss = torch.zeros(nb, device="cuda").index_add_(0, sid, o.sum(1))
    sq = torch.zeros(nb, device="cuda").index_add_(0, sid, (o * o).sum(1))
    close_stat(samp[0], ss, "samp_sum")
    close_stat(samp[1], sq, "samp_sq")


@pytest.mark.parametrize("M,N,K", [(32, 256, 512), (64, 512, 768), (128, 1000, 512), (40, 128, 1000), (8192, 768, 384)])
@pytest.mark.parametrize("a_mode", [0, 2, 5])
def test_pw_gemm_small_m_large_k(ops, M, N, K, a_mode):
    """late-stage shapes: fewer rows than one tile, weight panels that force narrower N tiles / single-CTA rings"""
    A, A2 = bf(rnd(M, K, seed=201)), bf(rnd(M, K, seed=202))
    W = bf(rnd(N, K, scale=K ** -0.5, seed=203))
    p = (1 + 0.2 * rnd(K, seed=204), 0.3 * rnd(K, seed=205), 0.1 * rnd(K, seed=206))
    col = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    out = ops.pw_gemm(A, W, N, a_mode=a_mode, A2=A2 if a_mode == 5 else None, a_p=p, col_stats=col)
    ref = load_ref(a_mode, A, p, A2) @ W.float().t()
    close(out, ref, what="out")
    close_stat(col[0], out.float().sum(0), "col_sum")


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (256, 64, 64), (1000, 128, 128), (513, 264, 40), (4096, 384, 192), (70000, 128, 64), (33, 1000, 512)])
@pytest.mark.parametrize("epi,a_mode", [("store", 0), ("store_r", 0), ("silu_bwd", 0), ("store", 2), ("store_r", 3), ("store", 4), ("store", 5),
                                         ("silu_bwd", 5), ("store", 1)])
def test_pw_gemm_tcgen05_vs_mma_sync(ops, M, N, K, epi, a_mode):
    """The wgmma kernel and the mma.sync kernel implement the same contract: same inputs -> same outputs / statistics
    (up to fp32 accumulation order), and both match the fp32 restatement."""
    rps = 64
    nb = (M + rps - 1) // rps
    A, A2 = bf(rnd(M, K, seed=301)), bf(rnd(M, K, seed=311))
    pk = (1 + 0.2 * rnd(K, seed=312), 0.3 * rnd(K, seed=313), 0.1 * rnd(K, seed=314))
    row = (0.2 * rnd(nb, seed=315), 1 + 0.3 * rnd(nb, seed=316).abs())
    kwa = dict(a_mode=a_mode, A2=A2 if a_mode == 5 else None, a_p=pk, row_stats=row if a_mode == 4 else None)
    W = bf(rnd(N, K, scale=K ** -0.5, seed=302))
    bias = rnd(N, seed=303)
    aux = bf(rnd(M, N, seed=304))
    sc, sh = 1 + 0.2 * rnd(N, seed=305), 0.3 * rnd(N, seed=306)
    outs = []
    for tc in (True, False):
        prev = ops.set_tc_enabled(tc)
        try:
            col = torch.zeros(2, N, device="cuda", dtype=torch.float64)
            samp = torch.zeros(2, nb, device="cuda", dtype=torch.float64)
            if epi == "store":
                o = ops.pw_gemm(A, W, N, bias=bias, col_stats=col, samp_stats=samp, rows_per_sample=rps, **kwa)
            elif epi == "store_r":
                o = ops.pw_gemm(A, W, N, bias=bias, R=aux, col_stats=col, samp_stats=samp, rows_per_sample=rps, **kwa)
            else:
                o = ops.pw_gemm(A, W, N, e_mode=ops.E_SILU_BWD, Y=aux, e_p=(sc, sh), col_stats=col, rows_per_sample=rps, **kwa)
            torch.cuda.synchronize()
            outs.append((o, col.clone(), samp.clone()))
        finally:
            ops.set_tc_enabled(prev)
    acc = load_ref(a_mode, A, pk, A2, row, rps) @ W.float().t()
    ref = acc + bias if epi == "store" else acc + bias + aux.float() if epi == "store_r" else acc * dsilu(sc * aux.float() + sh)
    for name, (o, col, samp) in zip(("wgmma", "mma.sync"), outs):
        close(o, ref, what=f"{name} out")
        of = o.float()
        close_stat(col[0], of.sum(0), f"{name} col_sum")
        close_stat(col[1], (of * (aux.float() if epi == "silu_bwd" else of)).sum(0), f"{name} col_sq")
    close(outs[0][0], outs[1][0], rtol=1e-2, atol=1e-2 * float(ref.abs().max()), what="wgmma vs mma.sync")
    if epi != "silu_bwd":
        close_stat(outs[0][2][0], outs[1][2][0], "samp_sum tc vs mma")
        close_stat(outs[0][2][1], outs[1][2][1], "samp_sq tc vs mma")


# the shapes bench.py times (SURVEY.md 8a a4-a7 at B = 128): the largest layer of the net and the three qkv projections (N = 2d + 8)
@pytest.mark.parametrize("M,N,K,a_mode", [(2097152, 128, 64, 0), (2097152, 128, 64, 1), (2097152, 64, 32, 2), (524288, 256, 128, 0),
                                           (131072, 264, 128, 4), (32768, 392, 192, 4), (8192, 520, 256, 4), (131072, 128, 264, 0),
                                           (32768, 192, 392, 0), (8192, 256, 520, 0)])
def test_pw_gemm_benched_shapes(ops, M, N, K, a_mode):
    rps = M // 128
    A = bf(rnd(M, K, seed=401))
    W = bf(rnd(N, K, scale=K ** -0.5, seed=402))
    bias = rnd(N, seed=403)
    p = (1 + 0.2 * rnd(K, seed=404), 0.3 * rnd(K, seed=405), None)
    row = (0.2 * rnd(128, seed=406), 1 + 0.3 * rnd(128, seed=407).abs())
    col = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    out = ops.pw_gemm(A, W, N, a_mode=a_mode, a_p=p, row_stats=row if a_mode == 4 else None, rows_per_sample=rps, bias=bias, col_stats=col)
    ref = load_ref(a_mode, A, p, None, row, rps) @ W.float().t() + bias
    close(out, ref, what="out")
    close_stat(col[0], out.float().sum(0), "col_sum")
    close_stat(col[1], (out.float() ** 2).sum(0), "col_sq")


@pytest.mark.parametrize("M,N,K,g_mode,a_mode", [(2097152, 128, 64, 5, 0), (2097152, 64, 64, 5, 2), (524288, 256, 128, 5, 0), (131072, 264, 128, 0, 4),
                                                  (32768, 392, 192, 0, 4), (8192, 520, 256, 0, 4)])
def test_pw_wgrad_benched_shapes(ops, M, N, K, g_mode, a_mode):
    rps = M // 128
    G, G2, A = bf(rnd(M, N, seed=411)), bf(rnd(M, N, seed=412)), bf(rnd(M, K, seed=413))
    gp = (1 + 0.2 * rnd(N, seed=414), 0.3 * rnd(N, seed=415), 0.1 * rnd(N, seed=416))
    ap = (1 + 0.2 * rnd(K, seed=417), 0.3 * rnd(K, seed=418))
    row = (0.2 * rnd(128, seed=419), 1 + 0.3 * rnd(128, seed=420).abs())
    db = torch.zeros(N, device="cuda")
    dW = ops.pw_wgrad(G, A, N, K, g_mode=g_mode, G2=G2 if g_mode == 5 else None, g_p=gp, a_mode=a_mode, a_p=ap,
                      row_stats=row if a_mode == 4 else None, rows_per_sample=rps, dbias=db)
    Gr = load_ref(g_mode, G, gp, G2).double()
    Ar = load_ref(a_mode, A, ap + (None,), None, row, rps).double()
    ref = (Gr.t() @ Ar).float()
    close(dW, ref, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) + 1e-5, what="dW", rel_l2=1e-3)
    close(db, Gr.sum(0).float(), rtol=2e-3, atol=2e-3 * float(Gr.sum(0).abs().max()) + 1e-4, what="dbias", rel_l2=1e-3)


def test_pw_gemm_silu(ops):
    M, N, K = 384, 96, 64
    A, W, bias = bf(rnd(M, K)), bf(rnd(N, K, scale=0.1)), rnd(N)
    out = ops.pw_gemm(A, W, N, bias=bias, e_mode=ops.E_SILU)
    close(out, silu(A.float() @ W.float().t() + bias), what="silu epilogue")


@pytest.mark.parametrize("M,N,K", [(512, 64, 128), (700, 136, 72)])
def test_pw_gemm_silu_bwd(ops, M, N, K):
    A, W = bf(rnd(M, K, seed=11)), bf(rnd(N, K, scale=K ** -0.5, seed=12))
    Y = bf(rnd(M, N, seed=13))
    sc, sh = 1 + 0.2 * rnd(N, seed=14), 0.3 * rnd(N, seed=15)
    col = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    out = ops.pw_gemm(A, W, N, e_mode=ops.E_SILU_BWD, Y=Y, e_p=(sc, sh), col_stats=col)
    ref = (A.float() @ W.float().t()) * dsilu(sc * Y.float() + sh)
    close(out, ref, what="silu_bwd")
    o = out.float()
    close_stat(col[0], o.sum(0), "sum dz")
    close_stat(col[1], (o * Y.float()).sum(0), "sum dz*y")
    # identity scale/shift when e_p is omitted
    out2 = ops.pw_gemm(A, W, N, e_mode=ops.E_SILU_BWD, Y=Y)
    close(out2, (A.float() @ W.float().t()) * dsilu(Y.float()), what="silu_bwd identity")


@pytest.mark.parametrize("M,N,K,rps,ws", [(512, 64, 136, 64, False), (768, 128, 256, 256, False), (160, 16, 40, 16, False),
                                           # with a workspace and rows_per_sample % 64 == 0 the epilogue runs on the wgmma kernel (sum form)
                                           (768, 128, 256, 256, True), (4096, 192, 392, 1024, True), (1280, 256, 520, 128, True), (1344, 256, 512, 64, True)])
@pytest.mark.parametrize("bnb", [False, True])
def test_pw_gemm_gn_bwd(ops, M, N, K, rps, ws, bnb):
    nb = M // rps
    A, W = bf(rnd(M, K, seed=21)), bf(rnd(N, K, scale=K ** -0.5, seed=22))
    X = bf(rnd(M, N, seed=23))
    gamma = 1 + 0.2 * rnd(N, seed=24)
    row = (0.2 * rnd(nb, seed=25), 1 + 0.3 * rnd(nb, seed=26).abs())
    col = torch.zeros(2, N, device="cuda", dtype=torch.float64)
    samp = torch.zeros(2, nb, device="cuda", dtype=torch.float64)
    gn_ws = torch.zeros(2, nb, N, device="cuda", dtype=torch.float64) if ws else None
    kw = {}
    Af = A.float()
    if bnb:
        A2 = bf(rnd(M, K, seed=27))
        c = (1 + 0.2 * rnd(K, seed=28), 0.1 * rnd(K, seed=29), 0.1 * rnd(K, seed=30))
        kw = dict(a_mode=5, A2=A2, a_p=c)
        Af = bf(c[0] * A.float() + c[1] * A2.float() + c[2]).float()
    out = ops.pw_gemm(A, W, N, e_mode=ops.E_GN_BWD, Y=X, e_p=(gamma, None), row_stats=row, rows_per_sample=rps, col_stats=col, samp_stats=samp,
                      gn_ws=gn_ws, **kw)
    v = Af @ W.float().t()
    xh = (X.float() - row[0].repeat_interleave(rps)[:, None]) * row[1].repeat_interleave(rps)[:, None]
    close(out, v * gamma, what="g")
    close_stat(col[0], v.sum(0), "dbeta", rtol=5e-3)
    close_stat(col[1], (v * xh).sum(0), "dgamma", rtol=5e-3)
    o = out.float()
    close_stat(samp[0], o.view(nb, -1).sum(1), "sum g", rtol=5e-3)
    close_stat(samp[1], (o * xh).view(nb, -1).sum(1), "sum g*xh", rtol=5e-3)


# ----------------------------------------------------------------------------------------------------------- GEMM wgrad
# K % 64 == 0 shapes run on the wgmma kernel (wgrad_tc.cu: MN-major operands, dW block in registers), the others on mma.sync
@pytest.mark.parametrize("M,N,K", [(1000, 64, 32), (4096, 128, 64), (777, 264, 40), (300, 72, 200), (5000, 192, 192), (3001, 264, 128),
                                   (2500, 64, 384), (20000, 256, 256), (700, 512, 768), (64, 128, 64)])
@pytest.mark.parametrize("g_mode,a_mode", [(0, 0), (5, 0), (5, 2), (0, 3), (0, 4), (5, 4), (0, 1)])
def test_pw_wgrad(ops, M, N, K, g_mode, a_mode):
    rps = 100
    nb = (M + rps - 1) // rps
    G, G2, A = bf(rnd(M, N, seed=31)), bf(rnd(M, N, seed=32)), bf(rnd(M, K, seed=33))
    gp = (1 + 0.2 * rnd(N, seed=34), 0.3 * rnd(N, seed=35), 0.1 * rnd(N, seed=36))
    ap = (1 + 0.2 * rnd(K, seed=37), 0.3 * rnd(K, seed=38))
    row = (0.2 * rnd(nb, seed=39), 1 + 0.3 * rnd(nb, seed=40).abs())
    db = torch.zeros(N, device="cuda")
    dW = ops.pw_wgrad(G, A, N, K, g_mode=g_mode, G2=G2 if g_mode == 5 else None, g_p=gp, a_mode=a_mode, a_p=ap,
                      row_stats=row if a_mode == 4 else None, rows_per_sample=rps, dbias=db)
    Gr = load_ref(g_mode, G, gp, G2)
    Ar = load_ref(a_mode, A, ap + (None,), None, row, rps)
    ref = Gr.t() @ Ar
    close(dW, ref, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) + 1e-5, what="dW")
    close(db, Gr.sum(0), rtol=2e-3, atol=2e-3 * float(Gr.sum(0).abs().max()) + 1e-4, what="dbias")


@pytest.mark.parametrize("M,N,K", [(9000, 128, 256), (4097, 392, 192)])
@pytest.mark.parametrize("g_mode,a_mode", [(0, 0), (5, 2), (0, 4)])
def test_pw_wgrad_tcgen05_vs_mma_sync(ops, M, N, K, g_mode, a_mode):
    """Both weight-gradient kernels on identical inputs (they round the transformed operands identically: differences are fp32 summation order)."""
    rps = 128
    nb = (M + rps - 1) // rps
    G, G2, A = bf(rnd(M, N, seed=51)), bf(rnd(M, N, seed=52)), bf(rnd(M, K, seed=53))
    gp = (1 + 0.2 * rnd(N, seed=54), 0.3 * rnd(N, seed=55), 0.1 * rnd(N, seed=56))
    ap = (1 + 0.2 * rnd(K, seed=57), 0.3 * rnd(K, seed=58))
    row = (0.2 * rnd(nb, seed=59), 1 + 0.3 * rnd(nb, seed=60).abs())
    outs = []
    for tc in (True, False):
        prev = ops.set_tc_enabled(tc)
        try:
            db = torch.zeros(N, device="cuda")
            dW = ops.pw_wgrad(G, A, N, K, g_mode=g_mode, G2=G2 if g_mode == 5 else None, g_p=gp, a_mode=a_mode, a_p=ap,
                              row_stats=row if a_mode == 4 else None, rows_per_sample=rps, dbias=db)
            outs.append((dW.clone(), db.clone()))
        finally:
            ops.set_tc_enabled(prev)
    scale = float(outs[1][0].abs().max())
    assert float((outs[0][0] - outs[1][0]).abs().max()) <= 2e-4 * scale + 1e-5
    assert float((outs[0][1] - outs[1][1]).abs().max()) <= 2e-4 * float(outs[1][1].abs().max()) + 1e-4


# ------------------------------------------------------------------------------------------------------------ depthwise
def _dw_ref(x_nhwc, B, H, W, C, stride, w, mode, p):
    xa = load_ref(mode, x_nhwc, p + (None,)).view(B, H, W, C).permute(0, 3, 1, 2)
    return torch.nn.functional.conv2d(xa, w, None, stride=stride, padding=1, groups=C), xa


@pytest.mark.parametrize("B,H,W,C,stride", [(2, 16, 16, 64, 1), (3, 20, 12, 32, 1), (2, 32, 32, 128, 2), (2, 8, 8, 72, 2), (1, 4, 4, 8, 1), (2, 36, 36, 64, 2)])
@pytest.mark.parametrize("x_mode", [0, 1, 2])
def test_dw_fwd(ops, B, H, W, C, stride, x_mode):
    X = bf(rnd(B * H * W, C, seed=41))
    w = bf(rnd(C, 1, 3, 3, scale=0.3, seed=42)).float()
    p = (1 + 0.2 * rnd(C, seed=43), 0.3 * rnd(C, seed=44))
    Wt = w.view(C, 9).t().contiguous()
    col = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    Y = ops.dw_fwd(X, B, H, W, C, stride, Wt, x_mode=x_mode, x_p=p, col_stats=col)
    ref, _ = _dw_ref(X, B, H, W, C, stride, w, x_mode, p)
    ref2 = ref.permute(0, 2, 3, 1).reshape(-1, C)
    close(Y, ref2, what="dw fwd")
    o = Y.float()
    close_stat(col[0], o.sum(0), "col_sum")
    close_stat(col[1], (o * o).sum(0), "col_sq")


@pytest.mark.parametrize("B,H,W,C,stride", [(2, 16, 16, 64, 1), (3, 20, 12, 32, 1), (2, 32, 32, 128, 2), (2, 8, 8, 72, 2), (5, 4, 4, 8, 1), (2, 36, 36, 64, 2)])
@pytest.mark.parametrize("g_mode,x_mode", [(0, 0), (5, 2), (5, 0), (0, 2), (5, 1)])
def test_dw_bwd(ops, B, H, W, C, stride, g_mode, x_mode):
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    X = bf(rnd(B * H * W, C, seed=51))
    DZ, Y2 = bf(rnd(B * Ho * Wo, C, seed=52)), bf(rnd(B * Ho * Wo, C, seed=53))
    w = bf(rnd(C, 1, 3, 3, scale=0.3, seed=54)).float()
    gp = (1 + 0.2 * rnd(C, seed=55), 0.3 * rnd(C, seed=56), 0.1 * rnd(C, seed=57))
    xp = (1 + 0.2 * rnd(C, seed=58), 0.3 * rnd(C, seed=59))
    Wt = w.view(C, 9).t().contiguous()
    col = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    DX, dWt = ops.dw_bwd(DZ, X, B, H, W, C, stride, Wt, g_mode=g_mode, Y2=Y2 if g_mode == 5 else None, g_p=gp, x_mode=x_mode, x_p=xp,
                         col_stats=col if x_mode != 0 else None)
    dy = load_ref(g_mode, DZ, gp, Y2).view(B, Ho, Wo, C).permute(0, 3, 1, 2)
    xa = load_ref(x_mode, X, xp + (None,)).view(B, H, W, C).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    wv = w.clone().requires_grad_(True)
    y = torch.nn.functional.conv2d(xa, wv, None, stride=stride, padding=1, groups=C)
    y.backward(dy)
    da = xa.grad.permute(0, 2, 3, 1).reshape(-1, C)
    if x_mode == 2:
        da = da * dsilu(xp[0] * X.float() + xp[1])
    close(DX, da, what="dX")
    close(dWt, wv.grad.view(C, 9).t(), rtol=3e-3, atol=3e-3 * float(wv.grad.abs().max()) + 1e-5, what="dW")
    if x_mode != 0:
        # interior tiles accumulate the statistics from the fp32 values (before the bf16 rounding of the store), edge tiles from the stored
        # values: the truth is the fp32 sum; a zero-mean sum of n rounded values differs from it by ~2^-9 / sqrt(3) of its own size (measured:
        # up to 3.1e-3 of the largest channel sum on these small cases)
        close_stat(col[0], da.sum(0), "sum dz", rtol=6e-3)
        close_stat(col[1], (da * X.float()).sum(0), "sum dz*x", rtol=6e-3)


@pytest.mark.parametrize("B,H,W,C,dil", [(2, 16, 16, 64, 2), (3, 12, 20, 48, 2), (2, 16, 16, 384, 4), (2, 8, 8, 72, 4), (1, 5, 7, 8, 3)])
@pytest.mark.parametrize("x_mode", [0, 1, 2])
def test_dw_fwd_dilated(ops, B, H, W, C, dil, x_mode):
    """Dilated depthwise conv (segmentation backbones, output_stride 8 / 16): pad = dilation, stride 1."""
    X = bf(rnd(B * H * W, C, seed=41))
    w = bf(rnd(C, 1, 3, 3, scale=0.3, seed=42)).float()
    p = (1 + 0.2 * rnd(C, seed=43), 0.3 * rnd(C, seed=44))
    Wt = w.view(C, 9).t().contiguous()
    col = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    Y = ops.dw_fwd(X, B, H, W, C, 1, Wt, x_mode=x_mode, x_p=p, col_stats=col, dilation=dil)
    xa = load_ref(x_mode, X, p + (None,)).view(B, H, W, C).permute(0, 3, 1, 2)
    ref = torch.nn.functional.conv2d(xa, w, None, stride=1, padding=dil, dilation=dil, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    close(Y, ref, what="dilated dw fwd")
    o = Y.float()
    close_stat(col[0], o.sum(0), "col_sum")
    close_stat(col[1], (o * o).sum(0), "col_sq")


@pytest.mark.parametrize("B,H,W,C,dil", [(2, 16, 16, 64, 2), (3, 12, 20, 48, 2), (2, 16, 16, 384, 4), (1, 5, 7, 8, 3)])
@pytest.mark.parametrize("g_mode,x_mode", [(0, 0), (5, 2), (5, 0), (0, 2), (5, 1)])
def test_dw_bwd_dilated(ops, B, H, W, C, dil, g_mode, x_mode):
    X = bf(rnd(B * H * W, C, seed=51))
    DZ, Y2 = bf(rnd(B * H * W, C, seed=52)), bf(rnd(B * H * W, C, seed=53))
    w = bf(rnd(C, 1, 3, 3, scale=0.3, seed=54)).float()
    gp = (1 + 0.2 * rnd(C, seed=55), 0.3 * rnd(C, seed=56), 0.1 * rnd(C, seed=57))
    xp = (1 + 0.2 * rnd(C, seed=58), 0.3 * rnd(C, seed=59))
    Wt = w.view(C, 9).t().contiguous()
    col = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    DX, dWt = ops.dw_bwd(DZ, X, B, H, W, C, 1, Wt, g_mode=g_mode, Y2=Y2 if g_mode == 5 else None, g_p=gp, x_mode=x_mode, x_p=xp,
                         col_stats=col if x_mode != 0 else None, dilation=dil)
    dy = load_ref(g_mode, DZ, gp, Y2).view(B, H, W, C).permute(0, 3, 1, 2)
    xa = load_ref(x_mode, X, xp + (None,)).view(B, H, W, C).permute(0, 3, 1, 2).contiguous().requires_grad_(True)
    wv = w.clone().requires_grad_(True)
    torch.nn.functional.conv2d(xa, wv, None, stride=1, padding=dil, dilation=dil, groups=C).backward(dy)
    da = xa.grad.permute(0, 2, 3, 1).reshape(-1, C)
    if x_mode == 2:
        da = da * dsilu(xp[0] * X.float() + xp[1])
    close(DX, da, what="dilated dX")
    close(dWt, wv.grad.view(C, 9).t(), rtol=3e-3, atol=3e-3 * float(wv.grad.abs().max()) + 1e-5, what="dilated dW")
    if x_mode != 0:
        o = DX.float()
        close_stat(col[0], o.sum(0), "sum dz")
        close_stat(col[1], (o * X.float()).sum(0), "sum dz*x")


# ----------------------------------------------------------------------------------------------------------- BN / GN / misc
def test_bn_finalize_and_bwd_finalize(ops):
    C, M = 96, 5000
    y = bf(rnd(M, C, seed=61) * 1.5 + 0.3).float()
    stats = torch.stack([y.sum(0), (y * y).sum(0)]).double()
    gamma, beta = 1 + 0.2 * rnd(C, seed=62), 0.1 * rnd(C, seed=63)
    rm, rv = torch.zeros(C, device="cuda"), torch.ones(C, device="cuda")
    nbt = torch.zeros((), device="cuda", dtype=torch.long)
    bn = ops.bn_finalize(stats, M, gamma, beta, 1e-5, 0.1, rm, rv, nbt)
    mean, var = y.mean(0), y.var(0, unbiased=False)
    close(bn[0], mean, rtol=1e-4, atol=1e-5, what="mean")
    close(bn[1], (var + 1e-5).rsqrt(), rtol=1e-4, atol=1e-5, what="rstd")
    close(bn[2], gamma * (var + 1e-5).rsqrt(), rtol=1e-4, atol=1e-5, what="scale")
    close(bn[3], beta - mean * gamma * (var + 1e-5).rsqrt(), rtol=1e-4, atol=1e-4, what="shift")
    close(rm, 0.1 * mean, rtol=1e-4, atol=1e-5, what="running_mean")
    close(rv, 0.9 + 0.1 * y.var(0, unbiased=True), rtol=1e-4, atol=1e-5, what="running_var")
    assert int(nbt) == 1
    # backward coefficients against autograd of batch_norm
    yv = y.clone().requires_grad_(True)
    g = gamma.clone().requires_grad_(True)
    b = beta.clone().requires_grad_(True)
    out = torch.nn.functional.batch_norm(yv, None, None, g, b, True, 0.1, 1e-5)
    dz = rnd(M, C, seed=64)
    out.backward(dz)
    sd = torch.stack([dz.sum(0), (dz * y).sum(0)]).double()
    dgb, coef = ops.bn_bwd_finalize(sd, M, gamma, bn)
    close(dgb[0], g.grad, rtol=2e-3, atol=2e-3 * float(g.grad.abs().max()), what="dgamma")
    close(dgb[1], b.grad, rtol=2e-3, atol=2e-3 * float(b.grad.abs().max()), what="dbeta")
    dy = coef[0] * dz + coef[1] * y + coef[2]
    close(dy, yv.grad, rtol=2e-3, atol=2e-3 * float(yv.grad.abs().max()), what="dy")
    ev = ops.bn_eval_scale_shift(gamma, beta, rm, rv, 1e-5)
    close(ev[2], gamma * (rv + 1e-5).rsqrt(), rtol=1e-5, atol=1e-6, what="eval scale")


@pytest.mark.parametrize("M,C", [(1000, 64), (333, 96), (4096, 768), (50, 8)])
def test_bn_apply_and_bwd_reduce(ops, M, C):
    Y, R, D = bf(rnd(M, C, seed=71)), bf(rnd(M, C, seed=72)), bf(rnd(M, C, seed=73))
    bn = torch.stack([rnd(C), rnd(C).abs() + 0.5, 1 + 0.2 * rnd(C, seed=74), 0.3 * rnd(C, seed=75)])
    close(ops.bn_apply(Y, bn, False, R), Y.float() * bn[2] + bn[3] + R.float(), what="bn_apply")
    close(ops.bn_apply(Y, bn, True), silu(Y.float() * bn[2] + bn[3]), what="bn_apply silu")
    st = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    assert ops.bn_bwd_reduce(D, Y, st) is None
    close_stat(st[0], D.float().sum(0), "sum dz")
    close_stat(st[1], (D.float() * Y.float()).sum(0), "sum dz*y")
    st.zero_()
    dz = ops.bn_bwd_reduce(D, Y, st, bn, act=True, store_dz=True)
    ref = D.float() * dsilu(Y.float() * bn[2] + bn[3])
    close(dz, ref, what="dz")
    close_stat(st[0], dz.float().sum(0), "sum dz (act)")
    close_stat(st[1], (dz.float() * Y.float()).sum(0), "sum dz*y (act)")


@pytest.mark.parametrize("B,rps,C", [(4, 64, 128), (3, 100, 24), (8, 16, 256)])
def test_gn_kernels(ops, B, rps, C):
    M = B * rps
    X, G, DR = bf(rnd(M, C, seed=81) + 0.5), bf(rnd(M, C, seed=82)), bf(rnd(M, C, seed=83))
    st = torch.zeros(2, B, device="cuda", dtype=torch.float64)
    ops.gn_stats(X, B, rps, st)
    xf = X.float().view(B, -1)
    close_stat(st[0], xf.sum(1), "gn sum")
    close_stat(st[1], (xf * xf).sum(1), "gn sq")
    gn = ops.gn_finalize(st, rps * C, 1e-5)
    close(gn[0], xf.mean(1), rtol=1e-4, atol=1e-5, what="gn mean")
    close(gn[1], (xf.var(1, unbiased=False) + 1e-5).rsqrt(), rtol=1e-4, atol=1e-5, what="gn rstd")
    # backward phase 2 against autograd of group_norm (gamma folded into g by the caller)
    xv = X.float().view(B, rps, C).permute(0, 2, 1).contiguous().requires_grad_(True)  # [B, C, rps]
    out = torch.nn.functional.group_norm(xv, 1, None, None, 1e-5)
    gg = G.float().view(B, rps, C).permute(0, 2, 1)
    out.backward(gg)
    xh = ((X.float().view(B, -1) - gn[0][:, None]) * gn[1][:, None]).view(M, C)
    ss = torch.stack([G.float().view(B, -1).sum(1), (G.float() * xh).view(B, -1).sum(1)]).double()
    cs = torch.zeros(C, device="cuda", dtype=torch.float64)
    DX = ops.gn_bwd_apply(G, X, gn, ss, rps * C, B, rps, DRES=DR, col_sum=cs)
    ref = xv.grad.permute(0, 2, 1).reshape(M, C) + DR.float()
    close(DX, ref, what="gn dx")
    close_stat(cs, ref.sum(0), "col sum of dx", rtol=5e-3)


@pytest.mark.parametrize("B,H,W,d", [(2, 8, 8, 16), (3, 16, 16, 128), (2, 8, 8, 192), (2, 4, 4, 256), (1, 32, 32, 128)])
def test_linattn(ops, B, H, W, d):
    ldq = 2 * d + 8
    M = B * H * W
    QKV = bf(rnd(M, ldq, seed=91))
    DO = bf(rnd(M, d, seed=92))
    O, S, CTX = ops.linattn_fwd(QKV, B, H, W, d)
    # reference through the ORIGINAL formulation: unfold -> [B, c, 4, N]
    q4 = QKV.float().view(B, H, W, ldq).permute(0, 3, 1, 2)

    def unfold(t):
        Bc, C = t.shape[:2]
        return torch.nn.functional.unfold(t, kernel_size=2, stride=2).reshape(Bc, C, 4, -1)

    def fold(p):
        Bc, C, P, N = p.shape
        return torch.nn.functional.fold(p.reshape(Bc, C * P, N), output_size=(H, W), kernel_size=2, stride=2)

    k = unfold(q4[:, :d]).requires_grad_(True)
    v = unfold(q4[:, d:2 * d]).requires_grad_(True)
    q = unfold(q4[:, 2 * d:2 * d + 1]).requires_grad_(True)
    s = torch.softmax(q, dim=-1)
    ctx = (k * s).sum(-1, keepdim=True)
    out = torch.relu(v) * ctx
    ref_O = fold(out).permute(0, 2, 3, 1).reshape(M, d)
    close(O, ref_O, what="O")
    close(CTX, ctx.squeeze(-1).permute(0, 2, 1), rtol=2e-3, atol=1e-4, what="ctx")
    close(S, s.squeeze(1), rtol=2e-3, atol=1e-5, what="scores")
    dOu = unfold(DO.float().view(B, H, W, d).permute(0, 3, 1, 2))
    out.backward(dOu)
    db = torch.zeros(ldq, device="cuda")
    DQKV = ops.linattn_bwd(QKV, DO, S, CTX, B, H, W, d, dbias=db)
    ref = torch.zeros(M, ldq, device="cuda")
    ref[:, :d] = fold(k.grad).permute(0, 2, 3, 1).reshape(M, d)
    ref[:, d:2 * d] = fold(v.grad).permute(0, 2, 3, 1).reshape(M, d)
    ref[:, 2 * d] = fold(q.grad).permute(0, 2, 3, 1).reshape(M)
    close(DQKV[:, :2 * d], ref[:, :2 * d], what="dK,dV")
    close(DQKV[:, 2 * d], ref[:, 2 * d], rtol=3e-2, atol=2e-2 * float(ref[:, 2 * d].abs().max()) + 1e-6, what="dq")
    assert float(DQKV[:, 2 * d + 1:].float().abs().max()) == 0.0
    close(db[:2 * d], DQKV[:, :2 * d].float().sum(0), rtol=2e-3, atol=2e-3 * float(db.abs().max()) + 1e-5, what="dbias")


def test_pool_im2col_prep(ops):
    B, HW, C = 5, 64, 96
    X = bf(rnd(B * HW, C, seed=101))
    p = ops.global_pool_fwd(X, B, HW)
    close(p, X.float().view(B, HW, C).mean(1), what="pool fwd")
    dx = ops.global_pool_bwd(p, B, HW)
    close(dx, (p.float() / HW)[:, None, :].expand(B, HW, C).reshape(-1, C), what="pool bwd")
    # stem im2col, NCHW and channels_last images
    img = rnd(2, 3, 16, 20, seed=103)
    for im in (img, img.contiguous(memory_format=torch.channels_last)):
        A = ops.stem_im2col(im)
        ref = torch.nn.functional.unfold(im.to(BF).float(), kernel_size=3, stride=2, padding=1)  # [B, 27, L]
        ref = ref.permute(0, 2, 1).reshape(-1, 27)
        close(A[:, :27], ref, rtol=0, atol=0, what="im2col")
        assert float(A[:, 27:].float().abs().max()) == 0.0
    # weight preparation
    d = 16
    w = torch.nn.Parameter(rnd(2 * d + 1, d, 1, 1, seed=104))
    bvec = torch.nn.Parameter(rnd(2 * d + 1, seed=105))
    wd = torch.nn.Parameter(rnd(24, 1, 3, 3, seed=106))
    P = ops.PreparedWeights()
    i0 = P.add(w, P.KIND_ROWMAJOR, rot=1, dst_rows=2 * d + 8)
    i1 = P.add(w, P.KIND_TRANSPOSED, rot=1, ldd=2 * d + 8)
    i2 = P.add(bvec, P.KIND_VECTOR_F32, rot=1, dst_rows=2 * d + 8)
    i3 = P.add(wd, P.KIND_TAPMAJOR_F32)
    P.prepare()
    w2 = w.detach().view(2 * d + 1, d)
    perm = torch.cat([w2[1:], w2[:1]])
    assert torch.equal(P.get(i0)[: 2 * d + 1], perm.to(BF)) and float(P.get(i0)[2 * d + 1:].float().abs().max()) == 0
    assert torch.equal(P.get(i1)[:, : 2 * d + 1], perm.t().to(BF)) and float(P.get(i1)[:, 2 * d + 1:].float().abs().max()) == 0
    assert torch.equal(P.get(i2)[: 2 * d + 1], torch.cat([bvec.detach()[1:], bvec.detach()[:1]]))
    assert torch.equal(P.get(i3), wd.detach().view(24, 9).t().to(BF).float())
    g = rnd(2 * d + 8, d, seed=107)
    back = ops.unprep_grad(g, 2 * d + 1, d, d, 0, rot=1)
    assert torch.equal(back[1:], g[: 2 * d]) and torch.equal(back[0], g[2 * d])
    gt = rnd(9, 24, seed=108)
    assert torch.equal(ops.unprep_grad(gt, 24, 9, 24, 2), gt.t())


# ------------------------------------------------------------------------------------------------- multi-head attention
def _mha_ref(qkv, B, S, H, c, scale, amask, kpm):
    """fp32 restatement of cvnets/layers/multi_head_attention.py:148-235 on the packed projection."""
    x = qkv.float().view(B, S, 3, H, c).permute(2, 0, 3, 1, 4)  # [3, B, H, S, c]
    q, k, v = x[0] * scale, x[1], x[2]
    att = q @ k.transpose(-1, -2)
    if amask is not None:
        att = att + amask[:, None]
    if kpm is not None:
        att = att.masked_fill(kpm[:, None, None, :].bool(), float("-inf"))
    att = torch.softmax(att, dim=-1)
    return (att @ v).transpose(1, 2).reshape(B * S, H * c)


@pytest.mark.parametrize("B,S,H,c", [(2, 197, 12, 64), (3, 77, 8, 64), (2, 256, 4, 16), (2, 64, 4, 32), (5, 16, 2, 16), (1, 130, 3, 32),
                                      (1, 16, 1, 64), (2, 128, 2, 64), (1, 129, 1, 64), (2, 256, 2, 64)])
@pytest.mark.parametrize("mask", ["none", "causal", "padding"])
def test_mha_fwd_bwd(ops, B, S, H, c, mask):
    C = H * c
    qkv = bf(rnd(B * S, 3 * C, seed=71))
    dO = bf(rnd(B * S, C, seed=72))
    amask = kpm = None
    if mask == "causal":
        amask = torch.full((S, S), float("-inf"), device="cuda").triu(1)[None].repeat(B, 1, 1).contiguous()
    if mask == "padding":
        kpm = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
        kpm[:, S - max(1, S // 5):] = 1
    scale = c ** -0.5
    O, LSE = ops.mha_fwd(qkv, B, S, H, c, scale, attn_mask=amask, key_padding_mask=kpm)
    x = qkv.float().requires_grad_(True)
    ref = _mha_ref(x, B, S, H, c, scale, amask, kpm)
    close(O, ref.detach(), what="mha fwd")
    ref.backward(dO.float())
    DQKV = ops.mha_bwd(qkv, O, dO, LSE, B, S, H, c, scale, attn_mask=amask, key_padding_mask=kpm)
    close(DQKV, x.grad, rtol=3e-2, atol=2e-2 * float(x.grad.abs().max()) + 1e-6, what="mha bwd")


@pytest.mark.parametrize("B,S,H", [(2, 197, 3), (2, 77, 2), (1, 250, 2)])
@pytest.mark.parametrize("mask", ["none", "padding"])
def test_mha_tc_matches_mma(ops, B, S, H, mask):
    """head_dim 64, S <= 256 without an additive mask has two implementations: wgmma (mha_tc.cu, the default) and mma.sync (mha.cu, test
    mode 1).  Same inputs -> same O / LSE / dQKV up to the bf16 rounding of P (the tensor-core operand) and the accumulation order."""
    from ml_cvnets_b200 import _lib as L
    lib = L.load()
    C = H * 64
    qkv = bf(rnd(B * S, 3 * C, seed=73))
    dO = bf(rnd(B * S, C, seed=74))
    kpm = None
    if mask == "padding":
        kpm = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
        kpm[:, S - max(1, S // 5):] = 1
    res = {}
    old = lib.cvb_set_mha_impl(0)
    try:
        for name, m in (("mma", 1), ("tc", 0)):
            lib.cvb_set_mha_impl(m)
            O, LSE = ops.mha_fwd(qkv, B, S, H, 64, 0.125, key_padding_mask=kpm)
            D = ops.mha_bwd(qkv, O, dO, LSE, B, S, H, 64, 0.125, key_padding_mask=kpm)
            res[name] = (O.float(), LSE.clone(), D.float())
    finally:
        lib.cvb_set_mha_impl(old)
    for i, what in enumerate(("O", "LSE", "dQKV")):
        a, b = res["tc"][i].double(), res["mma"][i].double()
        r = float((a - b).norm() / (b.norm() + 1e-30))
        assert r <= 4e-3, f"{what}: wgmma vs mma.sync rel-L2 {r:.3g}"


@pytest.mark.parametrize("M,K", [(1000, 768), (333, 64), (70, 3072)])
@pytest.mark.parametrize("a_mode", [1, 2, 3, 4, 5])
def test_apply_load_mode_prepass(ops, M, K, a_mode):
    """The wide-layer pre-pass (ops.WIDE_K / WIDE_N policy): OUT = load(A) materialised once, against the fp32 restatement of every load mode."""
    rps = 50
    nb = (M + rps - 1) // rps
    A, A2 = bf(rnd(M, K, seed=11)), bf(rnd(M, K, seed=12))
    p = (rnd(K, seed=13) * 0.5 + 1.0, rnd(K, seed=14) * 0.3, rnd(K, seed=15) * 0.2)
    row = (rnd(nb, seed=16) * 0.1, rnd(nb, seed=17).abs() + 0.5)
    out = ops.apply_load_mode(A, a_mode, K, A2=A2 if a_mode == 5 else None, a_p=p, row_stats=row if a_mode == 4 else None,
                              rows_per_sample=rps if a_mode == 4 else 0)
    ref = load_ref(a_mode, A, p, x2=A2, row=row, rps=rps)
    close(out, ref, what=f"apply_load_mode mode {a_mode}")


# ------------------------------------------------------------------------------------------ dropout / stochastic depth
def test_dropout_kernels(ops):
    """Hashed-mask dropout (csrc/dropout.cu): keep rate, scaling, residual add, key determinism, backward == forward mask, per-sample rows."""
    M, C, rps = 4000, 256, 40
    V = bf(rnd(M, C, seed=91))
    R = bf(rnd(M, C, seed=92))
    ones = torch.ones(M, C, device="cuda", dtype=BF)
    ops.rng_seed(1234)
    k1, k2 = ops.rng_next("cuda"), ops.rng_next("cuda")
    assert int(k1) != int(k2)
    ops.rng_seed(1234)
    assert int(ops.rng_next("cuda")) == int(k1) and int(ops.rng_next("cuda")) == int(k2)  # same seed -> same key sequence
    for p in (0.1, 0.5):
        m1 = ops.dropout_fwd(ones, None, p, k1).float()
        keep = float((m1 != 0).float().mean())
        sigma = (p * (1 - p) / (M * C)) ** 0.5
        assert abs(keep - (1 - p)) <= 5 * sigma + 2e-5, (p, keep)
        scale = float(torch.tensor(1.0 / (1 - p)).to(BF))
        assert torch.all((m1 == 0) | ((m1 - scale).abs() < 1e-6))
        assert torch.equal(m1, ops.dropout_fwd(ones, None, p, k1).float())          # deterministic in the key
        assert not torch.equal(m1, ops.dropout_fwd(ones, None, p, k2).float())      # a new key draws a new mask
        assert torch.equal(m1, ops.dropout_bwd(ones, p, k1).float())                # the backward regenerates the forward's mask
        Y = ops.dropout_fwd(V, R, p, k1).float()
        ref = R.float() + V.float() * (m1 != 0) / (1 - p)
        assert float((Y - ref).norm() / ref.norm()) <= 4e-3
        # columns are dropped independently of rows: no structure along either axis
        assert abs(float((m1 != 0).float().mean(0).std()) - ((p * (1 - p) / M) ** 0.5)) < 3e-3
    # stochastic depth: one Bernoulli per sample (rps rows), scaled by 1 / keep
    pr = 0.3
    mr = ops.dropout_fwd(ones, None, 0.0, k1, p_row=pr, rows_per_sample=rps).float().view(M // rps, rps * C)
    assert torch.all((mr == mr[:, :1]))
    vals = mr[:, 0]
    assert torch.all((vals == 0) | ((vals - float(torch.tensor(1 / (1 - pr)).to(BF))).abs() < 1e-6))
    assert 0.5 < float((vals != 0).float().mean()) < 0.9
    both = ops.dropout_fwd(ones, None, 0.2, k1, p_row=pr, rows_per_sample=rps).float().view(M // rps, rps * C)
    assert torch.all(both[vals == 0] == 0) and float((both[vals != 0] != 0).float().mean()) > 0.7
    assert torch.equal(ops.dropout_bwd(ones, 0.2, k1, p_row=pr, rows_per_sample=rps).float().view(M // rps, rps * C), both)


@pytest.mark.parametrize("M,C", [(1000, 768), (333, 64), (50, 1000)])
def test_ln_stats(ops, M, C):
    X = bf(rnd(M, C, seed=81) * 2 + 0.5)
    st = ops.ln_stats(X, 1e-5)
    xf = X.float()
    assert float((st[0] - xf.mean(1)).abs().max()) < 1e-4
    rstd = 1.0 / torch.sqrt(xf.var(1, unbiased=False) + 1e-5)
    assert float(((st[1] - rstd) / rstd).abs().max()) < 1e-3


@pytest.mark.parametrize("M,C", [(500, 768), (77, 64), (1000, 1024)])
@pytest.mark.parametrize("res", [False, True])
def test_ln_bwd(ops, M, C, res):
    X = bf(rnd(M, C, seed=91) * 1.5 + 0.3)
    V = bf(rnd(M, C, seed=92))
    R = bf(rnd(M, C, seed=93)) if res else None
    gamma = 1 + 0.2 * rnd(C, seed=94)
    beta = 0.1 * rnd(C, seed=95)
    ln = ops.ln_stats(X, 1e-5)
    col = torch.zeros(2, C, device="cuda", dtype=torch.float64)
    cs = torch.zeros(C, device="cuda", dtype=torch.float64)
    DX = ops.ln_bwd(V, X, ln, gamma, col, DRES=R, col_sum=cs)
    x = X.float().requires_grad_(True)
    g = gamma.clone().requires_grad_(True)
    b = beta.clone().requires_grad_(True)
    y = torch.nn.functional.layer_norm(x, (C,), g, b, 1e-5)
    y.backward(V.float())
    ref = x.grad + (R.float() if res else 0)
    close(DX, ref, what="ln_bwd dx")
    close_stat(col[0], b.grad, "dbeta", rtol=5e-3)
    close_stat(col[1], g.grad, "dgamma", rtol=5e-3)
    close_stat(cs, DX.float().sum(0), "col_sum", rtol=5e-3)


# ------------------------------------------------------------------------------------------------- fused training-step tail
def test_flat_adamw_matches_torch_pipeline(ops):
    """cvb_grad_norm + cvb_adamw_step vs GradScaler.unscale_ -> clip_grad_norm_(10) -> torch.optim.AdamW -> GradScaler.update
    (engine/training_engine.py:289-312), including a step with an inf gradient (skipped, scale backed off)."""
    import copy
    from ml_cvnets_b200.optim import FlatAdamW
    torch.manual_seed(0)
    net = torch.nn.Sequential(torch.nn.Linear(64, 96), torch.nn.BatchNorm1d(96), torch.nn.Linear(96, 33)).cuda()
    ref = copy.deepcopy(net)
    decay = [p for p in ref.parameters() if p.dim() > 1]
    no_decay = [p for p in ref.parameters() if p.dim() == 1]
    opt = torch.optim.AdamW([{"params": decay, "weight_decay": 0.05}, {"params": no_decay, "weight_decay": 0.0}], lr=2e-3, betas=(0.9, 0.999))
    scaler = torch.amp.GradScaler("cuda", enabled=True, growth_interval=3)
    scaler.scale(torch.zeros(1, device="cuda"))
    tail = FlatAdamW(net, lr=2e-3, weight_decay=0.05, max_norm=10.0, growth_interval=3)
    g = torch.Generator(device="cuda").manual_seed(5)
    for it in range(6):
        scale = float(scaler.get_scale())
        assert abs(float(tail.loss_scale()) - scale) < 1e-3 * scale
        for p_ours, p_ref in zip(net.parameters(), ref.parameters()):
            grad = torch.randn(p_ref.shape, device="cuda", generator=g) * (30.0 if it == 1 else 1.0)  # it == 1: the clip is active
            if it == 3 and p_ref.dim() == 2:
                grad[0, 0] = float("inf")
            p_ref.grad = grad * scale
            tail.ws.gview(p_ours).copy_(grad * scale)  # p.grad is a view of the flat gradient buffer
        scaler.unscale_(opt)
        torch.nn.utils.clip_grad_norm_(list(ref.parameters()), 10.0)
        scaler.step(opt)
        scaler.update()
        tail.step()
        for p_ours, p_ref in zip(net.parameters(), ref.parameters()):
            assert torch.isfinite(p_ours).all()
            err = float((p_ours - p_ref).abs().max())
            assert err <= 2e-6 + 1e-5 * float(p_ref.abs().max()), f"step {it}: max abs diff {err}"
    assert abs(float(tail.step_count) - 5.0) < 1e-6  # one of the six steps was skipped

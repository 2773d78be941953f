"""Micro-benchmark of the hot kernels on the MobileViTv2-1.0 B=128 shapes (CUDA-event timing, L2 flushed by size)."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ml_cvnets_b200 import ops
from ml_cvnets_b200.ops import *  # noqa

dev = "cuda"
BF = torch.bfloat16
which = sys.argv[1] if len(sys.argv) > 1 else "all"
reps = int(sys.argv[2]) if len(sys.argv) > 2 else 5

def t(fn, reps=reps):
    fn(); torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(reps): fn()
    e.record(); torch.cuda.synchronize()
    return s.elapsed_time(e) / reps

def tg(fn, n=20, reps=5):
    """Per-launch time of n back-to-back launches captured in one CUDA graph: no host-side launch cost, which dominates an eager loop of
    the small attention-stage kernels."""
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fn(); fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(n): fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): g.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (reps * n)

HBM_PEAK = 3.35e12  # H100 SXM data sheet, bytes/s

def report(name, ms, nbytes):
    print(f"{name:60s} {ms*1e3:9.1f} us  {nbytes/ms/1e6:8.1f} GB/s  {nbytes/(ms*1e-3)/HBM_PEAK:5.2f} of HBM peak ({nbytes/1e6:.1f} MB algorithmic)",
          flush=True)

B = 128
def vec(n, s=1.0, o=0.0): return torch.randn(n, device=dev) * s + o

prof = which in ("prof", "one")
if which in ("all", "gemm", "prof", "one"):
    for (name, HW, K, N, mode, stats) in [c for c in [
        ("gemm L1.exp   RAW  K32 N64  @128^2 +stats", 128*128, 32, 64, A_RAW, True),
        ("gemm L1.red   AFFS K64 N64  @128^2 +stats", 128*128, 64, 64, A_AFF_SILU, True),
        ("gemm L2.0.exp RAW  K64 N128 @128^2 +stats", 128*128, 64, 128, A_RAW, True),
        ("gemm L2.0.exp RAW  K64 N128 @128^2 nostats", 128*128, 64, 128, A_RAW, False),
        ("gemm L2.0.red AFFS K128 N128 @64^2 +stats", 64*64, 128, 128, A_AFF_SILU, True),
        ("gemm L2.1.exp RAW  K128 N256 @64^2 +stats", 64*64, 128, 256, A_RAW, True),
        ("gemm L3.ffn1  GN   K128 N256 @32^2", 32*32, 128, 256, A_GN, False),
    ] if not prof or c[0].startswith(("gemm L2.0.exp RAW  K64 N128 @128^2 +stats",) + (("gemm L2.0.red AFFS", "gemm L3.ffn1") if which == "prof" else ()))]:
        M = B * HW
        A = torch.randn(M, K, device=dev).to(BF); W = (torch.randn(N, K, device=dev) * K**-0.5).to(BF)
        p = (vec(K, 0.2, 1.0), vec(K, 0.3), None)
        row = (vec(B, 0.1), vec(B, 0.1, 1.0))
        col = torch.zeros(2, N, device=dev, dtype=torch.float64) if stats else None
        out = torch.empty(M, N, device=dev, dtype=BF)
        ms = t(lambda: ops.pw_gemm(A, W, N, a_mode=mode, a_p=p, row_stats=row if mode == A_GN else None, rows_per_sample=HW, col_stats=col, out=out))
        report(name, ms, 2.0 * M * (K + N))
    if which == "one":
        sys.exit(0)
    # BNB dX gemm with SILU_BWD epilogue (L2.0 red dX: K=128(cout) -> N=128(hid))
    M = B * 64 * 64; K = 128; N = 128
    A = torch.randn(M, K, device=dev).to(BF); A2 = torch.randn(M, K, device=dev).to(BF); W = (torch.randn(N, K, device=dev) * K**-0.5).to(BF)
    Y = torch.randn(M, N, device=dev).to(BF); out = torch.empty(M, N, device=dev, dtype=BF)
    c = (vec(K, 0.2, 1.0), vec(K, 0.1), vec(K, 0.1)); col = torch.zeros(2, N, device=dev, dtype=torch.float64)
    ms = t(lambda: ops.pw_gemm(A, W, N, a_mode=A_BNB, A2=A2, a_p=c, e_mode=E_SILU_BWD, Y=Y, e_p=(vec(N, 0.2, 1.0), vec(N, 0.2)), col_stats=col, out=out))
    report("gemm L2.0.red dX BNB K128 N128 @64^2 silu_bwd+stats", ms, 2.0 * M * (2 * K + 2 * N))

if which in ("all", "wgrad", "prof"):
    for (name, HW, N, K, gm, am) in [
        ("wgrad L1.red  BNB/AFFS N64 K64 @128^2", 128*128, 64, 64, A_BNB, A_AFF_SILU),
        ("wgrad L2.0.exp BNB/RAW N128 K64 @128^2", 128*128, 128, 64, A_BNB, A_RAW),
        ("wgrad L2.1.exp BNB/RAW N256 K128 @64^2", 64*64, 256, 128, A_BNB, A_RAW),
    ][: 1 if prof else 3]:
        M = B * HW
        G = torch.randn(M, N, device=dev).to(BF); G2 = torch.randn(M, N, device=dev).to(BF); A = torch.randn(M, K, device=dev).to(BF)
        gp = (vec(N, 0.2, 1.0), vec(N, 0.1), vec(N, 0.1)); ap = (vec(K, 0.2, 1.0), vec(K, 0.2))
        dW = torch.zeros(N, K, device=dev)
        ms = t(lambda: ops.pw_wgrad(G, A, N, K, g_mode=gm, G2=G2, g_p=gp, a_mode=am, a_p=ap, dW=dW))
        report(name, ms, 2.0 * M * (2 * N + K))

if which in ("all", "dw", "prof"):
    for (name, H, C, s) in [("dw L1 s1 C64 @128^2", 128, 64, 1), ("dw L2.0 s2 C128 @128^2", 128, 128, 2), ("dw L2.1 s1 C256 @64^2", 64, 256, 1)][0:2] if prof else [("dw L1 s1 C64 @128^2", 128, 64, 1), ("dw L2.0 s2 C128 @128^2", 128, 128, 2), ("dw L2.1 s1 C256 @64^2", 64, 256, 1)]:
        Ho = (H - 1) // s + 1
        X = torch.randn(B * H * H, C, device=dev).to(BF)
        Wt = torch.randn(9, C, device=dev).to(BF).float() * 0.3
        p = (vec(C, 0.2, 1.0), vec(C, 0.3))
        col = torch.zeros(2, C, device=dev, dtype=torch.float64)
        ms = t(lambda: ops.dw_fwd(X, B, H, H, C, s, Wt, x_mode=A_AFF_SILU, x_p=p, col_stats=col))
        report(name + " fwd", ms, 2.0 * C * B * (H * H + Ho * Ho))
        DZ = torch.randn(B * Ho * Ho, C, device=dev).to(BF); Y2 = torch.randn(B * Ho * Ho, C, device=dev).to(BF)
        gp = (vec(C, 0.2, 1.0), vec(C, 0.1), vec(C, 0.1))
        ms = t(lambda: ops.dw_bwd(DZ, X, B, H, H, C, s, Wt, g_mode=A_BNB, Y2=Y2, g_p=gp, x_mode=A_AFF_SILU, x_p=p, col_stats=col))
        report(name + " bwd", ms, 2.0 * C * B * (2 * H * H + 2 * Ho * Ho))

# the MobileViTv2 attention units' memory-bound kernels at the three transformer stages (feature map H x H, d channels), timed as graph
# replays; the 8^2 operands (13-25 MB) fit in the 50 MB L2, so their rates there are L2-assisted
if which in ("all", "attn"):
    for (H, d) in [(32, 128), (16, 192), (8, 256)]:
        M, ld = B * H * H, 2 * d + 8
        qkv = torch.randn(M, ld, device=dev).to(BF)
        O, S, CTX = ops.linattn_fwd(qkv, B, H, H, d)
        # reads key, value and the query column, writes O and the fp32 softmax S
        ms = tg(lambda: ops.linattn_fwd(qkv, B, H, H, d))
        report(f"linattn_fwd @{H}^2 d={d}", ms, M * (2.0 * 2 * d + 2 + 2 * d + 4))
        dO = torch.randn(M, d, device=dev).to(BF)
        dbq = torch.zeros(ld, device=dev)
        # reads value, dO, key, the query column and S; writes dV, dK and the 8-column dq chunk
        ms = tg(lambda: ops.linattn_bwd(qkv, dO, S, CTX, B, H, H, d, dbias=dbq))
        report(f"linattn_bwd @{H}^2 d={d} +dbias", ms, M * (2.0 * 5 * d + 2 + 4 + 16))
        G = torch.randn(M, d, device=dev).to(BF); X = torch.randn(M, d, device=dev).to(BF); R = torch.randn(M, d, device=dev).to(BF)
        gn = torch.stack([vec(B, 0.1), vec(B, 0.1, 1.0)]); ss = torch.randn(2, B, device=dev, dtype=torch.float64) * 100
        col = torch.zeros(d, device=dev, dtype=torch.float64)
        for (res, cs) in [(None, col), (R, col), (R, None), (None, None)]:
            ms = tg(lambda: ops.gn_bwd_apply(G, X, gn, ss, float(H * H * d), B, H * H, DRES=res, col_sum=cs))
            report(f"gn_bwd_apply @{H}^2 C={d} {'+DRES' if res is not None else '-DRES'} {'+col_sum' if cs is not None else '-col_sum'}", ms,
                   2.0 * M * d * (3 + (res is not None)))

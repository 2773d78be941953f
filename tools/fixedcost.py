"""Fixed per-launch cost of the library's kernels: N back-to-back launches captured in one CUDA graph, replayed and timed."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from ml_cvnets_b200 import ops
from ml_cvnets_b200.ops import *  # noqa

dev = "cuda"; BF = torch.bfloat16
NL = 40

def graph_time(fn, nl=NL, reps=5):
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        fn(); fn()
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        for _ in range(nl): fn()
    g.replay(); torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps): g.replay()
    e1.record(); torch.cuda.synchronize()
    return e0.elapsed_time(e1) / (reps * nl) * 1e3

def vec(n, s=1.0, o=0.0): return torch.randn(n, device=dev) * s + o

for pdl in (True, False):
    ops.set_pdl_enabled(pdl)
    print(f"==== PDL {'on' if pdl else 'off'}")
    C = 256
    s2 = torch.zeros(2, C, device=dev, dtype=torch.float64) + 1.0
    bn = torch.nn.BatchNorm2d(C).to(dev)
    outs = torch.empty(4, C, device=dev)
    lib = ops._lib()
    def fin():
        assert 0 == (lib.cvb_bn_finalize(s2[0].data_ptr(), s2[1].data_ptr(), 1000.0, bn.weight.data_ptr(), bn.bias.data_ptr(), 1e-5, 0.1, 0, 0, 0,
                                      outs[0].data_ptr(), outs[1].data_ptr(), outs[2].data_ptr(), outs[3].data_ptr(), C, torch.cuda.current_stream().cuda_stream))
    print(f"bn_finalize (1 tiny CTA x2)                     {graph_time(fin):8.2f} us/launch")
    # the MobileViTv2 attention units' non-GEMM kernels: one sample (fixed cost) and the B = 128 bench batch, back to back in a graph
    for (H, d) in [(32, 128), (16, 192), (8, 256)]:
        for Bq in (1, 128):
            M = Bq * H * H
            qkv = torch.randn(M, 2 * d + 8, device=dev).to(BF); dO = torch.randn(M, d, device=dev).to(BF); dbq = torch.zeros(2 * d + 8, device=dev)
            _, S, CTX = ops.linattn_fwd(qkv, Bq, H, H, d)
            G = torch.randn(M, d, device=dev).to(BF); X = torch.randn(M, d, device=dev).to(BF)
            gn = torch.stack([vec(Bq, 0.1), vec(Bq, 0.1, 1.0)]); ss = torch.randn(2, Bq, device=dev, dtype=torch.float64)
            col = torch.zeros(d, device=dev, dtype=torch.float64)
            uf = graph_time(lambda: ops.linattn_fwd(qkv, Bq, H, H, d))
            ub = graph_time(lambda: ops.linattn_bwd(qkv, dO, S, CTX, Bq, H, H, d, dbias=dbq))
            ug = graph_time(lambda: ops.gn_bwd_apply(G, X, gn, ss, float(H * H * d), Bq, H * H, DRES=dO, col_sum=col))
            print(f"B={Bq:3d} @{H}^2 d={d}: linattn_fwd {uf:8.2f}  linattn_bwd+dbias {ub:8.2f}  gn_bwd_apply+DRES+col_sum {ug:8.2f} us/launch")
    for tc in (True, False):
        ops.set_tc_enabled(tc)
        for (N, K, mode) in [(192, 192, A_RAW), (256, 128, A_RAW), (192, 384, A_SILU)]:
            for M in (128, 132 * 128, 32768, 131072, 524288):
                A = torch.randn(M, K, device=dev).to(BF); W = (torch.randn(N, K, device=dev) * K**-0.5).to(BF)
                out = torch.empty(M, N, device=dev, dtype=BF)
                us = graph_time(lambda: ops.pw_gemm(A, W, N, a_mode=mode, out=out))
                print(f"gemm {'tc ' if tc else 'mma'} N={N} K={K} mode={mode} M={M:7d} tiles/SM={M/128/132:6.2f}  {us:8.2f} us/launch  {2.0*M*(K+N)/us/1e3:8.1f} GB/s")
    ops.set_tc_enabled(True)
    for (N, K) in [(192, 192), (384, 192)]:
        for M in (8192, 32768, 131072):
            G = torch.randn(M, N, device=dev).to(BF); A = torch.randn(M, K, device=dev).to(BF); dW = torch.zeros(N, K, device=dev)
            us = graph_time(lambda: ops.pw_wgrad(G, A, N, K, dW=dW))
            print(f"wgrad N={N} K={K} M={M:7d}  {us:8.2f} us/launch  {2.0*M*(K+N)/us/1e3:8.1f} GB/s")

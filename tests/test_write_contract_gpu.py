"""What every kernel writes, and where (-m gpu).

The kernel suite compares the values a kernel computes inside an output sized exactly to the result.  This file checks the write set:
every output and accumulator is a guard-banded view (write_guard.Guarded: sentinel-filled guards in front and behind, a row pitch wider than
the region wherever the API takes a leading dimension), and after the call

  - guards and [width, ld) gaps still hold the sentinel, bit for bit (a store or atomic past row M or column N, into the padding of a
    strided output, lands there instead of in the next parameter's gradient or the next layer's statistics);
  - WRITTEN outputs hold no sentinel and match an fp64 restatement on the same bf16-rounded inputs;
  - ACCUMULATED outputs are pre-filled with a nonzero prior P and must equal P + out0, out0 being the same call on a zeroed region -- bit
    for bit where the header promises the same bits run to run, within the statistics bound below for the fp64 atomics;
  - PARTIAL outputs keep the sentinel in the columns / rows the kernel is documented not to touch.

Statistics of a kernel's own output (col_sum / col_sq / samp_* and the GroupNorm-backward sums) are compared with the fp64 sum of the STORED
output read back from the guarded buffer, within stat_bound(): the fp32 partial-sum error C_SUM * 2^-23 * sum |terms|.  Where a path sums
the fp32 values BEFORE the bf16 rounding of its store, and only there, the bound adds 6 sigma of that zero-mean rounding (rounded=True): the
wgmma GEMM's full tiles without a residual (gemm_tc.cu), the depthwise kernels' interior tiles (dwconv.cu), the LayerNorm / GroupNorm
backward's col_sum (norm.cu), and the GroupNorm-backward epilogue, whose sums are of the unrounded acc by definition.  The mma.sync GEMM, the
ragged wgmma tiles, the depthwise edge tiles and bn_bwd_reduce sum the stored values and get the plain fp32 bound.  Every statistic check
carries a negative control at its shape: what one phantom (or dropped) row would add -- a typical stored row of the terms, one row's sum for
the per-sample statistics, and for the bias epilogues the bias and bias^2 of a padding row -- must exceed the bound, so the bound is shown
to catch that defect where a fraction of the maximum would not.

Shapes sit at the tile sizes +-1 / +-8 of the kernels: gemm.cu BM = 128 (mma.sync), gemm_tc.cu TC_BM = TC_BN = 128 (wgmma), wgrad_tc.cu
WT_BMP = 64 pixels / WT_KB = 128 columns, dwconv.cu CB = 64 channels and 8-pixel strips, the 64-row attention tiles.

CONTRACT names, for every export of include/cvnets_b200.h that launches a kernel, its written, accumulated and partially written outputs and
the test here that checks them; test_write_contract_cpu.py keeps it complete."""
import ctypes
import math

import pytest
import torch

from test_kernels_gpu import bf, close, dsilu, load_ref, rnd, silu  # noqa: E402
from write_guard import Guarded, bits

pytestmark = pytest.mark.gpu

CONTRACT = {
    "cvb_pw_gemm": {"written": ["C"], "accumulated": ["col_sum", "col_sq", "samp_sum", "samp_sq", "gn_ws"], "partial": [],
                    "test": "test_pw_gemm_write_set"},
    "cvb_pw_wgrad": {"written": [], "accumulated": ["dW", "dbias"], "partial": [], "test": "test_pw_wgrad_accumulates"},
    "cvb_apply_load_mode": {"written": ["OUT"], "accumulated": [], "partial": [], "test": "test_apply_load_mode_ldo"},
    "cvb_dw_fwd": {"written": ["Y"], "accumulated": ["col_sum", "col_sq"], "partial": [], "test": "test_dw_write_set"},
    "cvb_dw_bwd": {"written": ["DX"], "accumulated": ["col_sum", "col_sq", "dWt"], "partial": [], "test": "test_dw_write_set"},
    "cvb_stem_im2col": {"written": ["A"], "accumulated": [], "partial": [], "test": "test_layout_glue"},
    "cvb_bn_finalize": {"written": ["mean", "rstd", "scale", "shift"], "accumulated": ["running_mean", "running_var", "num_batches_tracked"],
                        "partial": [], "test": "test_bn_write_set"},
    "cvb_bn_eval_scale_shift": {"written": ["mean", "rstd", "scale", "shift"], "accumulated": [], "partial": [], "test": "test_bn_write_set"},
    "cvb_bn_bwd_finalize": {"written": ["dgamma", "dbeta", "c1", "c2", "c3"], "accumulated": [], "partial": [], "test": "test_bn_write_set"},
    "cvb_bn_apply": {"written": ["OUT"], "accumulated": [], "partial": [], "test": "test_bn_write_set"},
    "cvb_bn_bwd_reduce": {"written": ["DZ"], "accumulated": ["sum_dz", "sum_dzy"], "partial": [], "test": "test_bn_write_set"},
    "cvb_gn_finalize": {"written": ["mean", "rstd"], "accumulated": [], "partial": [], "test": "test_gn_write_set"},
    "cvb_gn_stats": {"written": [], "accumulated": ["samp_sum", "samp_sq"], "partial": [], "test": "test_gn_write_set"},
    "cvb_gn_bwd_apply": {"written": ["DX"], "accumulated": ["col_sum"], "partial": [], "test": "test_gn_write_set"},
    "cvb_gn_bwd": {"written": ["DX"], "accumulated": ["dgamma", "dbeta", "samp_ws"], "partial": [], "test": "test_gn_write_set"},
    "cvb_linattn_fwd": {"written": ["O", "S", "CTX"], "accumulated": [], "partial": [], "test": "test_linattn_write_set"},
    "cvb_linattn_bwd": {"written": ["DQKV"], "accumulated": ["dbias"], "partial": [], "test": "test_linattn_write_set"},
    "cvb_linattn_cross_fwd": {"written": ["O", "S", "CTX"], "accumulated": [], "partial": [], "test": "test_linattn_cross_write_set"},
    "cvb_linattn_cross_bwd": {"written": [], "accumulated": ["dbias"], "partial": ["DQK_prev", "DV_x"], "test": "test_linattn_cross_write_set"},
    "cvb_mha_fwd": {"written": ["O", "LSE"], "accumulated": [], "partial": [], "test": "test_mha_write_set"},
    "cvb_mha_bwd": {"written": ["DQKV"], "accumulated": [], "partial": [], "test": "test_mha_write_set"},
    "cvb_ln_stats": {"written": ["mean", "rstd"], "accumulated": [], "partial": [], "test": "test_ln_write_set"},
    "cvb_ln_bwd": {"written": ["DX"], "accumulated": ["dgamma", "dbeta", "col_sum"], "partial": [], "test": "test_ln_write_set"},
    "cvb_act_fwd": {"written": ["Y"], "accumulated": [], "partial": [], "test": "test_elementwise_write_set"},
    "cvb_act_bwd": {"written": ["DX"], "accumulated": [], "partial": [], "test": "test_elementwise_write_set"},
    "cvb_se_scale_fwd": {"written": ["Y"], "accumulated": [], "partial": [], "test": "test_elementwise_write_set"},
    "cvb_se_scale_bwd": {"written": ["DX"], "accumulated": ["DS"], "partial": [], "test": "test_elementwise_write_set"},
    "cvb_rng_next": {"written": ["key_out"], "accumulated": ["state"], "partial": [], "test": "test_elementwise_write_set"},
    "cvb_dropout_fwd": {"written": ["Y"], "accumulated": [], "partial": [], "test": "test_elementwise_write_set"},
    "cvb_dropout_bwd": {"written": ["DV"], "accumulated": [], "partial": [], "test": "test_elementwise_write_set"},
    "cvb_na_plan": {"written": ["tab"], "accumulated": [], "partial": [], "test": "test_range_augment_write_set"},
    "cvb_na_noise": {"written": ["eps"], "accumulated": [], "partial": [], "test": "test_range_augment_write_set"},
    "cvb_na_stats": {"written": ["mu_x", "mu_e"], "accumulated": [], "partial": [], "test": "test_range_augment_write_set"},
    "cvb_na_compose": {"written": ["coef"], "accumulated": [], "partial": [], "test": "test_range_augment_write_set"},
    "cvb_na_apply": {"written": ["Y", "sq"], "accumulated": [], "partial": [], "test": "test_range_augment_write_set"},
    "cvb_na_bwd_reduce": {"written": ["red"], "accumulated": [], "partial": [], "test": "test_range_augment_write_set"},
    "cvb_na_param_grad": {"written": ["grads"], "accumulated": [], "partial": [], "test": "test_range_augment_write_set"},
    "cvb_na_loss_fwd": {"written": ["loss", "parts"], "accumulated": [], "partial": [], "test": "test_range_augment_write_set"},
    "cvb_na_loss_bwd": {"written": ["g_sq", "g_ce"], "accumulated": [], "partial": [], "test": "test_range_augment_write_set"},
    "cvb_stem_dgrad": {"written": ["dX"], "accumulated": [], "partial": [], "test": "test_stem_dgrad_write_set"},
    "cvb_patch_stem_dgrad": {"written": ["dX"], "accumulated": [], "partial": [], "test": "test_stem_dgrad_write_set"},
    "cvb_grad_norm": {"written": ["partials"], "accumulated": ["stats"], "partial": [], "test": "test_step_tail_write_set"},
    "cvb_adamw_step": {"written": [], "accumulated": ["params", "exp_avg", "exp_avg_sq", "stats", "scale", "step", "ema"], "partial": [],
                       "test": "test_step_tail_write_set"},
    "cvb_sgd_step": {"written": [], "accumulated": ["params", "momentum_buf", "stats", "scale", "step", "ema"], "partial": [],
                     "test": "test_step_tail_write_set"},
    "cvb_grad_accumulate": {"written": [], "accumulated": ["acc"], "partial": [], "test": "test_step_tail_write_set"},
    "cvb_ema_update": {"written": [], "accumulated": ["ema"], "partial": [], "test": "test_step_tail_write_set"},
    "cvb_ce_fwd": {"written": ["lse", "loss", "n_valid"], "accumulated": [], "partial": [], "test": "test_ce_write_set"},
    "cvb_ce_bwd": {"written": ["dlogits"], "accumulated": ["dlogit_scale"], "partial": [], "test": "test_ce_write_set"},
    "cvb_cast_f64_f32": {"written": ["dst"], "accumulated": [], "partial": [], "test": "test_layout_glue"},
    "cvb_embedding_fwd": {"written": ["out"], "accumulated": [], "partial": [], "test": "test_clip_edges_write_set"},
    "cvb_embedding_bwd": {"written": [], "accumulated": ["dtable", "dpos"], "partial": [], "test": "test_clip_edges_write_set"},
    "cvb_eot_gather_fwd": {"written": ["out", "idx"], "accumulated": [], "partial": [], "test": "test_clip_edges_write_set"},
    "cvb_eot_gather_bwd": {"written": ["dX"], "accumulated": [], "partial": [], "test": "test_clip_edges_write_set"},
    "cvb_l2norm_fwd": {"written": ["Y", "inv_norm"], "accumulated": [], "partial": [], "test": "test_clip_edges_write_set"},
    "cvb_l2norm_bwd": {"written": ["DX"], "accumulated": [], "partial": [], "test": "test_clip_edges_write_set"},
    "cvb_transpose_bf16": {"written": ["Y"], "accumulated": [], "partial": [], "test": "test_clip_edges_write_set"},
    "cvb_add_bf16_f32": {"written": ["OUT"], "accumulated": [], "partial": [], "test": "test_clip_edges_write_set"},
    "cvb_zs_class_embed": {"written": ["table"], "accumulated": [], "partial": [], "test": "test_metrics_write_set"},
    "cvb_zs_logits_topk": {"written": ["logits"], "accumulated": ["hits"], "partial": [], "test": "test_metrics_write_set"},
    "cvb_cls_metrics": {"written": [], "accumulated": ["loss_sum", "counts"], "partial": ["row_loss", "ticket"], "test": "test_metrics_write_set"},
    "cvb_global_pool_fwd": {"written": ["OUT"], "accumulated": [], "partial": [], "test": "test_layout_glue"},
    "cvb_global_pool_bwd": {"written": ["DX"], "accumulated": [], "partial": [], "test": "test_layout_glue"},
    "cvb_prep_weights": {"written": ["dst"], "accumulated": [], "partial": [], "test": "test_prep_weights_write_set"},
    "cvb_unprep_grad": {"written": ["dst"], "accumulated": [], "partial": [], "test": "test_prep_weights_write_set"},
    "cvb_im2col": {"written": ["A"], "accumulated": [], "partial": [], "test": "test_layout_glue"},
    "cvb_col2im": {"written": ["dX"], "accumulated": [], "partial": [], "test": "test_layout_glue"},
    "cvb_patch_permute": {"written": ["OUT"], "accumulated": [], "partial": [], "test": "test_layout_glue"},
    "cvb_concat2": {"written": ["OUT"], "accumulated": [], "partial": [], "test": "test_layout_glue"},
    "cvb_split2": {"written": ["DA", "DB"], "accumulated": [], "partial": [], "test": "test_layout_glue"},
    "cvb_vit_tokens_interp_fwd": {"written": ["out"], "accumulated": [], "partial": [], "test": "test_vit_tokens_write_set"},
    "cvb_vit_tokens_interp_bwd": {"written": ["dpatch"], "accumulated": ["dpos", "dcls"], "partial": [], "test": "test_vit_tokens_write_set"},
}

F64, F32, I64 = torch.float64, torch.float32, torch.int64
BF = torch.bfloat16
C_SUM = 64             # fp32 partial sums: |error| <= C_SUM * 2^-23 * sum |terms|
ROUND_SIGMAS = 6.0     # sums of the fp32 values before the bf16 rounding of the store: 6 sigma of the rounding's sum


@pytest.fixture(scope="module")
def lib():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    from ml_cvnets_b200 import _lib as L
    return L.load()


@pytest.fixture(scope="module")
def ops(lib):
    from ml_cvnets_b200 import ops as o
    return o


def S():
    return torch.cuda.current_stream().cuda_stream


def strided(x, pad=8):
    """x as a view with row pitch x.shape[1] + pad (a strided operand)"""
    buf = torch.zeros(x.shape[0], x.shape[1] + pad, device=x.device, dtype=x.dtype)
    buf[:, :x.shape[1]] = x
    return buf[:, :x.shape[1]]


def prior(shape, dtype=F64, seed=0):
    """a nonzero prior for an accumulator: out must be prior + out0"""
    return (rnd(*shape, seed=900 + seed) * 3 + 0.5).to(dtype)


def stat_bound(terms, dim, rounded):
    """|fp64 accumulator - fp64 sum of terms| bound along ``dim``: fp32 partial sums, and (rounded) the bf16 rounding of each term, which
    the hot paths sum before rounding -- zero mean, |delta| <= 2^-9 |t| per factor, std 2^-8 / sqrt(3) |t| for a product of two."""
    t = terms.double()
    b = C_SUM * 2.0 ** -23 * t.abs().sum(dim)
    if rounded:
        b = b + ROUND_SIGMAS * 2.0 ** -8 / math.sqrt(3.0) * (t * t).sum(dim).sqrt()
    return b


def check_stat(acc, P, terms, dim, what, rounded, row=None):
    """acc (an accumulator pre-filled with P) - P against the fp64 sum of ``terms`` along ``dim``; returns the bound.  Negative control:
    ``row``, what one phantom or dropped row would add (default: the mean |term| of one row along ``dim``), must exceed the bound."""
    got = acc.double() - P.double()
    ref = terms.double().sum(dim)
    bnd = stat_bound(terms, dim, rounded)
    err = (got - ref).abs()
    bad = err > bnd + 1e-9
    assert not bool(bad.any()), (f"{what}: {int(bad.sum())}/{bad.numel()} outside the fp32-sum bound, worst err {float(err.max()):.4g} "
                                 f"vs bound {float(bnd[bad].min()):.4g}")
    phantom_control(terms.double().abs().mean(dim) if row is None else row, bnd, what)
    return bnd


def phantom_control(contrib, bnd, what):
    """negative control: what one phantom padding row (or a row of the next sample) would add exceeds the bound, per channel / sample"""
    c = torch.as_tensor(contrib, dtype=F64, device=bnd.device).abs().expand_as(bnd)
    assert bool((c > bnd).all()), f"{what}: the bound ({float(bnd.max()):.4g}) would not see a phantom row (smallest {float(c.min()):.4g})"


def same_bits(a, b, what):
    assert torch.equal(bits(a.contiguous()), bits(b.contiguous())), f"{what}: not bit-identical"


# ------------------------------------------------------------------------------------------------------------------ GEMM
EPIS = {  # name: (a_mode, bias, residual, e_mode, e_p, gn workspace)
    "store": (0, False, False, 0, False, False),
    "store_b": (1, True, False, 0, False, False),
    "store_br": (4, True, True, 0, False, False),
    "silu": (0, True, False, 1, False, False),
    "silu_bwd": (5, False, False, 2, True, False),
    "silu_bwd_noep": (0, False, False, 2, False, False),
    "lin_bwd": (0, False, False, 4, False, False),
    "lin_bwd_bnb": (5, False, False, 4, False, False),
    "gn_bwd": (0, False, False, 3, True, False),
    "gn_bwd_ws": (5, False, False, 3, True, True),
}
# (M, N, K, rows_per_sample): M < one tile, tile multiples +-1, N 88 / 96 / 104 and a last N tile 8 wide (136 = 128 + 8)
GEMM_SHAPES = [(100, 96, 64, 50), (127, 104, 72, 64), (129, 88, 40, 100), (257, 136, 128, 128), (513, 264, 40, 50)]
# GroupNorm-backward epilogues: whole samples; rows_per_sample a multiple of 64 takes the workspace (wgmma) path when gn_ws is given
GN_SHAPES = [(192, 96, 64, 64), (300, 104, 72, 50), (384, 136, 128, 128), (1280, 88, 40, 128)]


def _gemm_case(lib, M, N, K, rps, epi, tc):
    a_mode, has_bias, has_r, e_mode, has_ep, ws = EPIS[epi]
    nb = (M + rps - 1) // rps
    A, A2 = strided(bf(rnd(M, K, seed=1))), strided(bf(rnd(M, K, seed=2)), 16)
    W = strided(bf(rnd(N, K, scale=K ** -0.5, seed=3)))
    p = (1 + 0.2 * rnd(K, seed=5), 0.3 * rnd(K, seed=6), 0.1 * rnd(K, seed=7))
    row = (0.2 * rnd(nb, seed=8), 1 + 0.3 * rnd(nb, seed=9).abs())
    r = rnd(N, seed=4)
    bias = torch.where(r >= 0, 3 + r, r - 3) if has_bias else None      # |bias| >= 3: a phantom row's bias^2 is visible in col_sq
    R = strided(bf(rnd(M, N, seed=10)), 16) if has_r else None
    Y = strided(bf(rnd(M, N, seed=11) + (0.5 if e_mode == 3 else 0)), 24) if e_mode >= 2 else None
    ep = (1 + 0.2 * rnd(N, seed=12), 0.3 * rnd(N, seed=13)) if has_ep else (None, None)
    if e_mode == 3:
        ep = (ep[0], None)

    def run(col, samp, gws, Cg):
        a = lib_args(lib)
        a.M, a.N, a.K = M, N, K
        a.A, a.lda, a.a_mode = A.data_ptr(), A.stride(0), a_mode
        if a_mode == 5:
            a.A2, a.lda2 = A2.data_ptr(), A2.stride(0)
        a.a_p0, a.a_p1, a.a_p2 = p[0].data_ptr(), p[1].data_ptr(), p[2].data_ptr()
        if a_mode == 4 or e_mode == 3:
            a.row_mean, a.row_rstd = row[0].data_ptr(), row[1].data_ptr()
        a.rows_per_sample = rps
        a.W, a.ldw = W.data_ptr(), W.stride(0)
        a.bias = bias.data_ptr() if bias is not None else None
        a.e_mode = e_mode
        if Y is not None:
            a.Y, a.ldy = Y.data_ptr(), Y.stride(0)
        a.e_p0 = ep[0].data_ptr() if ep[0] is not None else None
        a.e_p1 = ep[1].data_ptr() if ep[1] is not None else None
        if R is not None:
            a.R, a.ldr = R.data_ptr(), R.stride(0)
        a.C, a.ldc, a.c_fp32 = Cg.ptr, Cg.ld, 0
        a.col_sum, a.col_sq = col[0].ptr, col[1].ptr
        if samp is not None:
            a.samp_sum, a.samp_sq = samp[0].ptr, samp[1].ptr
        if gws is not None:
            a.gn_ws = gws.ptr
        prev = lib.cvb_set_tc_enabled(int(tc))
        try:
            lib.cvb_pw_gemm(ctypes.byref(a), S())
            torch.cuda.synchronize()
        finally:
            lib.cvb_set_tc_enabled(prev)

    Cg = Guarded((M, N), BF, ld=N + 8)
    Pc = [prior((N,), seed=1), prior((N,), seed=2)]
    col = [Guarded((N,), F64).fill(Pc[0]), Guarded((N,), F64).fill(Pc[1])]
    want_samp = e_mode in (0, 1, 3)
    Ps = [prior((nb,), seed=3), prior((nb,), seed=4)]
    samp = [Guarded((nb,), F64).fill(Ps[0]), Guarded((nb,), F64).fill(Ps[1])] if want_samp else None
    gws = Guarded((2 * nb * N,), F64).fill(torch.zeros(2 * nb * N)) if ws else None
    run(col, samp, gws, Cg)
    out = Cg.check(f"{epi} C")
    for g, n in zip(col, ("col_sum", "col_sq")):
        g.check_bands(f"{epi} {n}")
    if samp is not None:
        for g, n in zip(samp, ("samp_sum", "samp_sq")):
            g.check_bands(f"{epi} {n}")
    if gws is not None:
        gws.check_bands(f"{epi} gn_ws")

    # values against the fp64 restatement on the same bf16-rounded (transformed) operand
    Ar = load_ref(a_mode, A, p, A2, row, rps).double()
    acc = Ar @ W.double().t()
    mu_r = row[0].double().repeat_interleave(rps)[:M, None]
    rs_r = row[1].double().repeat_interleave(rps)[:M, None]
    yv = Y.double() if Y is not None else None
    if e_mode in (0, 1):
        z = acc + (bias.double() if bias is not None else 0)
        ref = (z + R.double() if R is not None else z) if e_mode == 0 else silu(z)
    elif e_mode == 2:
        ref = acc * (dsilu(ep[0].double() * yv + ep[1].double()) if has_ep else dsilu(yv))
    elif e_mode == 4:
        ref = acc
    else:
        ref = acc * ep[0].double()
    close(out, ref, what=f"{epi} C")

    o = out.double()
    sid = torch.arange(M, device="cuda") // rps
    # the wgmma kernel serves this N (gemm_tc.cu) and its full tiles without a residual sum the values before the store's rounding
    wg = tc and N >= 96 and not (N % 128 != 0 and N % 128 < 64 and N < 256)
    pre_round = wg and e_mode == 0 and R is None and M >= 128
    if e_mode == 3:
        # the GroupNorm-backward sums are of the unrounded acc; what the test reads back is bf16(acc * gamma)
        xh = (yv - mu_r) * rs_r
        v = o / ep[0].double()
        check_stat(col[0].region(), Pc[0], v, 0, f"{epi} col_sum (dbeta)", rounded=True)
        check_stat(col[1].region(), Pc[1], v * xh, 0, f"{epi} col_sq (dgamma)", rounded=True)
        terms_s, terms_q = o, o * xh
    else:
        second = o * yv if e_mode in (2, 4) else o * o
        bs = check_stat(col[0].region(), Pc[0], o, 0, f"{epi} col_sum", rounded=pre_round)
        bq = check_stat(col[1].region(), Pc[1], second, 0, f"{epi} col_sq", rounded=pre_round)
        if e_mode == 0 and bias is not None and M % 128:  # a phantom padding row of the last tile would add its bias
            phantom_control(bias, bs, f"{epi} col_sum")
            phantom_control(bias.double() ** 2, bq, f"{epi} col_sq")
        terms_s, terms_q = o, o * o
    if samp is not None:
        ts = torch.zeros(nb, N, device="cuda", dtype=F64).index_add_(0, sid, terms_s)
        tq = torch.zeros(nb, N, device="cuda", dtype=F64).index_add_(0, sid, terms_q)
        # a row of the next sample counted in this one (or one dropped): one row's sum over the channels
        check_stat(samp[0].region(), Ps[0], ts, 1, f"{epi} samp_sum", rounded=e_mode == 3, row=terms_s.abs().sum(1).mean())
        check_stat(samp[1].region(), Ps[1], tq, 1, f"{epi} samp_sq", rounded=e_mode == 3, row=terms_q.abs().sum(1).mean())


def lib_args(lib):
    from ml_cvnets_b200._lib import cvb_gemm_args
    return cvb_gemm_args()


@pytest.mark.parametrize("tc", [True, False], ids=["wgmma", "mma"])
@pytest.mark.parametrize("epi", [e for e in EPIS if not e.startswith("gn")])
@pytest.mark.parametrize("M,N,K,rps", GEMM_SHAPES)
def test_pw_gemm_write_set(lib, M, N, K, rps, epi, tc):
    _gemm_case(lib, M, N, K, rps, epi, tc)


@pytest.mark.parametrize("tc", [True, False], ids=["wgmma", "mma"])
@pytest.mark.parametrize("epi", ["gn_bwd", "gn_bwd_ws"])
@pytest.mark.parametrize("M,N,K,rps", GN_SHAPES)
def test_pw_gemm_gn_bwd_write_set(lib, M, N, K, rps, epi, tc):
    _gemm_case(lib, M, N, K, rps, epi, tc)


@pytest.mark.parametrize("M", [129, 1000])
def test_pw_gemm_k_streaming_write_set(lib, M):
    """narrow N with a K the mma.sync kernel's resident panel cannot hold: the wgmma kernel streams the weight (any N)"""
    _gemm_case_kstream(lib, M, 64, 3456)


def _gemm_case_kstream(lib, M, N, K):
    A, W = strided(bf(rnd(M, K, seed=31))), bf(rnd(N, K, scale=K ** -0.5, seed=32))
    r = rnd(N, seed=33)
    bias = torch.where(r >= 0, 3 + r, r - 3)
    Cg = Guarded((M, N), BF, ld=N + 16)
    P = [prior((N,), seed=5), prior((N,), seed=6)]
    col = [Guarded((N,), F64).fill(P[0]), Guarded((N,), F64).fill(P[1])]
    a = lib_args(lib)
    a.M, a.N, a.K = M, N, K
    a.A, a.lda, a.W, a.ldw, a.bias = A.data_ptr(), A.stride(0), W.data_ptr(), W.stride(0), bias.data_ptr()
    a.C, a.ldc = Cg.ptr, Cg.ld
    a.col_sum, a.col_sq = col[0].ptr, col[1].ptr
    lib.cvb_pw_gemm(ctypes.byref(a), S())
    torch.cuda.synchronize()
    out = Cg.check("k-streaming C")
    close(out, A.double() @ W.double().t() + bias.double(), what="k-streaming C")
    o = out.double()
    for g in col:
        g.check_bands("k-streaming col")
    bs = check_stat(col[0].region(), P[0], o, 0, "k-streaming col_sum", rounded=True)  # wgmma full tiles: sums before the rounding
    bq = check_stat(col[1].region(), P[1], o * o, 0, "k-streaming col_sq", rounded=True)
    phantom_control(bias, bs, "k-streaming col_sum")
    phantom_control(bias.double() ** 2, bq, "k-streaming col_sq")


# (M, N, K): K % 64 == 0 on the wgmma weight-gradient kernel, the others on mma.sync; M not a multiple of the 64-pixel stage
@pytest.mark.parametrize("tc", [True, False], ids=["wgmma", "mma"])
@pytest.mark.parametrize("M,N,K", [(129, 96, 64), (1000, 88, 72), (777, 264, 128), (63, 136, 192)])
@pytest.mark.parametrize("with_bias", [True, False])
def test_pw_wgrad_accumulates(lib, M, N, K, tc, with_bias):
    """dW [N, lddw > K] and dbias are added onto their prior contents, bit for bit: dW = P + dW0 (the fp64 partials are added to dW once)"""
    from ml_cvnets_b200._lib import cvb_wgrad_args
    G, G2, A = strided(bf(rnd(M, N, seed=41))), bf(rnd(M, N, seed=42)), strided(bf(rnd(M, K, seed=43)), 24)
    gp = (1 + 0.2 * rnd(N, seed=44), 0.3 * rnd(N, seed=45), 0.1 * rnd(N, seed=46))
    ap = (1 + 0.2 * rnd(K, seed=47), 0.3 * rnd(K, seed=48))
    res = []
    for fill in ("zero", "prior"):
        dW = Guarded((N, K), F32, ld=K + 8)
        db = Guarded((N,), F32)
        PW, Pb = prior((N, K), F32, seed=7), prior((N,), F32, seed=8)
        dW.fill(torch.zeros(N, K) if fill == "zero" else PW)
        db.fill(torch.zeros(N) if fill == "zero" else Pb)
        a = cvb_wgrad_args()
        a.M, a.N, a.K = M, N, K
        a.G, a.ldg, a.G2, a.ldg2, a.g_mode = G.data_ptr(), G.stride(0), G2.data_ptr(), G2.stride(0), 5
        a.g_p0, a.g_p1, a.g_p2 = gp[0].data_ptr(), gp[1].data_ptr(), gp[2].data_ptr()
        a.A, a.lda, a.a_mode = A.data_ptr(), A.stride(0), 2
        a.a_p0, a.a_p1 = ap[0].data_ptr(), ap[1].data_ptr()
        a.dW, a.lddw = dW.ptr, dW.ld
        a.dbias = db.ptr if with_bias else None
        prev = lib.cvb_set_tc_enabled(int(tc))
        try:
            lib.cvb_pw_wgrad(ctypes.byref(a), S())
            torch.cuda.synchronize()
        finally:
            lib.cvb_set_tc_enabled(prev)
        dW.check_bands("dW")
        db.check_bands("dbias")
        res.append((dW.region(), db.region(), PW, Pb))
    (w0, b0, _, _), (w1, b1, PW, Pb) = res
    Gr, Ar = load_ref(5, G, gp, G2).double(), load_ref(2, A, ap + (None,)).double()
    ref = Gr.t() @ Ar
    close(w0, ref, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) + 1e-5, what="dW")
    same_bits(w1, PW + w0, "dW += (onto a nonzero prior)")
    if with_bias:
        close(b0, Gr.sum(0), rtol=2e-3, atol=2e-3 * float(Gr.sum(0).abs().max()) + 1e-4, what="dbias")
        same_bits(b1, Pb + b0, "dbias +=")
    else:
        same_bits(b1, Pb, "dbias untouched when not requested")


@pytest.mark.parametrize("mode", [1, 2, 3, 4, 5])  # every transform (RAW has nothing to materialise and is rejected)
@pytest.mark.parametrize("M,K", [(129, 72), (1000, 392)])
def test_apply_load_mode_ldo(lib, M, K, mode):
    rps = 50
    nb = (M + rps - 1) // rps
    A, A2 = strided(bf(rnd(M, K, seed=51))), strided(bf(rnd(M, K, seed=52)), 16)
    p = (1 + 0.2 * rnd(K, seed=53), 0.3 * rnd(K, seed=54), 0.1 * rnd(K, seed=55))
    row = (0.2 * rnd(nb, seed=56), 1 + 0.3 * rnd(nb, seed=57).abs())
    O = Guarded((M, K), BF, ld=K + 8)
    lib.cvb_apply_load_mode(A.data_ptr(), A.stride(0), A2.data_ptr(), A2.stride(0), mode, p[0].data_ptr(), p[1].data_ptr(), p[2].data_ptr(),
                            row[0].data_ptr(), row[1].data_ptr(), rps, O.ptr, O.ld, M, K, S())
    out = O.check(f"apply_load_mode {mode}")
    close(out, load_ref(mode, A, p, A2, row, rps), what=f"apply_load_mode {mode}")


# ------------------------------------------------------------------------------------------------------------ depthwise
# (B, H, W, C, stride, ksize, dilation, backward too): H / W off the 8-pixel strips, C with a partial 64-channel block, the odd
# stride-2 maps of EfficientNet b1-b3 (15 / 65 / 75, forward only: the stride-2 backward needs even maps)
# interior tiles next to edge tiles and a partial channel block, forward and backward at stride 1, forward at stride 2 (the stride-2
# backward's interior statistics, summed before the rounding over >= 16 x 32 input pixels, carry more rounding noise than one typical row
# of some channels: no bound on them could show a phantom row there)
DW_CASES = [(1, 24, 26, 136, 1, 3, 1, True), (1, 36, 40, 136, 2, 3, 1, False),
            (2, 17, 13, 72, 1, 3, 1, True), (2, 15, 15, 40, 2, 3, 1, False), (1, 65, 65, 24, 2, 5, 1, False), (1, 75, 75, 16, 2, 3, 1, False),
            (2, 18, 14, 200, 2, 5, 1, True), (3, 12, 20, 136, 2, 3, 1, True), (2, 11, 9, 72, 1, 5, 1, True), (2, 13, 11, 72, 1, 3, 2, True),
            (1, 9, 12, 136, 1, 3, 4, True)]


def dw_interior(H, W, C, s, k, dil, bwd):
    """whether some CTA of the dense depthwise kernels takes the interior path (dwconv.cu: the whole tile and a full 64-channel block inside
    the map), whose statistics are summed before the bf16 rounding of the store; the dilated kernel sums the stored values"""
    if dil > 1 or C < 64:
        return False
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    TH = 16 if (s == 1 and k == 3 and Ho > 8) else 8
    if not bwd:
        TW = 16 if (s == 1 and Wo > 8) else 8
        return Ho >= TH and Wo >= TW
    TW = 16 if Wo > 8 else 8
    return H >= s * TH and W >= s * TW  # the backward's tile is one of input pixels


@pytest.mark.parametrize("B,H,W,C,stride,k,dil,bwd", DW_CASES)
def test_dw_write_set(lib, B, H, W, C, stride, k, dil, bwd):
    from ml_cvnets_b200._lib import cvb_dw_bwd_args, cvb_dw_fwd_args
    F = torch.nn.functional
    pad = (k // 2) * dil
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    X = bf(rnd(B * H * W, C, seed=61))
    w = bf(rnd(C, 1, k, k, scale=0.3, seed=62)).float()
    Wt = w.view(C, k * k).t().contiguous()
    xp = (1 + 0.2 * rnd(C, seed=63), 0.3 * rnd(C, seed=64))
    Yg = Guarded((B * Ho * Wo, C), BF)
    P = [prior((C,), seed=9), prior((C,), seed=10)]
    col = [Guarded((C,), F64).fill(P[0]), Guarded((C,), F64).fill(P[1])]
    a = cvb_dw_fwd_args()
    a.B, a.H, a.W, a.C, a.stride = B, H, W, C, stride
    a.X, a.x_mode, a.x_p0, a.x_p1 = X.data_ptr(), 2, xp[0].data_ptr(), xp[1].data_ptr()
    a.Wt, a.Y, a.dilation, a.ksize = Wt.data_ptr(), Yg.ptr, dil, k
    a.col_sum, a.col_sq = col[0].ptr, col[1].ptr
    lib.cvb_dw_fwd(ctypes.byref(a), S())
    torch.cuda.synchronize()
    y = Yg.check("dw_fwd Y")
    xa = load_ref(2, X, xp + (None,)).double().view(B, H, W, C).permute(0, 3, 1, 2)
    ref = F.conv2d(xa, w.double(), None, stride=stride, padding=pad, dilation=dil, groups=C).permute(0, 2, 3, 1).reshape(-1, C)
    close(y, ref, what="dw_fwd Y")
    for g in col:
        g.check_bands("dw_fwd col")
    yd = y.double()
    pre = dw_interior(H, W, C, stride, k, dil, bwd=False)
    check_stat(col[0].region(), P[0], yd, 0, "dw_fwd col_sum", rounded=pre)
    check_stat(col[1].region(), P[1], yd * yd, 0, "dw_fwd col_sq", rounded=pre)
    if not bwd:
        return
    DZ, Y2 = bf(rnd(B * Ho * Wo, C, seed=65)), bf(rnd(B * Ho * Wo, C, seed=66))
    gp = (1 + 0.2 * rnd(C, seed=67), 0.3 * rnd(C, seed=68), 0.1 * rnd(C, seed=69))
    res = []
    for fill in ("zero", "prior"):
        DX = Guarded((B * H * W, C), BF)
        Pw = prior((k * k, C), F32, seed=11)
        dWt = Guarded((k * k, C), F32).fill(torch.zeros(k * k, C) if fill == "zero" else Pw)
        Q = [prior((C,), seed=12), prior((C,), seed=13)]
        cb = [Guarded((C,), F64).fill(Q[0]), Guarded((C,), F64).fill(Q[1])]
        b = cvb_dw_bwd_args()
        b.B, b.H, b.W, b.C, b.stride = B, H, W, C, stride
        b.DZ, b.Y2, b.g_mode = DZ.data_ptr(), Y2.data_ptr(), 5
        b.g_p0, b.g_p1, b.g_p2 = gp[0].data_ptr(), gp[1].data_ptr(), gp[2].data_ptr()
        b.X, b.x_mode, b.x_p0, b.x_p1 = X.data_ptr(), 2, xp[0].data_ptr(), xp[1].data_ptr()
        b.Wt, b.DX, b.dWt, b.dilation, b.ksize = Wt.data_ptr(), DX.ptr, dWt.ptr, dil, k
        b.col_sum, b.col_sq = cb[0].ptr, cb[1].ptr
        lib.cvb_dw_bwd(ctypes.byref(b), S())
        torch.cuda.synchronize()
        dx = DX.check("dw_bwd DX")
        dWt.check_bands("dw_bwd dWt")
        for g in cb:
            g.check_bands("dw_bwd col")
        res.append((dx, dWt.region(), Pw, cb, Q))
    (dx0, w0, _, cb0, Q0), (dx1, w1, Pw, _, _) = res
    same_bits(dx1, dx0, "dw_bwd DX (independent of the accumulators' prior)")
    same_bits(w1, Pw + w0, "dw_bwd dWt +=")
    dy = load_ref(5, DZ, gp, Y2).double().view(B, Ho, Wo, C).permute(0, 3, 1, 2)
    xv = xa.clone().requires_grad_(True)
    wv = w.double().clone().requires_grad_(True)
    F.conv2d(xv, wv, None, stride=stride, padding=pad, dilation=dil, groups=C).backward(dy)
    da = xv.grad.permute(0, 2, 3, 1).reshape(-1, C) * dsilu(xp[0].double() * X.double() + xp[1].double())
    close(dx0, da, what="dw_bwd DX")
    gw = wv.grad.view(C, k * k).t()
    close(w0, gw, rtol=3e-3, atol=3e-3 * float(gw.abs().max()) + 1e-5, what="dw_bwd dWt")
    d = dx0.double()
    pre = dw_interior(H, W, C, stride, k, dil, bwd=True)
    check_stat(cb0[0].region(), Q0[0], d, 0, "dw_bwd col_sum", rounded=pre)
    check_stat(cb0[1].region(), Q0[1], d * X.double(), 0, "dw_bwd col_sq", rounded=pre)


# ------------------------------------------------------------------------------------------------------------ attention
def _mha_ref64(qkv, B, S_, H, c, scale):
    x = qkv.view(B, S_, 3, H, c).permute(2, 0, 3, 1, 4)
    att = torch.softmax((x[0] * scale) @ x[1].transpose(-1, -2), dim=-1)
    return (att @ x[2]).transpose(1, 2).reshape(B * S_, H * c)


@pytest.mark.parametrize("impl", [0, 1, 2])
@pytest.mark.parametrize("S_,H,c", [(63, 2, 64), (65, 2, 64), (129, 1, 64), (257, 2, 64), (65, 3, 32), (129, 2, 16)])
def test_mha_write_set(lib, impl, S_, H, c):
    if impl == 2 and c != 64:
        pytest.skip("the streaming kernels serve head_dim 64 only")
    B, C = 2, H * c
    qkv = strided(bf(rnd(B * S_, 3 * C, seed=71)), 8)
    dO = strided(bf(rnd(B * S_, C, seed=72)), 8)
    scale = c ** -0.5
    O = Guarded((B * S_, C), BF, ld=C + 16)
    LSE = Guarded((B * H * S_,), F32)
    DQ = Guarded((B * S_, 3 * C), BF, ld=3 * C + 24)
    old = lib.cvb_set_mha_impl(impl)
    try:
        lib.cvb_mha_fwd(qkv.data_ptr(), qkv.stride(0), B, S_, H, c, scale, None, None, O.ptr, O.ld, LSE.ptr, S())
        # the backward reads O and dO with one leading dimension: dO is copied into a buffer with O's pitch
        dOp = torch.zeros(B * S_, O.ld, device="cuda", dtype=BF)
        dOp[:, :C] = dO
        lib.cvb_mha_bwd(qkv.data_ptr(), qkv.stride(0), O.ptr, dOp.data_ptr(), O.ld, LSE.ptr, B, S_, H, c, scale, None, None, DQ.ptr, DQ.ld, S())
        torch.cuda.synchronize()
    finally:
        lib.cvb_set_mha_impl(old)
    o = O.check("mha O")
    LSE.check("mha LSE")
    dq = DQ.check("mha dQKV")
    x = qkv.double().requires_grad_(True)
    ref = _mha_ref64(x, B, S_, H, c, scale)
    close(o, ref.detach(), what="mha O")
    ref.backward(dO.double())
    close(dq, x.grad, rtol=3e-2, atol=2e-2 * float(x.grad.abs().max()) + 1e-6, what="mha dQKV")


def _linattn_ref(T, d, dO):
    """T [B, P, N, ld] fp64 (requires grad): keys [0, d), values [d, 2d), query column 2d"""
    s = torch.softmax(T[..., 2 * d], dim=-1)
    ctx = (T[..., :d] * s[..., None]).sum(2)
    out = torch.relu(T[..., d:2 * d]) * ctx[:, :, None]
    out.backward(dO)
    return out.detach(), s.detach(), ctx.detach()


def _fold_tokens(x, B, H, W):
    """feature map [B*H*W, c] -> [B, 4, (H/2)(W/2), c] (p = 2*row parity + column parity, n = (h/2)(W/2) + w/2) and back"""
    c = x.shape[-1]
    return x.view(B, H // 2, 2, W // 2, 2, c).permute(0, 2, 4, 1, 3, 5).reshape(B, 4, -1, c)


def _unfold_tokens(t, B, H, W):
    c = t.shape[-1]
    return t.view(B, 2, 2, H // 2, W // 2, c).permute(0, 3, 1, 4, 2, 5).reshape(B * H * W, c)


@pytest.mark.parametrize("patch,B,H,W,d", [(2, 2, 10, 14, 24), (2, 1, 18, 6, 64), (0, 2, 4, 37, 16), (0, 3, 2, 65, 40)])
def test_linattn_write_set(lib, patch, B, H, W, d):
    ldq = 2 * d + 16
    M = B * H * W
    QKV = bf(rnd(M, ldq, seed=81))
    DO = strided(bf(rnd(M, d, seed=82)), 8)
    Pp, N = (4, (H // 2) * (W // 2)) if patch == 2 else (H, W)
    O = Guarded((M, d), BF, ld=d + 8)
    Sg, CT = Guarded((B * Pp * N,), F32), Guarded((B * Pp * d,), F32)
    lib.cvb_linattn_fwd(QKV.data_ptr(), ldq, B, H, W, d, patch, O.ptr, O.ld, Sg.ptr, CT.ptr, S())
    res = []
    for fill in ("zero", "prior"):
        DQ = Guarded((M, ldq), BF)
        Pb = prior((2 * d + 1,), F32, seed=14)
        db = Guarded((2 * d + 1,), F32).fill(torch.zeros(2 * d + 1) if fill == "zero" else Pb)
        lib.cvb_linattn_bwd(QKV.data_ptr(), ldq, DO.data_ptr(), DO.stride(0), Sg.ptr, CT.ptr, B, H, W, d, patch, DQ.ptr, db.ptr, S())
        torch.cuda.synchronize()
        res.append((DQ.check("linattn DQKV"), db, Pb))
        db.check_bands("linattn dbias")
    o, s, ctx = O.check("linattn O"), Sg.check("linattn S"), CT.check("linattn CTX")
    (dq, db0, _), (dq1, db1, Pb) = res
    same_bits(dq1, dq, "linattn DQKV")
    same_bits(db1.region(), Pb + db0.region(), "linattn dbias +=")
    assert float(dq[:, 2 * d + 1:].float().abs().max()) == 0.0, "DQKV pad columns are documented as zeroed"
    T = QKV.double().view(B, Pp, N, ldq) if patch == 0 else _fold_tokens(QKV.double(), B, H, W)
    T = T.clone().requires_grad_(True)
    dO = DO.double().view(B, Pp, N, d) if patch == 0 else _fold_tokens(DO.double(), B, H, W)
    ro, rs, rc = _linattn_ref(T, d, dO)
    back = (lambda t: t.reshape(M, -1)) if patch == 0 else (lambda t: _unfold_tokens(t, B, H, W))
    close(o, back(ro), what="linattn O")
    close(s.view(B, Pp, N), rs, rtol=2e-3, atol=1e-5, what="linattn S")
    close(ctx.view(B, Pp, d), rc, rtol=2e-3, atol=1e-4, what="linattn CTX")
    g = back(T.grad)
    close(dq[:, :2 * d], g[:, :2 * d], what="linattn dK, dV")
    close(dq[:, 2 * d], g[:, 2 * d], rtol=3e-2, atol=2e-2 * float(g[:, 2 * d].abs().max()) + 1e-6, what="linattn dq")
    close(db0.region()[:2 * d], dq[:, :2 * d].double().sum(0), rtol=2e-3, atol=2e-3 * float(db0.region().abs().max()) + 1e-5, what="dbias")


@pytest.mark.parametrize("B,P,Mq,N,d", [(2, 4, 37, 29, 16), (1, 2, 65, 63, 40)])
def test_linattn_cross_write_set(lib, B, P, Mq, N, d):
    ldq = 2 * d + 16
    QK = bf(rnd(B * P * Mq, ldq, seed=91))
    VX = bf(rnd(B * P * N, ldq, seed=92))
    DO = bf(rnd(B * P * N, d, seed=93))
    O = Guarded((B * P * N, d), BF, ld=d + 8)
    Sg, CT = Guarded((B * P * Mq,), F32), Guarded((B * P * d,), F32)
    lib.cvb_linattn_cross_fwd(QK.data_ptr(), ldq, B, P, Mq, d, VX.data_ptr(), ldq, N, O.ptr, O.ld, Sg.ptr, CT.ptr, S())
    DQK, DV = Guarded((B * P * Mq, ldq), BF), Guarded((B * P * N, ldq), BF)
    Pb = prior((2 * d + 1,), F32, seed=15)
    db = Guarded((2 * d + 1,), F32).fill(Pb)
    lib.cvb_linattn_cross_bwd(QK.data_ptr(), ldq, VX.data_ptr(), ldq, DO.data_ptr(), d, Sg.ptr, CT.ptr, B, P, Mq, N, d, DQK.ptr, DV.ptr, db.ptr, S())
    torch.cuda.synchronize()
    o = O.check("cross O")
    Sg.check("cross S")
    CT.check("cross CTX")
    for g, what in ((DQK, "DQK_prev"), (DV, "DV_x"), (db, "dbias")):
        g.check_bands(what)
    DQK.check_written("DQK_prev key columns", slice(0, d))
    DQK.check_written("DQK_prev query and pad columns", slice(2 * d, ldq))
    assert not bool(DQK.view[:, 2 * d + 1:].float().any()), "DQK_prev: the pad columns are zeroed"
    DQK.check_untouched("DQK_prev value columns", slice(d, 2 * d))
    DV.check_written("DV_x value columns", slice(d, 2 * d))
    DV.check_untouched("DV_x key columns", slice(0, d))
    DV.check_untouched("DV_x query and pad columns", slice(2 * d, ldq))
    qk = QK.double().view(B, P, Mq, ldq).clone().requires_grad_(True)
    vx = VX.double().view(B, P, N, ldq).clone().requires_grad_(True)
    s = torch.softmax(qk[..., 2 * d], dim=-1)
    ctx = (qk[..., :d] * s[..., None]).sum(2)
    out = torch.relu(vx[..., d:2 * d]) * ctx[:, :, None]
    out.backward(DO.double().view(B, P, N, d))
    close(o, out.detach().reshape(-1, d), what="cross O")
    gk = qk.grad.reshape(-1, ldq)
    close(DQK.view[:, :d], gk[:, :d], what="cross dK")
    close(DV.view[:, d:2 * d], vx.grad.reshape(-1, ldq)[:, d:2 * d], what="cross dV")
    close(DQK.view[:, 2 * d], gk[:, 2 * d], rtol=3e-2, atol=2e-2 * float(gk[:, 2 * d].abs().max()) + 1e-6, what="cross dq")
    got = db.region().double() - Pb.double()
    ref = torch.cat([DQK.view[:, :d].double().sum(0), DV.view[:, d:2 * d].double().sum(0), DQK.view[:, 2 * d:2 * d + 1].double().sum(0)])
    close(got, ref, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) + 1e-5, what="cross dbias +=")


# ---------------------------------------------------------------------------------------------------------------- norms
@pytest.mark.parametrize("M,C", [(129, 1280), (77, 200), (1000, 72)])
def test_ln_write_set(lib, M, C):
    X = strided(bf(rnd(M, C, seed=101) * 1.5 + 0.3), 8)
    V, R = bf(rnd(M, C, seed=102)), bf(rnd(M, C, seed=103))
    gamma = 1 + 0.2 * rnd(C, seed=104)
    mean, rstd = Guarded((M,), F32), Guarded((M,), F32)
    lib.cvb_ln_stats(X.data_ptr(), X.stride(0), M, C, 1e-5, mean.ptr, rstd.ptr, S())
    torch.cuda.synchronize()
    mu, rs = mean.check("ln mean"), rstd.check("ln rstd")
    xd = X.double()
    close(mu, xd.mean(1), rtol=1e-4, atol=1e-5, what="ln mean")
    close(rs, (xd.var(1, unbiased=False) + 1e-5).rsqrt(), rtol=1e-3, atol=1e-5, what="ln rstd")
    Xc = X.contiguous()
    DX = Guarded((M, C), BF)
    P = [prior((C,), seed=16), prior((C,), seed=17), prior((C,), seed=18)]
    dg, dbt, cs = (Guarded((C,), F64).fill(p) for p in P)
    lib.cvb_ln_bwd(V.data_ptr(), Xc.data_ptr(), mean.ptr, rstd.ptr, gamma.data_ptr(), R.data_ptr(), DX.ptr, M, C, dg.ptr, dbt.ptr, cs.ptr, S())
    torch.cuda.synchronize()
    dx = DX.check("ln_bwd DX")
    for g in (dg, dbt, cs):
        g.check_bands("ln_bwd accumulators")
    x = xd.clone().requires_grad_(True)
    gm = gamma.double().clone().requires_grad_(True)
    torch.nn.functional.layer_norm(x, (C,), gm, None, 1e-5).backward(V.double())
    close(dx, x.grad + R.double(), what="ln_bwd DX")
    xh = (xd - mu.double()[:, None]) * rs.double()[:, None]
    check_stat(dbt.region(), P[1], V.double(), 0, "ln_bwd dbeta", rounded=False)
    check_stat(dg.region(), P[0], V.double() * xh, 0, "ln_bwd dgamma", rounded=False)
    check_stat(cs.region(), P[2], dx.double(), 0, "ln_bwd col_sum (of the stored DX)", rounded=True)  # summed before the rounding


@pytest.mark.parametrize("B,rps,C", [(3, 37, 72), (2, 129, 200), (4, 64, 1280)])
def test_gn_write_set(lib, B, rps, C):
    M = B * rps
    X = strided(bf(rnd(M, C, seed=111) + 0.5), 8)
    G, DR = bf(rnd(M, C, seed=112)), bf(rnd(M, C, seed=113))
    P = [prior((B,), seed=19), prior((B,), seed=20)]
    ss = [Guarded((B,), F64).fill(P[0]), Guarded((B,), F64).fill(P[1])]
    lib.cvb_gn_stats(X.data_ptr(), X.stride(0), B, rps, C, ss[0].ptr, ss[1].ptr, S())
    torch.cuda.synchronize()
    for g in ss:
        g.check_bands("gn_stats")
    xs = X.double().reshape(B, -1)
    # a row of the next sample counted in this one (a sample boundary off by one) would add that row's sums
    xr = X.double().view(B, rps, C)
    check_stat(ss[1].region(), P[1], xs * xs, 1, "gn_stats samp_sq", rounded=False, row=(xr * xr).sum(2).mean(1))
    check_stat(ss[0].region(), P[0], xs, 1, "gn_stats samp_sum", rounded=False, row=xr.abs().sum(2).mean(1))
    zs = torch.stack([xs.sum(1), (xs * xs).sum(1)])
    zst = zs.clone()
    mean, rstd = Guarded((B,), F32), Guarded((B,), F32)
    lib.cvb_gn_finalize(zst[0].data_ptr(), zst[1].data_ptr(), float(rps * C), 1e-5, mean.ptr, rstd.ptr, B, S())
    torch.cuda.synchronize()
    mu, rs = mean.check("gn mean"), rstd.check("gn rstd")
    close(mu, xs.mean(1), rtol=1e-5, atol=1e-6, what="gn mean")
    close(rs, (xs.var(1, unbiased=False) + 1e-5).rsqrt(), rtol=1e-4, atol=1e-6, what="gn rstd")
    Xc = X.contiguous()
    xh = ((xs - mu.double()[:, None]) * rs.double()[:, None]).view(M, C)
    sg = torch.stack([G.double().view(B, -1).sum(1), (G.double() * xh).view(B, -1).sum(1)])
    DX = Guarded((M, C), BF)
    Q = prior((C,), seed=21)
    cs = Guarded((C,), F64).fill(Q)
    lib.cvb_gn_bwd_apply(G.data_ptr(), Xc.data_ptr(), mean.ptr, rstd.ptr, sg[0].data_ptr(), sg[1].data_ptr(), float(rps * C), DR.data_ptr(), DX.ptr,
                         B, rps, C, cs.ptr, S())
    torch.cuda.synchronize()
    dx = DX.check("gn_bwd_apply DX")
    cs.check_bands("gn_bwd_apply col_sum")
    m1, m2 = (sg[0] / (rps * C)).repeat_interleave(rps)[:, None], (sg[1] / (rps * C)).repeat_interleave(rps)[:, None]
    ref = rs.double().repeat_interleave(rps)[:, None] * (G.double() - m1 - xh * m2) + DR.double()
    close(dx, ref, what="gn_bwd_apply DX")
    check_stat(cs.region(), Q, dx.double(), 0, "gn_bwd_apply col_sum (of the stored DX)", rounded=True)  # summed before the rounding
    # the stand-alone backward
    gamma = 1 + 0.2 * rnd(C, seed=114)
    DX2 = Guarded((M, C), BF)
    Pg = [prior((C,), seed=22), prior((C,), seed=23)]
    dgm, dbt = Guarded((C,), F64).fill(Pg[0]), Guarded((C,), F64).fill(Pg[1])
    ws = Guarded((2 * B,), F64).fill(torch.zeros(2 * B))
    lib.cvb_gn_bwd(G.data_ptr(), Xc.data_ptr(), mean.ptr, rstd.ptr, gamma.data_ptr(), float(rps * C), None, DX2.ptr, B, rps, C, dgm.ptr, dbt.ptr,
                   ws.ptr, S())
    torch.cuda.synchronize()
    dx2 = DX2.check("gn_bwd DX")
    for g in (dgm, dbt, ws):
        g.check_bands("gn_bwd accumulators")
    check_stat(dbt.region(), Pg[1], G.double(), 0, "gn_bwd dbeta", rounded=False)
    check_stat(dgm.region(), Pg[0], G.double() * xh, 0, "gn_bwd dgamma", rounded=False)
    vg = G.double() * gamma.double()
    mv = vg.view(B, -1).mean(1).repeat_interleave(rps)[:, None]
    mvx = (vg * xh).view(B, -1).mean(1).repeat_interleave(rps)[:, None]
    close(dx2, rs.double().repeat_interleave(rps)[:, None] * (vg - mv - xh * mvx), what="gn_bwd DX")


@pytest.mark.parametrize("M,C", [(129, 200), (1000, 72)])
def test_bn_write_set(lib, M, C):
    y = bf(rnd(M, C, seed=121) * 1.5 + 0.3)
    yd = y.double()
    st = torch.stack([yd.sum(0), (yd * yd).sum(0)]).contiguous()
    gamma, beta = 1 + 0.2 * rnd(C, seed=122), 0.1 * rnd(C, seed=123)
    out = [Guarded((C,), F32) for _ in range(4)]
    rm0, rv0 = 0.1 * rnd(C, seed=124), 1 + 0.2 * rnd(C, seed=125).abs()
    rm, rv = Guarded((C,), F32).fill(rm0), Guarded((C,), F32).fill(rv0)
    nbt = Guarded((1,), I64).fill(torch.tensor([7]))
    lib.cvb_bn_finalize(st[0].data_ptr(), st[1].data_ptr(), float(M), gamma.data_ptr(), beta.data_ptr(), 1e-5, 0.1, rm.ptr, rv.ptr, nbt.ptr,
                        *[g.ptr for g in out], C, S())
    torch.cuda.synchronize()
    mean, rstd, scale, shift = [g.check(f"bn_finalize out {i}") for i, g in enumerate(out)]
    for g in (rm, rv, nbt):
        g.check_bands("bn_finalize running statistics")
    assert int(nbt.region()[0]) == 8, "num_batches_tracked += 1"
    mu, var = yd.mean(0), yd.var(0, unbiased=False)
    close(mean, mu, rtol=1e-5, atol=1e-6, what="mean")
    close(rstd, (var + 1e-5).rsqrt(), rtol=1e-4, atol=1e-6, what="rstd")
    close(scale, gamma.double() * (var + 1e-5).rsqrt(), rtol=1e-4, atol=1e-6, what="scale")
    close(rm.region(), 0.9 * rm0.double() + 0.1 * mu, rtol=1e-5, atol=1e-6, what="running_mean (in place)")
    close(rv.region(), 0.9 * rv0.double() + 0.1 * yd.var(0, unbiased=True), rtol=1e-5, atol=1e-6, what="running_var (in place)")
    ev = [Guarded((C,), F32) for _ in range(4)]
    lib.cvb_bn_eval_scale_shift(gamma.data_ptr(), beta.data_ptr(), rm0.data_ptr(), rv0.data_ptr(), 1e-5, *[g.ptr for g in ev], C, S())
    torch.cuda.synchronize()
    e = [g.check(f"bn_eval out {i}") for i, g in enumerate(ev)]
    close(e[2], gamma.double() * (rv0.double() + 1e-5).rsqrt(), rtol=1e-5, atol=1e-6, what="eval scale")
    dz = bf(rnd(M, C, seed=126))
    sd = torch.stack([dz.double().sum(0), (dz.double() * yd).sum(0)]).contiguous()
    bo = [Guarded((C,), F32) for _ in range(5)]
    lib.cvb_bn_bwd_finalize(sd[0].data_ptr(), sd[1].data_ptr(), float(M), gamma.data_ptr(), out[0].ptr, out[1].ptr, 0,
                            *[g.ptr for g in bo], C, S())
    torch.cuda.synchronize()
    dgam, dbet = [bo[i].check(f"bn_bwd_finalize out {i}") for i in range(2)]
    for i in range(2, 5):
        bo[i].check(f"bn_bwd_finalize coef {i - 2}")
    close(dbet, sd[0], rtol=1e-5, atol=1e-5, what="dbeta")
    close(dgam, (sd[1] - mu * sd[0]) * (var + 1e-5).rsqrt(), rtol=1e-4, atol=1e-4, what="dgamma")
    R = bf(rnd(M, C, seed=127))
    OUT = Guarded((M, C), BF)
    lib.cvb_bn_apply(y.data_ptr(), out[2].ptr, out[3].ptr, 1, R.data_ptr(), OUT.ptr, M, C, S())
    torch.cuda.synchronize()
    ref = silu(yd * scale.double() + shift.double()) + R.double()
    close(OUT.check("bn_apply OUT"), ref, what="bn_apply")
    DZ = Guarded((M, C), BF)
    Q = [prior((C,), seed=24), prior((C,), seed=25)]
    acc = [Guarded((C,), F64).fill(Q[0]), Guarded((C,), F64).fill(Q[1])]
    lib.cvb_bn_bwd_reduce(dz.data_ptr(), y.data_ptr(), out[2].ptr, out[3].ptr, 1, DZ.ptr, acc[0].ptr, acc[1].ptr, M, C, S())
    torch.cuda.synchronize()
    d = DZ.check("bn_bwd_reduce DZ")
    for g in acc:
        g.check_bands("bn_bwd_reduce sums")
    close(d, dz.double() * dsilu(yd * scale.double() + shift.double()), what="bn_bwd_reduce DZ")
    dd = d.double()
    check_stat(acc[0].region(), Q[0], dd, 0, "bn_bwd_reduce sum_dz (of the stored DZ)", rounded=False)
    check_stat(acc[1].region(), Q[1], dd * yd, 0, "bn_bwd_reduce sum_dzy", rounded=False)


# ------------------------------------------------------------------------------------------------------- loss / metrics
@pytest.mark.parametrize("B,C,ld,ldd", [(37, 997, 1000, 1016), (5, 10, 16, 24), (130, 1000, 1000, 1008)])
def test_ce_write_set(lib, B, C, ld, ldd):
    full = torch.zeros(B, ld, device="cuda", dtype=BF)  # logits [B, C] at row pitch ld
    full[:, :C] = bf(rnd(B, C, seed=131) * 2)
    tgt = torch.randint(0, C, (B,), device="cuda", generator=torch.Generator("cuda").manual_seed(B))
    tgt[1] = -100
    lse, loss, nv = Guarded((B,), F32), Guarded((1,), F32), Guarded((1,), F32)
    lib.cvb_ce_fwd(full.data_ptr(), ld, B, C, tgt.data_ptr(), -100, 0.1, lse.ptr, loss.ptr, nv.ptr, None, None, S())
    D = Guarded((B, ldd), BF)
    lib.cvb_ce_bwd(full.data_ptr(), ld, B, C, tgt.data_ptr(), -100, 0.1, lse.ptr, nv.ptr, None, None, D.ptr, ldd, None, None, None, S())
    torch.cuda.synchronize()
    for g, n in ((lse, "lse"), (loss, "loss"), (nv, "n_valid")):
        g.check(f"ce_fwd {n}")
    d = D.check("ce_bwd dlogits")
    assert not bool(d[:, C:].float().abs().any()), "ce_bwd: dlogits columns >= C are documented as zeroed"
    x = full[:, :C].double().requires_grad_(True)
    ref = torch.nn.functional.cross_entropy(x, tgt, ignore_index=-100, label_smoothing=0.1)
    ref.backward()
    close(loss.region(), ref.detach().reshape(1), rtol=1e-4, atol=1e-5, what="ce loss")
    assert float(nv.region()[0]) == B - 1
    close(d[:, :C], x.grad, rtol=2e-2, atol=1e-2 * float(x.grad.abs().max()), what="ce dlogits")
    # CLIP's learnable temperature: the loss of clamp(exp(logit_scale), 0, 100) * raw; d loss / d logit_scale is added onto a prior
    ls = torch.tensor([math.log(3.0)], device="cuda")
    lse2, loss2, nv2 = Guarded((B,), F32), Guarded((1,), F32), Guarded((1,), F32)
    lib.cvb_ce_fwd(full.data_ptr(), ld, B, C, tgt.data_ptr(), -100, 0.1, lse2.ptr, loss2.ptr, nv2.ptr, None, ls.data_ptr(), S())
    D2 = Guarded((B, ldd), BF)
    dls = Guarded((1,), F32).fill(torch.tensor([0.75]))
    lib.cvb_ce_bwd(full.data_ptr(), ld, B, C, tgt.data_ptr(), -100, 0.1, lse2.ptr, nv2.ptr, None, None, D2.ptr, ldd, None, ls.data_ptr(), dls.ptr, S())
    torch.cuda.synchronize()
    for g, n in ((lse2, "lse"), (loss2, "loss"), (nv2, "n_valid")):
        g.check(f"ce_fwd (logit_scale) {n}")
    d2 = D2.check("ce_bwd (logit_scale) dlogits")
    dls.check_bands("dlogit_scale")
    assert not bool(d2[:, C:].float().any()), "ce_bwd (logit_scale): dlogits columns >= C are zeroed"
    x2 = full[:, :C].double().requires_grad_(True)
    p = ls.double().requires_grad_(True)
    ref2 = torch.nn.functional.cross_entropy(p.exp().clamp(max=100.0) * x2, tgt, ignore_index=-100, label_smoothing=0.1)
    ref2.backward()
    close(loss2.region(), ref2.detach().reshape(1), rtol=1e-4, atol=1e-5, what="ce loss (logit_scale)")
    close(d2[:, :C], x2.grad, rtol=2e-2, atol=1e-2 * float(x2.grad.abs().max()), what="ce dlogits (logit_scale)")
    close(dls.region() - 0.75, p.grad, rtol=1e-3, atol=1e-5, what="dlogit_scale +=")


def test_metrics_write_set(lib):
    B, C = 77, 1000
    g = torch.Generator("cuda").manual_seed(3)
    logits = strided(bf(torch.randn(B, C, device="cuda", generator=g) * 3), 8)
    tgt = torch.randint(0, C, (B,), device="cuda", generator=g)
    tgt[:10] = logits[:10].float().argmax(1)
    tgt[10] = -1
    res = []
    for fill in ("zero", "prior"):
        Pl, Pc = torch.tensor([12.5], dtype=F64), torch.tensor([3, 5, 11])
        ls = Guarded((1,), F64).fill(torch.zeros(1) if fill == "zero" else Pl)
        cn = Guarded((3,), I64).fill(torch.zeros(3) if fill == "zero" else Pc)
        rl = Guarded((B,), F32)
        tk = Guarded((1,), torch.int32).fill(torch.zeros(1))
        lib.cvb_cls_metrics(logits.data_ptr(), logits.stride(0), B, C, tgt.data_ptr(), -1, ls.ptr, cn.ptr, rl.ptr, tk.ptr, S())
        torch.cuda.synchronize()
        for q in (ls, cn, rl, tk):
            q.check_bands("cls_metrics")
        assert int(tk.region()[0]) == 0, "cls_metrics leaves the ticket zero"
        res.append((ls.region(), cn.region(), Pl.cuda(), Pc.cuda()))
    (l0, c0, _, _), (l1, c1, Pl, Pc) = res
    same_bits(c1, Pc + c0, "cls_metrics counts +=")
    same_bits(l1, Pl + l0, "cls_metrics loss_sum +=")
    lf = logits.double()
    valid = tgt != -1
    rank = (lf > lf.gather(1, tgt.clamp(min=0)[:, None])).sum(1)
    assert c0.tolist() == [int(((rank < 1) & valid).sum()), int(((rank < 5) & valid).sum()), int(valid.sum())]
    ce = (torch.logsumexp(lf, 1) - lf.gather(1, tgt.clamp(min=0)[:, None])[:, 0])[valid].sum()
    assert abs(float(l0[0]) - float(ce)) <= 1e-5 * float(ce.abs())
    # CLIP zero-shot: class table (written) and top-k hits (accumulated)
    R_, d, Cl, Mc = 61, 136, 9, 5
    X = strided(bf(rnd(R_, d, seed=141)), 8)
    perm = torch.randint(0, R_, (Cl * Mc,), device="cuda", generator=g).int()
    T = Guarded((d, Cl), F32)
    lib.cvb_zs_class_embed(X.data_ptr(), X.stride(0), R_, perm.data_ptr(), Cl, Mc, d, T.ptr, S())
    torch.cuda.synchronize()
    tab = T.check("zs_class_embed table")
    xn = torch.nn.functional.normalize(X.double()[perm.long()].view(Cl, Mc, d), dim=-1).mean(1)
    close(tab, torch.nn.functional.normalize(xn, dim=-1).t(), rtol=1e-4, atol=1e-6, what="zs table")
    img = strided(bf(torch.nn.functional.normalize(rnd(B, d, seed=142), dim=-1)), 8)
    zt = torch.randint(0, Cl, (B,), device="cuda", generator=g)
    tc = tab.contiguous()
    res = []
    for fill in ("zero", "prior"):
        Ph = torch.tensor([4, 9])
        hits = Guarded((2,), I64).fill(torch.zeros(2) if fill == "zero" else Ph)
        lg = Guarded((B, Cl), F32)
        lib.cvb_zs_logits_topk(img.data_ptr(), img.stride(0), tc.data_ptr(), B, d, Cl, 100.0, zt.data_ptr(), lg.ptr, hits.ptr, S())
        torch.cuda.synchronize()
        hits.check_bands("zs hits")
        res.append((lg.check("zs logits"), hits.region(), Ph.cuda()))
    (lg0, h0, _), (_, h1, Ph) = res
    same_bits(h1, Ph + h0, "zs_logits_topk hits +=")
    ref = 100.0 * img.double() @ tc.double()
    close(lg0, ref, rtol=1e-4, atol=1e-3, what="zs logits")


# ------------------------------------------------------------------------------------------------------- step tail
@pytest.mark.parametrize("n", [1021, 1030, 4099])
def test_step_tail_write_set(lib, n):
    """params, moments, EMA, accumulator: exactly n elements updated; stats[3] (and [0], [1]) left zero by the step kernel"""
    g = torch.Generator("cuda").manual_seed(n)
    grads = torch.randn(n, device="cuda", generator=g)
    p0 = torch.randn(n, device="cuda", generator=g)
    wd = (torch.rand(n, device="cuda", generator=g) < 0.5).float() * 0.05
    hp = torch.tensor([1e-2], device="cuda")
    nblk = lib.cvb_grad_norm_blocks(n)
    for opt in ("adamw", "sgd"):
        params = Guarded((n,), F32).fill(p0)
        m1, m2 = Guarded((n,), F32).fill(torch.zeros(n)), Guarded((n,), F32).fill(torch.zeros(n))
        ema0 = p0 + 0.1
        ema = Guarded((n,), F32).fill(ema0)
        stats = Guarded((4,), F32).fill(torch.zeros(4))
        scale = Guarded((2,), F32).fill(torch.tensor([1.0, 0.0]))
        step = Guarded((1,), F32).fill(torch.zeros(1))
        part = Guarded((2 * nblk,), F32)
        lib.cvb_grad_norm(grads.data_ptr(), n, scale.ptr, 1.0, stats.ptr, part.ptr, S())
        if opt == "adamw":
            lib.cvb_adamw_step(params.ptr, grads.data_ptr(), m1.ptr, m2.ptr, wd.data_ptr(), n, hp.data_ptr(), 0.9, 0.999, 1e-8, 0.0, stats.ptr,
                               scale.ptr, step.ptr, 2.0, 0.5, 2000, ema.ptr, 0.25, part.ptr, S())
        else:
            lib.cvb_sgd_step(params.ptr, grads.data_ptr(), m1.ptr, wd.data_ptr(), n, hp.data_ptr(), 0.9, 1, 0.0, stats.ptr, scale.ptr, step.ptr,
                             2.0, 0.5, 2000, ema.ptr, 0.25, part.ptr, S())
        torch.cuda.synchronize()
        for q, what in ((params, "params"), (m1, "moment 1"), (m2, "moment 2"), (ema, "ema"), (stats, "stats"), (scale, "scale"), (step, "step")):
            q.check_bands(f"{opt} {what}")
        part.check(f"{opt} partials")
        st = stats.region()
        assert float(st[3]) == 0.0 and float(st[1]) == 0.0 and float(st[2]) == 1.0, f"{opt}: stats {st.tolist()}"
        close(st[0:1], (grads.double() ** 2).sum().reshape(1), rtol=1e-5, atol=0, what=f"{opt}: stats[0] = the step's squared norm")
        assert float(step.region()[0]) == 1.0
        gd, pd = grads.double(), p0.double()
        if opt == "adamw":
            m = 0.1 * gd
            v = 0.001 * gd * gd
            ref = pd * (1 - 1e-2 * wd.double()) - 1e-2 * (m / 0.1) / ((v / 0.001).sqrt() + 1e-8)
            close(m2.region(), v, rtol=3e-5, atol=1e-12, what="adamw exp_avg_sq")  # 1 - beta2 is formed in fp32: 1.3e-5 off 0.001
        else:
            m = gd + wd.double() * pd
            ref = pd - 1e-2 * (m + 0.9 * m)
        close(m1.region(), m, rtol=1e-5, atol=1e-9, what=f"{opt} moment")
        close(params.region(), ref, rtol=1e-5, atol=1e-6, what=f"{opt} params")
        close(ema.region(), 0.75 * ema0.double() + 0.25 * params.region().double(), rtol=1e-5, atol=1e-6, what=f"{opt} ema")
    acc0 = torch.randn(n, device="cuda", generator=g)
    acc = Guarded((n,), F32).fill(acc0)
    lib.cvb_grad_accumulate(acc.ptr, grads.data_ptr(), n, S())
    torch.cuda.synchronize()
    acc.check_bands("grad_accumulate")
    same_bits(acc.region(), acc0 + grads, "grad_accumulate acc += g")
    e = Guarded((n,), F32).fill(acc0)
    lib.cvb_ema_update(e.ptr, grads.data_ptr(), n, 0.001, S())
    torch.cuda.synchronize()
    e.check_bands("ema_update")
    close(e.region(), acc0.double() * 0.999 + 0.001 * grads.double(), rtol=1e-6, atol=1e-7, what="ema_update")


# ---------------------------------------------------------------------------------------------- element-wise passes
def test_elementwise_write_set(lib, ops):
    n = 8 * 1037
    X, DY = bf(rnd(n, seed=151) * 2), bf(rnd(n, seed=152))
    F = torch.nn.functional
    acts = {0: lambda z: F.silu(z), 1: lambda z: F.gelu(z), 2: F.relu, 3: F.hardswish, 4: F.hardsigmoid, 5: torch.sigmoid}
    for kind, f in acts.items():
        Y, DX = Guarded((n,), BF), Guarded((n,), BF)
        lib.cvb_act_fwd(X.data_ptr(), Y.ptr, n, kind, S())
        lib.cvb_act_bwd(DY.data_ptr(), X.data_ptr(), DX.ptr, n, kind, S())
        torch.cuda.synchronize()
        close(Y.check(f"act_fwd {kind}"), f(X.double()), what=f"act_fwd {kind}")
        x = X.double().requires_grad_(True)
        f(x).backward(DY.double())
        keep = (X.float().abs() != 3) & (X.float() != 0)  # the hard activations' kinks: either one-sided derivative is right
        close(DX.check(f"act_bwd {kind}")[keep], x.grad[keep], what=f"act_bwd {kind}")
    # squeeze-excitation scaling: DS accumulated, the same bits run to run
    B, HW, C = 3, 37, 200
    Xs, Ss, Ds = bf(rnd(B * HW, C, seed=153)), bf(rnd(B, C, seed=154)), bf(rnd(B * HW, C, seed=155))
    Y = Guarded((B * HW, C), BF)
    lib.cvb_se_scale_fwd(Xs.data_ptr(), Ss.data_ptr(), Y.ptr, B, HW, C, S())
    res = []
    for fill in ("zero", "prior"):
        DX = Guarded((B * HW, C), BF)
        P = prior((B, C), F32, seed=26)
        DSg = Guarded((B, C), F32).fill(torch.zeros(B, C) if fill == "zero" else P)
        lib.cvb_se_scale_bwd(Ds.data_ptr(), Xs.data_ptr(), Ss.data_ptr(), DX.ptr, DSg.ptr, B, HW, C, S())
        torch.cuda.synchronize()
        DSg.check_bands("se DS")
        res.append((DX.check("se DX"), DSg.region(), P))
    close(Y.check("se Y"), (Xs.double().view(B, HW, C) * Ss.double()[:, None]).view(-1, C), what="se Y")
    (dx0, ds0, _), (dx1, ds1, P) = res
    same_bits(dx1, dx0, "se DX")
    same_bits(ds1, P + ds0, "se DS +=")
    close(ds0, (Ds.double() * Xs.double()).view(B, HW, C).sum(1), rtol=1e-4, atol=1e-4, what="se DS")
    # dropout / stochastic depth: Y = R + V * mask, DV = DY * mask (the same mask)
    M, C = 129, 72
    V, R = bf(rnd(M, C, seed=156)), bf(rnd(M, C, seed=157))
    state = Guarded((2,), I64).fill(torch.tensor([1234, 5]))
    key = Guarded((1,), I64)
    lib.cvb_rng_next(state.ptr, key.ptr, S())
    torch.cuda.synchronize()
    key.check("rng key")
    state.check_bands("rng state")
    assert state.region().tolist() == [1234, 6], "rng_next advances the counter in place"
    Yd, DV = Guarded((M, C), BF), Guarded((M, C), BF)
    lib.cvb_dropout_fwd(V.data_ptr(), R.data_ptr(), Yd.ptr, M, C, 43, 0.2, 0.3, key.ptr, S())
    lib.cvb_dropout_bwd(V.data_ptr(), DV.ptr, M, C, 43, 0.2, 0.3, key.ptr, S())
    torch.cuda.synchronize()
    y, dv = Yd.check("dropout Y"), DV.check("dropout DV")
    close(y, R.double() + dv.double(), what="dropout Y = R + DV(V)")


# ---------------------------------------------------------------------------------------------------- RangeAugment
def test_range_augment_write_set(lib, ops):
    B, H, W = 5, 24, 20
    x = torch.rand(B, 3, H, W, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    key = torch.tensor([987654321], device="cuda", dtype=I64)
    tab = Guarded((4 + 3 * B,), F32)
    lib.cvb_na_plan(key.data_ptr(), B, 7, tab.ptr, S())
    eps = Guarded((B * 3 * H * W,), F32)
    lib.cvb_na_noise(key.data_ptr(), B, H, W, eps.ptr, S())
    mux, mue = Guarded((3 * B,), F64), Guarded((3 * B,), F64)
    lib.cvb_na_stats(x.data_ptr(), None, key.data_ptr(), B, H, W, 1, mux.ptr, mue.ptr, S())
    raw = [torch.tensor([v], device="cuda") for v in (0.3, 0.6, 0.4, 0.7, -2.0, -1.0)]
    coef = Guarded((3 * B * 3,), F32)
    lib.cvb_na_compose(tab.ptr, mux.ptr, mue.ptr, ops._ptr6(raw), B, coef.ptr, S())
    Y, sq = Guarded((B * 3 * H * W,), F32), Guarded((3 * B,), F64)
    lib.cvb_na_apply(x.data_ptr(), None, key.data_ptr(), coef.ptr, B, H, W, 1, Y.ptr, sq.ptr, S())
    target = torch.tensor([20.0, 30.0], device="cuda")
    stp = torch.tensor([1], device="cuda", dtype=I64)
    ce = torch.tensor([2.5], device="cuda")
    loss, parts = Guarded((1,), F32), Guarded((2,), F32)
    lib.cvb_na_loss_fwd(sq.ptr, B, H, W, target.data_ptr(), 2, stp.data_ptr(), 1.0, 0.5, ce.data_ptr(), 1.0, loss.ptr, parts.ptr, S())
    gsq, gce = Guarded((3 * B,), F64), Guarded((1,), F32)
    lib.cvb_na_loss_bwd(sq.ptr, B, H, W, target.data_ptr(), 2, stp.data_ptr(), 1.0, 0.5, None, None, gsq.ptr, gce.ptr, 1.0, S())
    dY = torch.randn(B, 3, H, W, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    red = Guarded((3 * B * 3,), F64)
    lib.cvb_na_bwd_reduce(dY.data_ptr(), gsq.ptr, x.data_ptr(), None, key.data_ptr(), coef.ptr, B, H, W, 1, red.ptr, S())
    grads = Guarded((6,), F32)
    gp = (ctypes.c_void_p * 6)(*[grads.ptr + 4 * i for i in range(6)])
    lib.cvb_na_param_grad(tab.ptr, mux.ptr, mue.ptr, red.ptr, ops._ptr6(raw), B, gp, S())
    torch.cuda.synchronize()
    for g, what in ((tab, "tab"), (eps, "eps"), (mux, "mu_x"), (mue, "mu_e"), (coef, "coef"), (Y, "Y"), (sq, "sq"), (loss, "loss"), (parts, "parts"),
                    (gsq, "g_sq"), (gce, "g_ce"), (red, "red"), (grads, "grads")):
        g.check(f"RangeAugment {what}")
    close(mux.region(), x.double().mean([2, 3]).reshape(-1), rtol=1e-9, atol=1e-9, what="mu_x")
    yv = Y.region().view(B, 3, H, W).double()
    close(sq.region(), ((yv - x.double()) ** 2).sum([2, 3]).reshape(-1), rtol=1e-6, atol=1e-9, what="sq")
    assert float(parts.region()[0]) == 2.5 and float(gce.region()[0]) == 1.0


# ------------------------------------------------------------------------------------------------------- layout glue
def test_layout_glue(lib):
    F = torch.nn.functional
    # dense im2col with lda > k*k*Cin: the pad columns are written with zeros; col2im writes every element of dX
    B, Cin, H, W, k, st, pad = 2, 8, 11, 13, 3, 2, 1
    x = bf(rnd(B, H, W, Cin, seed=161)).permute(0, 3, 1, 2)
    Ho, Wo = (H + 2 * pad - k) // st + 1, (W + 2 * pad - k) // st + 1
    lda = k * k * Cin + 8
    A = Guarded((B * Ho * Wo, lda), BF)
    lib.cvb_im2col(x.data_ptr(), 0, *x.stride(), B, Cin, H, W, k, st, pad, A.ptr, lda, S())
    torch.cuda.synchronize()
    a = A.check("im2col A")
    ref = F.unfold(x.double(), k, padding=pad, stride=st).view(B, Cin, k * k, -1).permute(0, 3, 2, 1).reshape(-1, k * k * Cin)
    same_bits(a[:, :k * k * Cin], ref.to(BF), "im2col")
    assert not bool(a[:, k * k * Cin:].float().any()), "im2col pad columns are zero"
    dA = bf(rnd(B * Ho * Wo, lda, seed=162))
    DX = Guarded((B * H * W, Cin), BF)
    lib.cvb_col2im(dA.data_ptr(), lda, B, Cin, H, W, k, st, pad, DX.ptr, S())
    torch.cuda.synchronize()
    cols = dA[:, :k * k * Cin].double().view(B, Ho * Wo, k * k, Cin).permute(0, 3, 2, 1).reshape(B, Cin * k * k, -1)
    close(DX.check("col2im dX"), F.fold(cols, (H, W), k, padding=pad, stride=st).permute(0, 2, 3, 1).reshape(-1, Cin), what="col2im")
    # the MobileViTv2 stem's patch matrix: 32 columns, 27..31 zero
    img = rnd(2, 3, 18, 14, seed=163)
    As = Guarded((2 * 9 * 7, 32), BF)
    lib.cvb_stem_im2col(img.data_ptr(), *img.stride(), 2, 18, 14, As.ptr, None, S())
    torch.cuda.synchronize()
    a = As.check("stem_im2col A")
    same_bits(a[:, :27], F.unfold(img.to(BF).double(), 3, padding=1, stride=2).permute(0, 2, 1).reshape(-1, 27).to(BF), "stem_im2col")
    assert not bool(a[:, 27:].float().any()), "stem_im2col columns 27..31 are zero"
    # MobileViT-v1 unfold / fold, concat / split, global pool
    Bp, Hp, Wp, C = 2, 6, 10, 24
    X = bf(rnd(Bp * Hp * Wp, C, seed=164))
    T, Bk = Guarded((Bp * Hp * Wp, C), BF), Guarded((Bp * Hp * Wp, C), BF)
    lib.cvb_patch_permute(X.data_ptr(), T.ptr, Bp, Hp, Wp, C, 2, 2, 0, S())
    lib.cvb_patch_permute(T.ptr, Bk.ptr, Bp, Hp, Wp, C, 2, 2, 1, S())
    torch.cuda.synchronize()
    T.check("patch_permute unfold")
    same_bits(Bk.check("patch_permute fold"), X, "fold(unfold(x))")
    M, C1, C2 = 129, 40, 24
    A1, A2 = bf(rnd(M, C1, seed=165)), bf(rnd(M, C2, seed=166))
    OUT = Guarded((M, C1 + C2), BF)
    lib.cvb_concat2(A1.data_ptr(), A2.data_ptr(), C1, C2, M, OUT.ptr, S())
    DA, DB = Guarded((M, C1), BF), Guarded((M, C2), BF)
    lib.cvb_split2(OUT.ptr, C1, C2, M, DA.ptr, DB.ptr, S())
    torch.cuda.synchronize()
    same_bits(OUT.check("concat2"), torch.cat([A1, A2], 1), "concat2")
    same_bits(DA.check("split2 DA"), A1, "split2 DA")
    same_bits(DB.check("split2 DB"), A2, "split2 DB")
    Bg, HW, Cg = 3, 49, 200
    Xg = bf(rnd(Bg * HW, Cg, seed=167))
    PO, PX = Guarded((Bg, Cg), BF), Guarded((Bg * HW, Cg), BF)
    lib.cvb_global_pool_fwd(Xg.data_ptr(), Bg, HW, Cg, PO.ptr, S())
    lib.cvb_global_pool_bwd(PO.ptr, Bg, HW, Cg, PX.ptr, S())
    torch.cuda.synchronize()
    po = PO.check("global_pool_fwd")
    close(po, Xg.double().view(Bg, HW, Cg).mean(1), what="global_pool_fwd")
    close(PX.check("global_pool_bwd"), (po.double() / HW)[:, None].expand(Bg, HW, Cg).reshape(-1, Cg), what="global_pool_bwd")
    # batched fp64 -> fp32 cast: exactly n elements per descriptor
    from ml_cvnets_b200._lib import cvb_cast_desc
    srcs = [rnd(n, seed=168 + n).double() for n in (13, 1, 257)]
    dsts = [Guarded((s.numel(),), F32) for s in srcs]
    descs = (cvb_cast_desc * 3)(*[cvb_cast_desc(s.data_ptr(), d.ptr, s.numel(), 0) for s, d in zip(srcs, dsts)])
    table = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).cuda()
    lib.cvb_cast_f64_f32(table.data_ptr(), 3, 257, S())
    torch.cuda.synchronize()
    for s, d in zip(srcs, dsts):
        same_bits(d.check("cast_f64_f32"), s.float(), "cast_f64_f32")


def test_prep_weights_write_set(lib):
    """every layout kind in one launch, each destination padded by ldd and dst_rows: the padding is written with zeros"""
    from ml_cvnets_b200._lib import cvb_prep_desc
    rows, cols = 33, 20
    src = rnd(rows, cols, seed=171)
    wd = rnd(24, 9, seed=172)
    vec = rnd(rows, seed=173)
    dense = rnd(16, 3 * 9, seed=174)  # [Cout, Cin * taps]
    kinds = [  # (kind, src, rows, cols, ldd, dst_rows, rot, dst shape, dtype)
        (0, src, rows, cols, 32, 40, 1, (40, 32), BF),
        (1, src, rows, cols, 48, cols, 1, (cols, 48), BF),
        (2, wd, 24, 9, 24, 9, 0, (9, 24), F32),
        (3, vec, rows, 1, 1, 40, 1, (40,), F32),
        (4, dense, 16, 27, 32, 24, 9, (24, 32), BF),
        (5, dense, 16, 27, 24, 32, 9, (32, 24), BF),
    ]
    dsts = [Guarded(shape, dt) for (_, _, _, _, _, _, _, shape, dt) in kinds]
    descs = (cvb_prep_desc * len(kinds))(*[cvb_prep_desc(s.data_ptr(), d.ptr, r, c, ldd, dr, kd, rot)
                                          for (kd, s, r, c, ldd, dr, rot, _, _), d in zip(kinds, dsts)])
    table = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8).cuda()
    lib.cvb_prep_weights(table.data_ptr(), len(kinds), 40 * 48, S())
    torch.cuda.synchronize()
    out = [d.check(f"prep kind {k[0]}") for k, d in zip(kinds, dsts)]
    perm = torch.cat([src[1:], src[:1]])
    ref0 = torch.zeros(40, 32, device="cuda")
    ref0[:rows, :cols] = perm
    same_bits(out[0], ref0.to(BF), "ROWMAJOR (zero padded)")
    ref1 = torch.zeros(cols, 48, device="cuda")
    ref1[:, :rows] = perm.t()
    same_bits(out[1], ref1.to(BF), "TRANSPOSED (zero padded)")
    same_bits(out[2], wd.t().to(BF).float(), "TAPMAJOR_F32")
    ref3 = torch.zeros(40, device="cuda")
    ref3[:rows] = torch.cat([vec[1:], vec[:1]])
    same_bits(out[3], ref3, "VECTOR_F32 (zero padded)")
    pm = dense.view(16, 3, 9).permute(0, 2, 1).reshape(16, 27)  # (tap, ci) order
    ref4 = torch.zeros(24, 32, device="cuda")
    ref4[:16, :27] = pm
    same_bits(out[4], ref4.to(BF), "PATCH (zero padded)")
    ref5 = torch.zeros(32, 24, device="cuda")
    ref5[:27, :16] = pm.t()
    same_bits(out[5], ref5.to(BF), "PATCH_T (zero padded)")
    # gradient scatter-back: exactly rows * cols elements of the parameter's layout
    g = rnd(40, 24, seed=175)
    gp = rnd(16, 40, seed=176)
    cases = [  # (kind, src, rows, cols, lds, rot, expected parameter-layout gradient)
        (0, g, rows, 16, 24, 1, torch.cat([g[rows - 1:rows, :16], g[:rows - 1, :16]])),
        (2, g, 24, 9, 24, 0, g[:9].t()),
        (4, gp, 16, 27, 40, 9, gp[:, :27].reshape(16, 9, 3).permute(0, 2, 1).reshape(16, 27)),
    ]
    for kind, src_g, r, c, lds, rot, ref in cases:
        dst = Guarded((r, c), F32)
        lib.cvb_unprep_grad(src_g.data_ptr(), dst.ptr, r, c, lds, kind, rot, S())
        torch.cuda.synchronize()
        same_bits(dst.check(f"unprep kind {kind}"), ref, f"unprep kind {kind}")


@pytest.mark.parametrize("B,Ho,Wo,C0", [(2, 9, 7, 32), (1, 16, 16, 16)])
def test_stem_dgrad_write_set(lib, B, Ho, Wo, C0):
    F = torch.nn.functional
    dz, y = bf(rnd(B * Ho * Wo, C0, seed=181)), bf(rnd(B * Ho * Wo, C0, seed=182))
    coef = torch.stack([1 + 0.2 * rnd(C0, seed=183), 0.1 * rnd(C0, seed=184), 0.05 * rnd(C0, seed=185)]).contiguous()
    dy = bf(coef[0] * dz.float() + coef[1] * y.float() + coef[2]).double().view(B, Ho, Wo, C0).permute(0, 3, 1, 2)
    w3 = bf(rnd(C0, 3, 3, 3, scale=0.3, seed=186))
    wprep = torch.zeros(C0, 32, device="cuda", dtype=BF)
    wprep[:, :27] = w3.reshape(C0, 27)
    dX = Guarded((B * 3 * 2 * Ho * 2 * Wo,), F32)
    lib.cvb_stem_dgrad(dz.data_ptr(), y.data_ptr(), coef.data_ptr(), wprep.data_ptr(), B, Ho, Wo, C0, dX.ptr, S())
    torch.cuda.synchronize()
    ref = F.conv_transpose2d(dy, w3.double(), stride=2, padding=1, output_padding=1)
    close(dX.check("stem_dgrad dX").view(B, 3, 2 * Ho, 2 * Wo), ref, rtol=1e-3, atol=1e-4 * float(ref.abs().max()), what="stem_dgrad")
    if C0 % 16:
        return
    w4 = bf(rnd(C0, 3, 4, 4, scale=0.3, seed=187))
    wp = w4.permute(0, 2, 3, 1).reshape(C0, 48).contiguous()  # columns (u*4 + v)*3 + ci
    dXp = Guarded((B * 3 * 4 * Ho * 4 * Wo,), F32)
    lib.cvb_patch_stem_dgrad(dz.data_ptr(), y.data_ptr(), coef.data_ptr(), wp.data_ptr(), B, Ho, Wo, C0, dXp.ptr, S())
    torch.cuda.synchronize()
    ref = F.conv_transpose2d(dy, w4.double(), stride=4, padding=1, output_padding=2)
    got = dXp.check("patch_stem_dgrad dX (every element written)").view(B, 3, 4 * Ho, 4 * Wo)
    close(got, ref, rtol=1e-3, atol=1e-4 * float(ref.abs().max()), what="patch_stem_dgrad")


@pytest.mark.parametrize("B,N,n_pos,C,cls", [(2, 49, 196, 72, True), (3, 196, 196, 40, False), (2, 63, 49, 200, True)])
def test_vit_tokens_write_set(lib, B, N, n_pos, C, cls):
    patch = bf(rnd(B * N, C, seed=191))
    pos = rnd(n_pos, C, seed=192)
    cv = rnd(C, seed=193)
    Sq = N + int(cls)
    out = Guarded((B * Sq, C), BF)
    lib.cvb_vit_tokens_interp_fwd(patch.data_ptr(), pos.data_ptr(), n_pos, cv.data_ptr() if cls else None, out.ptr, B, N, C, S())
    torch.cuda.synchronize()
    o = out.check("vit_tokens out").view(B, Sq, C)
    posr = torch.nn.functional.interpolate(pos.double()[None, None], size=(N, C), mode="bilinear", align_corners=False)[0, 0]
    close(o[:, int(cls):], patch.double().view(B, N, C) + posr, what="vit_tokens patch rows")
    if cls:
        same_bits(o[:, 0], cv.to(BF)[None].expand(B, C), "vit_tokens class token")
    dout = bf(rnd(B * Sq, C, seed=194))
    res = []
    for fill in ("zero", "prior"):
        dp = Guarded((B * N, C), BF)
        Pp, Pc = prior((n_pos, C), F32, seed=27), prior((C,), F32, seed=28)
        dpos = Guarded((n_pos, C), F32).fill(torch.zeros(n_pos, C) if fill == "zero" else Pp)
        dcls = Guarded((C,), F32).fill(torch.zeros(C) if fill == "zero" else Pc)
        lib.cvb_vit_tokens_interp_bwd(dout.data_ptr(), dp.ptr, dpos.ptr, n_pos, dcls.ptr if cls else None, B, N, C, S())
        torch.cuda.synchronize()
        dpos.check_bands("dpos")
        dcls.check_bands("dcls")
        res.append((dp.check("vit_tokens dpatch"), dpos.region(), dcls.region(), Pp, Pc))
    (dp0, p0, c0, _, _), (dp1, p1, c1, Pp, Pc) = res
    same_bits(dp1, dp0, "dpatch")
    same_bits(p1, Pp + p0, "dpos +=")
    same_bits(c1, Pc + c0 if cls else Pc, "dcls +=" if cls else "dcls untouched without a class token")
    same_bits(dp0, dout.view(B, Sq, C)[:, int(cls):].reshape(-1, C), "dpatch = dout rows")


def test_clip_edges_write_set(lib):
    B, S_, C, V = 3, 17, 72, 50
    g = torch.Generator("cuda").manual_seed(5)
    tokens = torch.randint(1, V - 1, (B, S_), device="cuda", generator=g)
    tokens[:, 5] = V - 1  # the end-of-text token: argmax
    table, pos = rnd(V, C, seed=201), rnd(S_, C, seed=202)
    out = Guarded((B * S_, C), BF)
    lib.cvb_embedding_fwd(tokens.data_ptr(), table.data_ptr(), pos.data_ptr(), out.ptr, B, S_, C, V, S())
    torch.cuda.synchronize()
    same_bits(out.check("embedding out"), (table[tokens] + pos).to(BF).view(-1, C), "embedding")
    dout = bf(rnd(B * S_, C, seed=203))
    Pt, Pp = prior((V, C), F32, seed=29), prior((S_, C), F32, seed=30)
    dtab, dpos = Guarded((V, C), F32).fill(Pt), Guarded((S_, C), F32).fill(Pp)
    lib.cvb_embedding_bwd(dout.data_ptr(), tokens.data_ptr(), dtab.ptr, dpos.ptr, B, S_, C, V, S())
    torch.cuda.synchronize()
    dtab.check_bands("dtable")
    dpos.check_bands("dpos")
    d3 = dout.double().view(B, S_, C)
    rt = torch.zeros(V, C, device="cuda", dtype=F64).index_add_(0, tokens.reshape(-1), d3.reshape(-1, C))
    close(dtab.region(), Pt.double() + rt, rtol=1e-5, atol=1e-5, what="dtable +=")
    close(dpos.region(), Pp.double() + d3.sum(0), rtol=1e-5, atol=1e-5, what="dpos +=")
    X = bf(rnd(B * S_, C, seed=204))
    go, gi = Guarded((B, C), BF), Guarded((B,), torch.int32)
    lib.cvb_eot_gather_fwd(X.data_ptr(), tokens.data_ptr(), B, S_, C, go.ptr, gi.ptr, S())
    torch.cuda.synchronize()
    idx = gi.check("eot idx")
    assert idx.tolist() == [5] * B
    same_bits(go.check("eot out"), X.view(B, S_, C)[:, 5], "eot gather")
    dgo = bf(rnd(B, C, seed=205))
    dX = Guarded((B * S_, C), BF)
    lib.cvb_eot_gather_bwd(dgo.data_ptr(), gi.ptr, B, S_, C, dX.ptr, S())
    torch.cuda.synchronize()
    dX.check_bands("eot dX")
    rows = torch.arange(B, device="cuda") * S_ + 5
    other = torch.ones(B * S_, dtype=torch.bool, device="cuda")
    other[rows] = False
    dx = dX.check("eot dX")
    same_bits(dx[rows], dgo, "eot dX gathered rows")
    assert not bool(dx[other].float().any()), "eot_gather_bwd writes zeros into the other rows"
    Y, inv = Guarded((B * S_, C), BF), Guarded((B * S_,), F32)
    lib.cvb_l2norm_fwd(X.data_ptr(), Y.ptr, inv.ptr, B * S_, C, 1e-12, S())
    DY = bf(rnd(B * S_, C, seed=206))
    DXn = Guarded((B * S_, C), BF)
    lib.cvb_l2norm_bwd(DY.data_ptr(), Y.ptr, inv.ptr, DXn.ptr, B * S_, C, S())
    torch.cuda.synchronize()
    x = X.double().requires_grad_(True)
    yn = torch.nn.functional.normalize(x, dim=-1)
    yn.backward(DY.double())
    close(Y.check("l2norm Y"), yn.detach(), what="l2norm Y")
    inv.check("l2norm inv")
    close(DXn.check("l2norm DX"), x.grad, what="l2norm DX")
    Tt = Guarded((C, B * S_), BF)
    lib.cvb_transpose_bf16(X.data_ptr(), Tt.ptr, B * S_, C, S())
    n = B * S_ * C
    Bf = rnd(n, seed=207)
    AO = Guarded((n,), BF)
    lib.cvb_add_bf16_f32(X.data_ptr(), Bf.data_ptr(), AO.ptr, n, S())
    torch.cuda.synchronize()
    same_bits(Tt.check("transpose"), X.t(), "transpose")
    close(AO.check("add_bf16_f32"), X.double().reshape(-1) + Bf.double(), what="add_bf16_f32")

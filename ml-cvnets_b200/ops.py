"""Thin Python wrappers over the C ABI (one function per kernel entry point).

Tensors are torch CUDA tensors used purely as device memory (allocation through the caching allocator, current stream);
every wrapper launches on ``torch.cuda.current_stream()`` and never synchronises.  2-D activation matrices are
``[M, C]`` bf16 (channels-last feature maps viewed as matrices).
"""
from __future__ import annotations

import ctypes
from typing import Optional, Sequence, Tuple

import torch

from . import _lib as L
from ._lib import (A_AFF, A_AFF_SILU, A_BNB, A_GN, A_RAW, A_SILU, E_GN_BWD, E_LIN_BWD, E_SILU, E_SILU_BWD, E_STORE,  # noqa: F401
                   ACT_GELU, ACT_HARDSIGMOID, ACT_HARDSWISH, ACT_RELU, ACT_SIGMOID, ACT_SILU,
                   PATCH_FOLD, PATCH_FOLD_T, PATCH_UNFOLD, PATCH_UNFOLD_T,
                   cvb_dw_bwd_args, cvb_dw_fwd_args, cvb_gemm_args, cvb_prep_desc, cvb_wgrad_args)

Tensor = torch.Tensor
launch_count = 0  # number of kernels launched through this module (bench.py reports it as gpu_launches)


def _p(t: Optional[Tensor]):
    return None if t is None else t.data_ptr()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _lib():
    return L.load()


# ---------------------------------------------------------------------------------------------------- side stream
# Weight-gradient GEMMs are off the critical path of the backward pass (their results are only needed by the optimizer), so the
# autograd functions issue them on a second stream: `side=True` forks from the current stream (everything enqueued so far is a
# dependency), and `join_side()` at the end of each backward makes the current stream wait for them.  Under CUDA-graph capture this
# becomes a parallel branch of the graph whose CTAs fill the tails of the main-branch kernels.  "on" is a testing hook: the reproducibility
# tests also run the step with every weight gradient on the current stream.
_SIDE = {"on": True, "streams": {}, "dirty": False, "held": []}


class _SideCtx:
    def __init__(self, active: bool):
        self.active = active and _SIDE["on"]

    def __enter__(self):
        if not self.active:
            return self
        main = torch.cuda.current_stream()
        dev = main.device
        side = _SIDE["streams"].get(dev)
        if side is None:
            side = _SIDE["streams"][dev] = torch.cuda.Stream(device=dev)
        side.wait_stream(main)
        self._cm = torch.cuda.stream(side)
        self._cm.__enter__()
        _SIDE["dirty"] = True
        return self

    def __exit__(self, *exc):
        if self.active:
            self._cm.__exit__(*exc)
        return False


def join_side():
    """Make the current stream wait for everything issued with ``side=True`` (call before the results are consumed)."""
    if _SIDE["dirty"]:
        main = torch.cuda.current_stream()
        side = _SIDE["streams"].get(main.device)
        if side is not None:
            main.wait_stream(side)
        _SIDE["dirty"] = False
    _SIDE["held"].clear()


def _hold(*tensors):
    """Keep the operands of side-stream work alive until join_side(): the caching allocator only knows about the stream a block was
    allocated on, so a tensor freed (name rebound) on the main stream while a queued side-stream kernel still reads it could be handed
    to a later main-stream allocation -- a write-after-read race, also between the parallel branches of a captured graph."""
    if _SIDE["dirty"]:
        _SIDE["held"].extend(t for t in tensors if t is not None)


def _count(n=1):
    global launch_count
    launch_count += n


def set_tc_enabled(on: bool) -> bool:
    """Testing hook: route prologue-free GEMMs to the wgmma kernel (default) or to the mma.sync kernel."""
    return bool(_lib().cvb_set_tc_enabled(int(on)))


def set_pdl_enabled(on: bool) -> bool:
    """Testing hook: programmatic dependent launch for every kernel (default) or plain stream-ordered launches."""
    return bool(_lib().cvb_set_pdl_enabled(int(on)))


# --------------------------------------------------------------------------------------------------------------- GEMM
# wide-layer policy: when the prologue would be re-applied by MANY N tiles (ViT / CLIP: K = 768 / 3072 under 18-24 N tiles) it is applied once
# by a pre-pass instead.  With 8 transform warps the in-kernel prologue won on every MobileViTv2 layer (same-box A/B: 12.47 -> 12.23 ms per
# step without the pre-pass), so the policy now needs N >= WIDE_N as well.
WIDE_K = 384
WIDE_N = 1024
# weight gradients: every 128-row block of dW (N / 128 CTAs per K block) re-applies the prologue to the SAME activation operand inside its transform
# warps.  For the LayerNorm-fused weight gradients of the ViT-B qkv_proj / ffn.1 (N = 2304 / 3072, 18 / 24 blocks) that repeated prologue costs
# far more than one pre-pass -> one pre-pass, then the RAW kernel.
WIDE_N_WGRAD = 1536


def pw_gemm(A: Tensor, W: Tensor, N: int, *, K: Optional[int] = None, a_mode: int = A_RAW, A2: Optional[Tensor] = None,
            a_p: Sequence[Optional[Tensor]] = (None, None, None), row_stats: Optional[Tuple[Tensor, Tensor]] = None,
            rows_per_sample: int = 0, bias: Optional[Tensor] = None, e_mode: int = E_STORE, Y: Optional[Tensor] = None,
            e_p: Sequence[Optional[Tensor]] = (None, None), R: Optional[Tensor] = None, out: Optional[Tensor] = None,
            col_stats: Optional[Tensor] = None, samp_stats: Optional[Tensor] = None, gn_ws: Optional[Tensor] = None) -> Tensor:
    """C[M,N] = epi(load(A)[M,K] @ W[N,K]^T + bias).  ``col_stats``/``samp_stats``: fp64 [2, *] accumulators (pre-zeroed)."""
    lib = _lib()
    M = A.shape[0]
    K = A.shape[1] if K is None else K
    if a_mode != A_RAW and K >= WIDE_K and N >= WIDE_N:
        # wide late-stage layer (small, L2-resident operand): apply the prologue once instead of once per N tile, then run the
        # prologue-free (wgmma) GEMM
        A = apply_load_mode(A, a_mode, K, A2=A2, a_p=a_p, row_stats=row_stats, rows_per_sample=rows_per_sample)
        a_mode, A2, a_p = A_RAW, None, (None, None, None)
        if e_mode != E_GN_BWD:  # the GroupNorm-backward epilogue reads the same per-sample statistics
            row_stats = None
    if out is None:
        out = torch.empty((M, N), device=A.device, dtype=torch.bfloat16)
    a = cvb_gemm_args()
    a.M, a.N, a.K = M, N, K
    a.A, a.lda = A.data_ptr(), A.stride(0)
    if A2 is not None:
        a.A2, a.lda2 = A2.data_ptr(), A2.stride(0)
    a.a_mode = a_mode
    a.a_p0, a.a_p1, a.a_p2 = _p(a_p[0]), _p(a_p[1]), _p(a_p[2] if len(a_p) > 2 else None)
    if row_stats is not None:
        a.row_mean, a.row_rstd = row_stats[0].data_ptr(), row_stats[1].data_ptr()
    a.rows_per_sample = rows_per_sample
    a.W, a.ldw = W.data_ptr(), W.stride(0)
    a.bias = _p(bias)
    a.e_mode = e_mode
    if Y is not None:
        a.Y, a.ldy = Y.data_ptr(), Y.stride(0)
    a.e_p0, a.e_p1 = _p(e_p[0]), _p(e_p[1])
    if R is not None:
        a.R, a.ldr = R.data_ptr(), R.stride(0)
    a.C, a.ldc, a.c_fp32 = out.data_ptr(), out.stride(0), int(out.dtype == torch.float32)
    if col_stats is not None:
        a.col_sum, a.col_sq = col_stats[0].data_ptr(), col_stats[1].data_ptr()
    if samp_stats is not None:
        a.samp_sum, a.samp_sq = samp_stats[0].data_ptr(), samp_stats[1].data_ptr()
    if gn_ws is not None:
        a.gn_ws = gn_ws.data_ptr()
    lib.cvb_pw_gemm(ctypes.byref(a), _stream())
    _count()
    return out


def apply_load_mode(A: Tensor, mode: int, K: int, *, A2: Optional[Tensor] = None, a_p: Sequence[Optional[Tensor]] = (None, None, None),
                    row_stats: Optional[Tuple[Tensor, Tensor]] = None, rows_per_sample: int = 0) -> Tensor:
    lib = _lib()
    M = A.shape[0]
    out = torch.empty((M, K), device=A.device, dtype=torch.bfloat16)
    p2 = a_p[2] if len(a_p) > 2 else None
    lib.cvb_apply_load_mode(A.data_ptr(), A.stride(0), _p(A2), A2.stride(0) if A2 is not None else 0, mode, _p(a_p[0]), _p(a_p[1]), _p(p2),
                            _p(row_stats[0]) if row_stats is not None else None, _p(row_stats[1]) if row_stats is not None else None,
                            rows_per_sample, out.data_ptr(), out.stride(0), M, K, _stream())
    _count()
    return out


def pw_wgrad(G: Tensor, A: Tensor, N: int, K: int, *, g_mode: int = A_RAW, G2: Optional[Tensor] = None,
             g_p: Sequence[Optional[Tensor]] = (None, None, None), a_mode: int = A_RAW,
             a_p: Sequence[Optional[Tensor]] = (None, None), row_stats: Optional[Tuple[Tensor, Tensor]] = None,
             rows_per_sample: int = 0, dW: Optional[Tensor] = None, dbias: Optional[Tensor] = None, side: bool = False) -> Tensor:
    """dW[N,K] (fp32, zero-initialised here unless given) += load(G)^T @ load(A).  ``side``: issue on the side stream (see join_side)."""
    lib = _lib()
    if dW is None:
        dW = torch.zeros((N, K), device=G.device, dtype=torch.float32)
    with _SideCtx(side):
        A0 = A
        if a_mode != A_RAW and K >= WIDE_K and N >= WIDE_N_WGRAD:
            A = apply_load_mode(A, a_mode, K, a_p=a_p, row_stats=row_stats, rows_per_sample=rows_per_sample)  # on the stream of the weight gradient
            a_mode, a_p, row_stats = A_RAW, (None, None), None
        a = cvb_wgrad_args()
        a.M, a.N, a.K = G.shape[0], N, K
        a.G, a.ldg, a.g_mode = G.data_ptr(), G.stride(0), g_mode
        if G2 is not None:
            a.G2, a.ldg2 = G2.data_ptr(), G2.stride(0)
        a.g_p0, a.g_p1, a.g_p2 = _p(g_p[0]), _p(g_p[1]), _p(g_p[2])
        a.A, a.lda, a.a_mode = A.data_ptr(), A.stride(0), a_mode
        a.a_p0, a.a_p1 = _p(a_p[0]), _p(a_p[1])
        if row_stats is not None:
            a.row_mean, a.row_rstd = row_stats[0].data_ptr(), row_stats[1].data_ptr()
        a.rows_per_sample = rows_per_sample
        a.dW, a.lddw = dW.data_ptr(), dW.stride(0)
        a.dbias = _p(dbias)
        lib.cvb_pw_wgrad(ctypes.byref(a), _stream())
        if side:
            _hold(G, G2, A, A0, dW, dbias)
    _count()
    return dW


# ---------------------------------------------------------------------------------------------------------- depthwise
def dw_fwd(X: Tensor, B: int, H: int, W: int, C: int, stride: int, Wt: Tensor, *, x_mode: int = A_RAW,
           x_p: Sequence[Optional[Tensor]] = (None, None), col_stats: Optional[Tensor] = None, dilation: int = 1, ksize: int = 3) -> Tensor:
    """Depthwise ksize x ksize conv (ksize 3 or 5, pad (ksize-1)/2 * dilation); ``Wt`` is tap-major fp32 [ksize*ksize, C]."""
    lib = _lib()
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    Y = torch.empty((B * Ho * Wo, C), device=X.device, dtype=torch.bfloat16)
    a = cvb_dw_fwd_args()
    a.B, a.H, a.W, a.C, a.stride = B, H, W, C, stride
    a.X, a.x_mode, a.x_p0, a.x_p1 = X.data_ptr(), x_mode, _p(x_p[0]), _p(x_p[1])
    a.Wt, a.Y, a.dilation, a.ksize = Wt.data_ptr(), Y.data_ptr(), int(dilation), int(ksize)
    if col_stats is not None:
        a.col_sum, a.col_sq = col_stats[0].data_ptr(), col_stats[1].data_ptr()
    lib.cvb_dw_fwd(ctypes.byref(a), _stream())
    _count()
    return Y


def dw_bwd(DZ: Tensor, X: Tensor, B: int, H: int, W: int, C: int, stride: int, Wt: Tensor, *, g_mode: int = A_RAW,
           Y2: Optional[Tensor] = None, g_p: Sequence[Optional[Tensor]] = (None, None, None), x_mode: int = A_RAW,
           x_p: Sequence[Optional[Tensor]] = (None, None), col_stats: Optional[Tensor] = None,
           dWt: Optional[Tensor] = None, dilation: int = 1, ksize: int = 3) -> Tuple[Tensor, Tensor]:
    """Returns (DX bf16 [B*H*W, C], dWt fp32 [ksize*ksize, C]); ``dWt`` if given must be zero-initialised (it is accumulated into)."""
    lib = _lib()
    DX = torch.empty((B * H * W, C), device=X.device, dtype=torch.bfloat16)
    if dWt is None:
        dWt = torch.zeros((ksize * ksize, C), device=X.device, dtype=torch.float32)
    a = cvb_dw_bwd_args()
    a.B, a.H, a.W, a.C, a.stride = B, H, W, C, stride
    a.DZ, a.Y2, a.g_mode = DZ.data_ptr(), _p(Y2), g_mode
    a.g_p0, a.g_p1, a.g_p2 = _p(g_p[0]), _p(g_p[1]), _p(g_p[2])
    a.X, a.x_mode, a.x_p0, a.x_p1 = X.data_ptr(), x_mode, _p(x_p[0]), _p(x_p[1])
    a.Wt, a.DX, a.dWt, a.dilation, a.ksize = Wt.data_ptr(), DX.data_ptr(), dWt.data_ptr(), int(dilation), int(ksize)
    if col_stats is not None:
        a.col_sum, a.col_sq = col_stats[0].data_ptr(), col_stats[1].data_ptr()
    lib.cvb_dw_bwd(ctypes.byref(a), _stream())
    _count()
    return DX, dWt


def im2col(x: Tensor, k: int, stride: int, pad: int, lda: Optional[int] = None) -> Tuple[Tensor, int, int]:
    """x: [B, Cin, H, W] logical (fp32 or bf16, any strides) -> bf16 patch matrix [B*Ho*Wo, lda], columns (u, v, ci), zero padded."""
    B, Cin, H, W = x.shape
    Ho, Wo = (H + 2 * pad - k) // stride + 1, (W + 2 * pad - k) // stride + 1
    lda = lda or (k * k * Cin + 7) // 8 * 8
    A = torch.empty((B * Ho * Wo, lda), device=x.device, dtype=torch.bfloat16)
    assert x.dtype in (torch.float32, torch.bfloat16)
    sn, sc, sh, sw = x.stride()
    _lib().cvb_im2col(x.data_ptr(), int(x.dtype == torch.float32), sn, sc, sh, sw, B, Cin, H, W, k, stride, pad, A.data_ptr(), lda, _stream())
    _count()
    return A, Ho, Wo


def col2im(dA: Tensor, B: int, Cin: int, H: int, W: int, k: int, stride: int, pad: int) -> Tensor:
    """adjoint of im2col for channels-last bf16: returns dX as the [B*H*W, Cin] matrix."""
    dX = torch.empty((B * H * W, Cin), device=dA.device, dtype=torch.bfloat16)
    _lib().cvb_col2im(dA.data_ptr(), dA.stride(0), B, Cin, H, W, k, stride, pad, dX.data_ptr(), _stream())
    _count()
    return dX


def embedding_fwd(tokens: Tensor, table: Tensor, pos: Optional[Tensor]) -> Tensor:
    B, S = tokens.shape
    V, C = table.shape
    out = torch.empty((B, S, C), device=table.device, dtype=torch.bfloat16)
    _lib().cvb_embedding_fwd(tokens.data_ptr(), table.data_ptr(), _p(pos), out.data_ptr(), B, S, C, V, _stream())
    _count()
    return out


def embedding_bwd(dout: Tensor, tokens: Tensor, dtable: Tensor, dpos: Optional[Tensor]) -> None:
    B, S = tokens.shape
    V, C = dtable.shape
    _lib().cvb_embedding_bwd(dout.data_ptr(), tokens.data_ptr(), dtable.data_ptr(), _p(dpos), B, S, C, V, _stream())
    _count()


def eot_gather_fwd(X: Tensor, tokens: Tensor):
    B, S, C = X.shape
    out = torch.empty((B, C), device=X.device, dtype=torch.bfloat16)
    idx = torch.empty((B,), device=X.device, dtype=torch.int32)
    _lib().cvb_eot_gather_fwd(X.data_ptr(), tokens.data_ptr(), B, S, C, out.data_ptr(), idx.data_ptr(), _stream())
    _count()
    return out, idx


def eot_gather_bwd(dout: Tensor, idx: Tensor, B: int, S: int, C: int) -> Tensor:
    dX = torch.empty((B, S, C), device=dout.device, dtype=torch.bfloat16)
    _lib().cvb_eot_gather_bwd(dout.data_ptr(), idx.data_ptr(), B, S, C, dX.data_ptr(), _stream())
    _count()
    return dX


def l2norm_fwd(X: Tensor, eps: float = 1e-12):
    M, C = X.shape
    Y = torch.empty_like(X)
    inv = torch.empty((M,), device=X.device, dtype=torch.float32)
    _lib().cvb_l2norm_fwd(X.data_ptr(), Y.data_ptr(), inv.data_ptr(), M, C, float(eps), _stream())
    _count()
    return Y, inv


def l2norm_bwd(DY: Tensor, Y: Tensor, inv: Tensor) -> Tensor:
    M, C = Y.shape
    DX = torch.empty_like(Y)
    _lib().cvb_l2norm_bwd(DY.data_ptr(), Y.data_ptr(), inv.data_ptr(), DX.data_ptr(), M, C, _stream())
    _count()
    return DX


def transpose_bf16(X: Tensor) -> Tensor:
    R, C = X.shape
    Y = torch.empty((C, R), device=X.device, dtype=torch.bfloat16)
    _lib().cvb_transpose_bf16(X.data_ptr(), Y.data_ptr(), R, C, _stream())
    _count()
    return Y


def add_bf16_f32(A: Optional[Tensor], Bf: Tensor) -> Tensor:
    out = torch.empty(Bf.shape, device=Bf.device, dtype=torch.bfloat16)
    _lib().cvb_add_bf16_f32(_p(A), Bf.data_ptr(), out.data_ptr(), Bf.numel(), _stream())
    _count()
    return out


def zs_class_embed(X: Tensor, perm: Tensor, Cl: int, M: int) -> Tensor:
    """fp32 [d, Cl] class table from the bf16 projected caption features X [R, d] (unnormalised); perm: int32 [Cl * M] row of caption m of
    class c at c * M + m."""
    R, d = X.shape
    if X.dtype != torch.bfloat16 or X.stride(1) != 1:
        raise ValueError("zs_class_embed: X must be bf16 with unit column stride")
    if perm.dtype != torch.int32 or perm.numel() != Cl * M or not perm.is_contiguous():
        raise ValueError(f"zs_class_embed: perm must be a contiguous int32 tensor of Cl * M = {Cl * M} elements")
    table = torch.empty((d, Cl), device=X.device, dtype=torch.float32)
    _lib().cvb_zs_class_embed(X.data_ptr(), X.stride(0), R, perm.data_ptr(), Cl, M, d, table.data_ptr(), _stream())
    _count()
    return table


def zs_logits_topk(img: Tensor, table: Tensor, scale: float = 100.0, targets: Optional[Tensor] = None, hits: Optional[Tensor] = None,
                   want_logits: bool = True) -> Optional[Tensor]:
    """fp32 logits [B, Cl] = scale * img @ table (None when ``want_logits`` is False); with ``targets`` (int64 [B]) and ``hits`` (int64 [2]),
    the top-1 / top-5 hits of the batch are added into ``hits`` on the device."""
    B, d = img.shape
    if img.dtype != torch.bfloat16 or img.stride(1) != 1:
        raise ValueError("zs_logits_topk: img must be bf16 with unit column stride")
    if table.dtype != torch.float32 or table.dim() != 2 or table.shape[0] != d or not table.is_contiguous():
        raise ValueError(f"zs_logits_topk: table must be a contiguous fp32 [{d}, classes] tensor, got {tuple(table.shape)} {table.dtype}")
    if (targets is None) != (hits is None):
        raise ValueError("zs_logits_topk: targets and hits go together")
    if targets is not None:
        if targets.dtype != torch.int64 or targets.shape != (B,) or not targets.is_contiguous():
            raise ValueError(f"zs_logits_topk: targets must be a contiguous int64 [{B}] tensor")
        if hits.dtype != torch.int64 or hits.numel() != 2 or not hits.is_contiguous():
            raise ValueError("zs_logits_topk: hits must be a contiguous int64 [2] tensor")
    Cl = table.shape[1]
    logits = torch.empty((B, Cl), device=img.device, dtype=torch.float32) if want_logits else None
    _lib().cvb_zs_logits_topk(img.data_ptr(), img.stride(0), table.data_ptr(), B, d, Cl, float(scale), _p(targets), _p(logits), _p(hits),
                              _stream())
    _count()
    return logits


def cls_metrics(logits: Tensor, target: Tensor, loss_sum: Tensor, counts: Tensor, row_loss: Tensor, ticket: Tensor,
                ignore_index: int = -1) -> None:
    """Validation metrics of one batch, added on the device (no host sync): ``loss_sum`` (fp64 [1]) += the summed cross entropy without
    label smoothing, ``counts`` (int64 [3]) += {top-1 hits, top-5 hits, counted rows}.  logits: bf16 [B, C] with unit column stride (a view
    of the classifier's padded output is fine); target: int64 [B], rows with ``ignore_index`` skipped.  Top-k rule: fewer than k classes with
    a logit strictly greater than the target's.  ``row_loss`` (fp32, >= B elements) and ``ticket`` (int32 [1], zero before the first call)
    are scratch."""
    if logits.dim() != 2 or logits.dtype != torch.bfloat16 or logits.stride(1) != 1 or logits.stride(0) < logits.shape[1]:
        raise ValueError("cls_metrics: logits must be a bf16 [B, C] matrix with unit column stride and row stride >= C")
    B, C = logits.shape
    if target.dtype != torch.int64 or tuple(target.shape) != (B,) or not target.is_contiguous():
        raise ValueError(f"cls_metrics: target must be a contiguous int64 [{B}] tensor")
    if loss_sum.dtype != torch.float64 or loss_sum.numel() != 1 or counts.dtype != torch.int64 or counts.numel() != 3:
        raise ValueError("cls_metrics: loss_sum must be fp64 [1] and counts int64 [3]")
    if row_loss.dtype != torch.float32 or row_loss.numel() < B or ticket.dtype != torch.int32 or ticket.numel() != 1:
        raise ValueError(f"cls_metrics: row_loss must be fp32 with >= {B} elements and ticket int32 [1]")
    _lib().cvb_cls_metrics(logits.data_ptr(), logits.stride(0), B, C, target.data_ptr(), int(ignore_index), loss_sum.data_ptr(),
                           counts.data_ptr(), row_loss.data_ptr(), ticket.data_ptr(), _stream())
    _count()


def ema_update(ema: Tensor, src: Tensor, momentum: float) -> None:
    """ema = ema * (1 - momentum) + momentum * src over two contiguous fp32 buffers of equal size (the reference's operation order)."""
    if ema.dtype != torch.float32 or src.dtype != torch.float32 or ema.numel() != src.numel() or not (ema.is_contiguous() and src.is_contiguous()):
        raise ValueError("ema_update: ema and src must be contiguous fp32 tensors of the same size")
    if not 0.0 <= float(momentum) <= 1.0:
        raise ValueError(f"ema_update: momentum {momentum} is outside [0, 1]")
    _lib().cvb_ema_update(ema.data_ptr(), src.data_ptr(), ema.numel(), float(momentum), _stream())
    _count()


def grad_accumulate(acc: Tensor, g: Tensor) -> None:
    """acc += g over two contiguous, 16-byte aligned fp32 buffers of equal size (bitwise torch's fp32 add): gradient accumulation."""
    if acc.dtype != torch.float32 or g.dtype != torch.float32 or acc.numel() != g.numel() or not (acc.is_contiguous() and g.is_contiguous()):
        raise ValueError("grad_accumulate: acc and g must be contiguous fp32 tensors of the same size")
    _lib().cvb_grad_accumulate(acc.data_ptr(), g.data_ptr(), acc.numel(), _stream())
    _count()


def patch_grid(H: int, W: int, ph: int, pw: int):
    """the Hn x Wn grid MobileViT-v1 tiles with patches: H, W rounded up to multiples of the patch (mobilevit_block.py:191-192)"""
    return -(-H // ph) * ph, -(-W // pw) * pw


def patch_permute(X: Tensor, B: int, H: int, W: int, ph: int, pw: int, inverse: bool = False, direction: Optional[int] = None) -> Tensor:
    """MobileViT-v1 unfold (feature-map rows [B*H*W, C] -> token rows [B*P*N, C]) / fold, or their transposes; ``direction`` is a
    PATCH_* constant and defaults to PATCH_FOLD if ``inverse`` else PATCH_UNFOLD.  Where H or W is not a multiple of the patch the tokens
    cover the bilinearly up-resized Hn x Wn map (``patch_grid``), as in the reference."""
    if direction is None:
        direction = PATCH_FOLD if inverse else PATCH_UNFOLD
    Hn, Wn = patch_grid(H, W, ph, pw)
    rows = B * (Hn * Wn if direction in (PATCH_UNFOLD, PATCH_FOLD_T) else H * W)
    out = torch.empty((rows, X.shape[1]), device=X.device, dtype=X.dtype)
    _lib().cvb_patch_permute(X.data_ptr(), out.data_ptr(), B, H, W, X.shape[1], ph, pw, int(direction), _stream())
    _count()
    return out


def concat2(A: Tensor, Bt: Tensor) -> Tensor:
    M, C1, C2 = A.shape[0], A.shape[1], Bt.shape[1]
    out = torch.empty((M, C1 + C2), device=A.device, dtype=torch.bfloat16)
    _lib().cvb_concat2(A.data_ptr(), Bt.data_ptr(), C1, C2, M, out.data_ptr(), _stream())
    _count()
    return out


def split2(G: Tensor, C1: int, C2: int) -> Tuple[Tensor, Tensor]:
    M = G.shape[0]
    da = torch.empty((M, C1), device=G.device, dtype=torch.bfloat16)
    db = torch.empty((M, C2), device=G.device, dtype=torch.bfloat16)
    _lib().cvb_split2(G.data_ptr(), C1, C2, M, da.data_ptr(), db.data_ptr(), _stream())
    _count()
    return da, db


def vit_tokens_interp_fwd(patch: Tensor, pos: Tensor, cls: Optional[Tensor], B: int, N: int, C: int) -> Tensor:
    """Token assembly with the positional table ``pos`` ([.., n_pos, C] fp32) linearly resampled to N rows (F.interpolate, align_corners=False)."""
    S = N + (1 if cls is not None else 0)
    out = torch.empty((B, S, C), device=patch.device, dtype=torch.bfloat16)
    _lib().cvb_vit_tokens_interp_fwd(patch.data_ptr(), pos.data_ptr(), pos.shape[-2], _p(cls), out.data_ptr(), B, N, C, _stream())
    _count()
    return out


def vit_tokens_interp_bwd(dout: Tensor, dpos: Tensor, dcls: Optional[Tensor], B: int, N: int, C: int) -> Tensor:
    """Adjoint of vit_tokens_interp_fwd: returns dpatch, adds into dpos ([n_pos, C] fp32) and dcls."""
    dpatch = torch.empty((B * N, C), device=dout.device, dtype=torch.bfloat16)
    _lib().cvb_vit_tokens_interp_bwd(dout.data_ptr(), dpatch.data_ptr(), dpos.data_ptr(), dpos.shape[-2], _p(dcls), B, N, C, _stream())
    _count()
    return dpatch


def stem_im2col(x: Tensor, mix: Optional[Tensor] = None) -> Tensor:
    """fp32 image [B,3,H,W] (any strides) -> bf16 patch matrix [B*(H/2)*(W/2), 32]; ``mix`` (device float[6]) folds mixup / cutmix in."""
    lib = _lib()
    B, C, H, W = x.shape
    assert C == 3 and x.dtype == torch.float32
    A = torch.empty((B * (H // 2) * (W // 2), 32), device=x.device, dtype=torch.bfloat16)
    sn, sc, sh, sw = x.stride()
    lib.cvb_stem_im2col(x.data_ptr(), sn, sc, sh, sw, B, H, W, A.data_ptr(), _p(mix), _stream())
    _count()
    return A


# ------------------------------------------------------------------------------------------------------------- BN / GN
def bn_finalize(stats: Tensor, count: float, gamma: Tensor, beta: Tensor, eps: float, momentum: float,
                running_mean: Optional[Tensor], running_var: Optional[Tensor], nbt: Optional[Tensor]) -> Tensor:
    """stats: fp64 [2, C].  Returns fp32 [4, C] = (mean, rstd, scale, shift); updates the running buffers in place."""
    lib = _lib()
    C = stats.shape[1]
    out = torch.empty((4, C), device=stats.device, dtype=torch.float32)
    lib.cvb_bn_finalize(stats[0].data_ptr(), stats[1].data_ptr(), float(count), _p(gamma), _p(beta), eps, momentum,
                        _p(running_mean), _p(running_var), _p(nbt), out[0].data_ptr(), out[1].data_ptr(), out[2].data_ptr(),
                        out[3].data_ptr(), C, _stream())
    _count()
    return out


def bn_eval_scale_shift(gamma: Tensor, beta: Tensor, running_mean: Tensor, running_var: Tensor, eps: float) -> Tensor:
    lib = _lib()
    C = running_mean.shape[0]
    out = torch.empty((4, C), device=running_mean.device, dtype=torch.float32)
    lib.cvb_bn_eval_scale_shift(_p(gamma), _p(beta), running_mean.data_ptr(), running_var.data_ptr(), eps, out[0].data_ptr(),
                                out[1].data_ptr(), out[2].data_ptr(), out[3].data_ptr(), C, _stream())
    _count()
    return out


def bn_bwd_finalize(stats: Tensor, count: float, gamma: Tensor, bn: Tensor, eval_mode: bool = False,
                    out: Optional[Tuple[Tensor, Tensor]] = None) -> Tuple[Tensor, Tensor]:
    """stats: fp64 [2, C] (sum dz, sum dz*y); bn: the [4, C] forward record.  Returns (dgb = (dgamma, dbeta) fp32 [C] each -- written into
    ``out`` when given, e.g. slices of the flat gradient buffer --, coef fp32 [3,C])."""
    lib = _lib()
    C = stats.shape[1]
    dgb = torch.empty((2, C), device=stats.device, dtype=torch.float32) if out is None else out
    coef = torch.empty((3, C), device=stats.device, dtype=torch.float32)
    lib.cvb_bn_bwd_finalize(stats[0].data_ptr(), stats[1].data_ptr(), float(count), _p(gamma), bn[0].data_ptr(), bn[1].data_ptr(),
                            int(eval_mode), dgb[0].data_ptr(), dgb[1].data_ptr(), coef[0].data_ptr(), coef[1].data_ptr(),
                            coef[2].data_ptr(), C, _stream())
    _count()
    return dgb, coef


def bn_apply(Y: Tensor, bn: Tensor, act: bool, R: Optional[Tensor] = None) -> Tensor:
    lib = _lib()
    M, C = Y.shape
    out = torch.empty_like(Y)
    lib.cvb_bn_apply(Y.data_ptr(), bn[2].data_ptr(), bn[3].data_ptr(), int(act), _p(R), out.data_ptr(), M, C, _stream())
    _count()
    return out


def bn_bwd_reduce(DOUT: Tensor, Y: Tensor, stats: Tensor, bn: Optional[Tensor] = None, act: bool = False, store_dz: bool = False):
    lib = _lib()
    M, C = Y.shape
    DZ = torch.empty_like(Y) if store_dz else None
    lib.cvb_bn_bwd_reduce(DOUT.data_ptr(), Y.data_ptr(), _p(bn[2]) if act else None, _p(bn[3]) if act else None, int(act), _p(DZ),
                          stats[0].data_ptr(), stats[1].data_ptr(), M, C, _stream())
    _count()
    return DZ


def gn_finalize(stats: Tensor, count: float, eps: float) -> Tensor:
    """stats fp64 [2, B] -> fp32 [2, B] (mean, rstd)."""
    lib = _lib()
    B = stats.shape[1]
    out = torch.empty((2, B), device=stats.device, dtype=torch.float32)
    lib.cvb_gn_finalize(stats[0].data_ptr(), stats[1].data_ptr(), float(count), eps, out[0].data_ptr(), out[1].data_ptr(), B, _stream())
    _count()
    return out


def gn_stats(X: Tensor, B: int, rows_per_sample: int, stats: Tensor):
    lib = _lib()
    lib.cvb_gn_stats(X.data_ptr(), X.stride(0), B, rows_per_sample, X.shape[1], stats[0].data_ptr(), stats[1].data_ptr(), _stream())
    _count()


def gn_bwd_apply(G: Tensor, X: Tensor, gn: Tensor, sstats: Tensor, count: float, B: int, rows_per_sample: int,
                 DRES: Optional[Tensor] = None, col_sum: Optional[Tensor] = None) -> Tensor:
    lib = _lib()
    DX = torch.empty_like(G)
    lib.cvb_gn_bwd_apply(G.data_ptr(), X.data_ptr(), gn[0].data_ptr(), gn[1].data_ptr(), sstats[0].data_ptr(), sstats[1].data_ptr(),
                         float(count), _p(DRES), DX.data_ptr(), B, rows_per_sample, G.shape[1], _p(col_sum), _stream())
    _count()
    return DX


# ---------------------------------------------------------------------------------------------------------- attention
def linattn_fwd(QKV: Tensor, B: int, H: int, W: int, d: int, patch: int = 2):
    """patch = 2: QKV is the folded feature map [B, H, W, ld] (2x2 patches by indexing); patch = 0: QKV is the unfolded [B, P=H, N=W, ld]."""
    lib = _lib()
    M = QKV.shape[0]
    Pp, N = (4, (H // 2) * (W // 2)) if patch == 2 else (H, W)
    O = torch.empty((M, d), device=QKV.device, dtype=torch.bfloat16)
    S = torch.empty((B, Pp, N), device=QKV.device, dtype=torch.float32)
    CTX = torch.empty((B, Pp, d), device=QKV.device, dtype=torch.float32)
    lib.cvb_linattn_fwd(QKV.data_ptr(), QKV.stride(0), B, H, W, d, patch, O.data_ptr(), O.stride(0), S.data_ptr(), CTX.data_ptr(), _stream())
    _count()
    return O, S, CTX


def linattn_bwd(QKV: Tensor, DO: Tensor, S: Tensor, CTX: Tensor, B: int, H: int, W: int, d: int, dbias: Optional[Tensor] = None,
                patch: int = 2) -> Tensor:
    lib = _lib()
    DQKV = torch.empty_like(QKV)
    lib.cvb_linattn_bwd(QKV.data_ptr(), QKV.stride(0), DO.data_ptr(), DO.stride(0), S.data_ptr(), CTX.data_ptr(), B, H, W, d, patch,
                        DQKV.data_ptr(), _p(dbias), _stream())
    _count()
    return DQKV


def linattn_cross_fwd(QKP: Tensor, QKVX: Tensor, B: int, Pp: int, Mp: int, N: int, d: int):
    """query/key from QKP [B*P*M, ld] (projection of x_prev), values from QKVX [B*P*N, ld] (projection of x)."""
    O = torch.empty((B * Pp * N, d), device=QKP.device, dtype=torch.bfloat16)
    S = torch.empty((B, Pp, Mp), device=QKP.device, dtype=torch.float32)
    CTX = torch.empty((B, Pp, d), device=QKP.device, dtype=torch.float32)
    _lib().cvb_linattn_cross_fwd(QKP.data_ptr(), QKP.stride(0), B, Pp, Mp, d, QKVX.data_ptr(), QKVX.stride(0), N, O.data_ptr(), O.stride(0),
                                 S.data_ptr(), CTX.data_ptr(), _stream())
    _count()
    return O, S, CTX


def linattn_cross_bwd(QKP: Tensor, QKVX: Tensor, DO: Tensor, S: Tensor, CTX: Tensor, B: int, Pp: int, Mp: int, N: int, d: int,
                      dbias: Optional[Tensor] = None):
    DQKP, DQKVX = torch.zeros_like(QKP), torch.zeros_like(QKVX)  # the kernel writes k/q columns of the first, v columns of the second
    _lib().cvb_linattn_cross_bwd(QKP.data_ptr(), QKP.stride(0), QKVX.data_ptr(), QKVX.stride(0), DO.data_ptr(), DO.stride(0), S.data_ptr(),
                                 CTX.data_ptr(), B, Pp, Mp, N, d, DQKP.data_ptr(), DQKVX.data_ptr(), _p(dbias), _stream())
    _count()
    return DQKP, DQKVX


def gn_bwd(V: Tensor, X: Tensor, gn: Tensor, gamma: Tensor, count: float, B: int, rows_per_sample: int, dgamma: Tensor, dbeta: Tensor, samp_ws: Tensor,
           DRES: Optional[Tensor] = None) -> Tensor:
    """Stand-alone GroupNorm(1, C) backward (two launches); dgamma/dbeta fp64 [C] accumulators, samp_ws zeroed fp64 [2, B]."""
    DX = torch.empty_like(V)
    _lib().cvb_gn_bwd(V.data_ptr(), X.data_ptr(), gn[0].data_ptr(), gn[1].data_ptr(), gamma.data_ptr(), float(count), _p(DRES), DX.data_ptr(), B,
                      rows_per_sample, V.shape[1], dgamma.data_ptr(), dbeta.data_ptr(), samp_ws.data_ptr(), _stream())
    _count(2)
    return DX


def mha_fwd(QKV: Tensor, B: int, S: int, H: int, head_dim: int, scale: float, attn_mask: Optional[Tensor] = None,
            key_padding_mask: Optional[Tensor] = None):
    """softmax(scale * Q K^T + masks) V for the packed projection QKV [B*S, 3*H*head_dim]; returns O [B*S, H*head_dim] and LSE [B,H,S]."""
    lib = _lib()
    O = torch.empty((B * S, H * head_dim), device=QKV.device, dtype=torch.bfloat16)
    LSE = torch.empty((B, H, S), device=QKV.device, dtype=torch.float32)
    lib.cvb_mha_fwd(QKV.data_ptr(), QKV.stride(0), B, S, H, head_dim, float(scale), _p(attn_mask), _p(key_padding_mask), O.data_ptr(),
                    O.stride(0), LSE.data_ptr(), _stream())
    _count()
    return O, LSE


def mha_bwd(QKV: Tensor, O: Tensor, DO: Tensor, LSE: Tensor, B: int, S: int, H: int, head_dim: int, scale: float,
            attn_mask: Optional[Tensor] = None, key_padding_mask: Optional[Tensor] = None) -> Tensor:
    lib = _lib()
    DQKV = torch.empty_like(QKV)
    lib.cvb_mha_bwd(QKV.data_ptr(), QKV.stride(0), O.data_ptr(), DO.data_ptr(), O.stride(0), LSE.data_ptr(), B, S, H, head_dim, float(scale),
                    _p(attn_mask), _p(key_padding_mask), DQKV.data_ptr(), DQKV.stride(0), _stream())
    _count()
    return DQKV


MHA_SMEM_MAX = 226 * 1024  # csrc/mha.cu: the dynamic shared memory one attention CTA may opt into


def mha_max_seq(head_dim: int, backward: bool = True) -> Optional[int]:
    """the longest sequence cvb_mha_fwd / cvb_mha_bwd take at ``head_dim``, or None (any length) for head_dim 64, whose long sequences run on
    the streaming kernels.  Every other head dim runs on the mma.sync kernels, which keep one head's Q, K, V (and dO, LSE, D in the backward)
    in shared memory, the head dim padded to 16 / 32 / 48 / 64 and S to a multiple of 64 (csrc/mha.cu mha_smem_bytes)."""
    if head_dim == 64:
        return None
    ld = next(p for p in (16, 32, 48, 64) if head_dim <= p) + 8
    per64 = 64 * ((4 * ld * 2 + 8) if backward else 3 * ld * 2)
    return MHA_SMEM_MAX // per64 * 64


def ln_bwd(V: Tensor, X: Tensor, ln: Tensor, gamma: Tensor, col_stats: Tensor, DRES: Optional[Tensor] = None,
           col_sum: Optional[Tensor] = None) -> Tensor:
    """One-pass LayerNorm backward; ``col_stats`` fp64 [2, C] receives (dbeta, dgamma) like the GN_BWD epilogue's col_stats."""
    M, C = V.shape
    DX = torch.empty_like(V)
    _lib().cvb_ln_bwd(V.data_ptr(), X.data_ptr(), ln[0].data_ptr(), ln[1].data_ptr(), gamma.data_ptr(), _p(DRES), DX.data_ptr(), M, C,
                      col_stats[1].data_ptr(), col_stats[0].data_ptr(), _p(col_sum), _stream())
    _count()
    return DX


def act_fwd(X: Tensor, kind: int) -> Tensor:
    Y = torch.empty_like(X)
    _lib().cvb_act_fwd(X.data_ptr(), Y.data_ptr(), X.numel(), kind, _stream())
    _count()
    return Y


def act_bwd(DY: Tensor, X: Tensor, kind: int) -> Tensor:
    DX = torch.empty_like(DY)
    _lib().cvb_act_bwd(DY.data_ptr(), X.data_ptr(), DX.data_ptr(), X.numel(), kind, _stream())
    _count()
    return DX


def se_scale_fwd(X: Tensor, S: Tensor, B: int, HW: int) -> Tensor:
    """Y[b,p,c] = X[b,p,c] * S[b,c]: X bf16 [B*HW, C] channels-last rows, S bf16 [B, C] (squeeze_excitation.py:82-83)."""
    Y = torch.empty_like(X)
    _lib().cvb_se_scale_fwd(X.data_ptr(), S.data_ptr(), Y.data_ptr(), B, HW, X.shape[1], _stream())
    _count()
    return Y


def se_scale_bwd(DY: Tensor, X: Tensor, S: Tensor, B: int, HW: int):
    """DX = DY * S (bf16) and DS[b,c] = sum_p DY * X (fp32 [B, C])."""
    DX = torch.empty_like(DY)
    DS = torch.zeros((B, X.shape[1]), device=X.device, dtype=torch.float32)
    _lib().cvb_se_scale_bwd(DY.data_ptr(), X.data_ptr(), S.data_ptr(), DX.data_ptr(), DS.data_ptr(), B, HW, X.shape[1], _stream())
    _count()
    return DX, DS


# ---------------------------------------------------------------------------------------------------------- dropout
_RNG = {}


def _rng_device(device) -> torch.device:
    dev = torch.device("cuda") if device is None else torch.device(device)
    return torch.device("cuda", torch.cuda.current_device()) if dev.index is None else dev  # "cuda" and "cuda:0" are ONE generator


def rng_seed(seed: Optional[int] = None, device=None) -> None:
    """(Re)seed the device-resident dropout generator {seed, counter}; default seed = torch.initial_seed() (utils/common_utils.py:68-71 seeds torch)."""
    dev = _rng_device(device)
    seed = torch.initial_seed() if seed is None else int(seed)
    _RNG[dev] = torch.tensor([seed & 0x7FFFFFFFFFFFFFFF, 0], device=dev, dtype=torch.int64)


def rng_next(device) -> Tensor:
    """Draw a 64-bit mask key on the device (int64 [1]); the counter advances on the device, also when replayed inside a CUDA graph."""
    dev = _rng_device(device)
    if dev not in _RNG:
        rng_seed(device=dev)
    key = torch.empty(1, device=dev, dtype=torch.int64)
    _lib().cvb_rng_next(_RNG[dev].data_ptr(), key.data_ptr(), _stream())
    _count()
    return key


def dropout_fwd(V: Tensor, R: Optional[Tensor], p: float, key: Tensor, p_row: float = 0.0, rows_per_sample: int = 0) -> Tensor:
    """Y = R + V * mask / (1 - p) [* per-sample stochastic-depth factor] on bf16 [M, C] (see cvb_dropout_fwd)."""
    M, C = V.shape
    Y = torch.empty_like(V)
    _lib().cvb_dropout_fwd(V.data_ptr(), _p(R), Y.data_ptr(), M, C, rows_per_sample, float(p), float(p_row), key.data_ptr(), _stream())
    _count()
    return Y


def dropout_bwd(DY: Tensor, p: float, key: Tensor, p_row: float = 0.0, rows_per_sample: int = 0) -> Tensor:
    M, C = DY.shape
    DV = torch.empty_like(DY)
    _lib().cvb_dropout_bwd(DY.data_ptr(), DV.data_ptr(), M, C, rows_per_sample, float(p), float(p_row), key.data_ptr(), _stream())
    _count()
    return DV


# ----------------------------------------------------------------------------------------------------- RangeAugment
def _ptr6(ts: Sequence[Optional[Tensor]]):
    return (ctypes.c_void_p * 6)(*[_p(t) for t in ts])


def na_plan(key: Tensor, B: int, enabled: int, tab: Tensor) -> Tensor:
    """Draw table fp32 [4 + 3 B] of one step (see cvb_na_plan); ``enabled`` bit k = brightness / contrast / noise."""
    _lib().cvb_na_plan(key.data_ptr(), B, int(enabled), tab.data_ptr(), _stream())
    _count()
    return tab


def na_noise(key: Tensor, B: int, H: int, W: int) -> Tensor:
    """The N(0, 1) field fp32 [B, 3, H, W] that the RangeAugment kernels recompute from ``key``."""
    eps = torch.empty((B, 3, H, W), device=key.device, dtype=torch.float32)
    _lib().cvb_na_noise(key.data_ptr(), B, H, W, eps.data_ptr(), _stream())
    _count()
    return eps


def na_stats(x: Tensor, mix: Optional[Tensor], key: Tensor, need_eps: bool, mu: Tensor) -> Tensor:
    """Per-plane means of the mixed image and of eps into fp64 ``mu`` [2, B * 3]."""
    B, _, H, W = x.shape
    _lib().cvb_na_stats(x.data_ptr(), _p(mix), key.data_ptr(), B, H, W, int(need_eps), mu[0].data_ptr(), mu[1].data_ptr(), _stream())
    _count()
    return mu


def na_compose(tab: Tensor, mu: Tensor, raw: Sequence[Optional[Tensor]], B: int, coef: Tensor) -> Tensor:
    """coef fp32 [B * 3, 3] = (A, Bc, C) per plane; ``raw`` = (_low, _high) x (brightness, contrast, noise), None where disabled."""
    _lib().cvb_na_compose(tab.data_ptr(), mu[0].data_ptr(), mu[1].data_ptr(), _ptr6(raw), B, coef.data_ptr(), _stream())
    _count()
    return coef


def na_apply(x: Tensor, mix: Optional[Tensor], key: Tensor, coef: Tensor, need_eps: bool, sq: Tensor) -> Tensor:
    """x_aug fp32 [B, 3, H, W]; writes the per-plane squared errors into fp64 ``sq`` [B, 3]."""
    B, _, H, W = x.shape
    Y = torch.empty_like(x)
    _lib().cvb_na_apply(x.data_ptr(), _p(mix), key.data_ptr(), coef.data_ptr(), B, H, W, int(need_eps), Y.data_ptr(), sq.data_ptr(), _stream())
    _count()
    return Y


def na_bwd_reduce(dY: Optional[Tensor], g_sq: Optional[Tensor], x: Tensor, mix: Optional[Tensor], key: Tensor, coef: Tensor, need_eps: bool,
                  red: Tensor) -> Tensor:
    B, _, H, W = x.shape
    _lib().cvb_na_bwd_reduce(_p(dY), _p(g_sq), x.data_ptr(), _p(mix), key.data_ptr(), coef.data_ptr(), B, H, W, int(need_eps), red.data_ptr(),
                             _stream())
    _count()
    return red


def na_param_grad(tab: Tensor, mu: Tensor, red: Tensor, raw: Sequence[Optional[Tensor]], B: int, grads: Sequence[Optional[Tensor]]):
    _lib().cvb_na_param_grad(tab.data_ptr(), mu[0].data_ptr(), mu[1].data_ptr(), red.data_ptr(), _ptr6(raw), B, _ptr6(grads), _stream())
    _count()


def na_loss_fwd(sq: Tensor, H: int, W: int, target: Tensor, step: Tensor, alpha: float, loss: Tensor, w_na: float = 1.0, ce: Optional[Tensor] = None,
                w_ce: float = 1.0, parts: Optional[Tensor] = None) -> Tensor:
    """loss (0-dim fp32) = w_na * L_na(sq) + w_ce * ce; ``parts`` fp32 [2] receives (ce, L_na)."""
    _lib().cvb_na_loss_fwd(sq.data_ptr(), sq.shape[0], H, W, target.data_ptr(), target.numel(), step.data_ptr(), float(alpha), float(w_na), _p(ce),
                           float(w_ce), loss.data_ptr(), _p(parts), _stream())
    _count()
    return loss


def na_loss_bwd(sq: Tensor, H: int, W: int, target: Tensor, step: Tensor, alpha: float, grad_out: Optional[Tensor], grad_scale: Optional[Tensor],
                w_na: float = 1.0, g_ce: Optional[Tensor] = None, w_ce: float = 1.0) -> Tensor:
    g_sq = torch.empty_like(sq)
    _lib().cvb_na_loss_bwd(sq.data_ptr(), sq.shape[0], H, W, target.data_ptr(), target.numel(), step.data_ptr(), float(alpha), float(w_na),
                           _p(grad_out), _p(grad_scale), g_sq.data_ptr(), _p(g_ce), float(w_ce), _stream())
    _count()
    return g_sq


def stem_dgrad(dz: Tensor, y: Tensor, coef: Tensor, Ws: Tensor, B: int, Ho: int, Wo: int) -> Tensor:
    """Stem input gradient fp32 [B, 3, 2 Ho, 2 Wo] from dz / y bf16 [B*Ho*Wo, C0], the BatchNorm-backward coef [3, C0] and the prepared weight."""
    C0 = dz.shape[1]
    dX = torch.empty((B, 3, 2 * Ho, 2 * Wo), device=dz.device, dtype=torch.float32)
    _lib().cvb_stem_dgrad(dz.data_ptr(), y.data_ptr(), coef.data_ptr(), Ws.data_ptr(), B, Ho, Wo, C0, dX.data_ptr(), _stream())
    _count()
    return dX


def patch_stem_dgrad(dz: Tensor, y: Tensor, coef: Tensor, Wp: Tensor, B: int, Ho: int, Wo: int) -> Tensor:
    """Input gradient of the ViT conv stem's 4x4 stride-4 pad-1 conv, fp32 NCHW [B, 3, 4 Ho, 4 Wo], from dz / y bf16 [B*Ho*Wo, C0], the
    BatchNorm-backward coef [3, C0] and the prepared patch-order weight [C0, 48]."""
    C0 = dz.shape[1]
    if not (dz.is_contiguous() and y.is_contiguous() and coef.is_contiguous() and tuple(Wp.shape) == (C0, 48) and Wp.is_contiguous()):
        raise ValueError("patch_stem_dgrad: dz / y [B*Ho*Wo, C0], coef [3, C0] and the weight [C0, 48] must be contiguous")
    dX = torch.empty((B, 3, 4 * Ho, 4 * Wo), device=dz.device, dtype=torch.float32)
    _lib().cvb_patch_stem_dgrad(dz.data_ptr(), y.data_ptr(), coef.data_ptr(), Wp.data_ptr(), B, Ho, Wo, C0, dX.data_ptr(), _stream())
    _count()
    return dX


def ln_stats(X: Tensor, eps: float) -> Tensor:
    """per-token LayerNorm statistics of a bf16 [M, C] matrix -> fp32 [2, M] (mean, rstd)."""
    lib = _lib()
    M, C = X.shape
    out = torch.empty((2, M), device=X.device, dtype=torch.float32)
    lib.cvb_ln_stats(X.data_ptr(), X.stride(0), M, C, float(eps), out[0].data_ptr(), out[1].data_ptr(), _stream())
    _count()
    return out


# --------------------------------------------------------------------------------------------------------------- misc
def global_pool_fwd(X: Tensor, B: int, HW: int) -> Tensor:
    lib = _lib()
    C = X.shape[1]
    out = torch.empty((B, C), device=X.device, dtype=torch.bfloat16)
    lib.cvb_global_pool_fwd(X.data_ptr(), B, HW, C, out.data_ptr(), _stream())
    _count()
    return out


def global_pool_bwd(DOUT: Tensor, B: int, HW: int) -> Tensor:
    lib = _lib()
    C = DOUT.shape[1]
    DX = torch.empty((B * HW, C), device=DOUT.device, dtype=torch.bfloat16)
    lib.cvb_global_pool_bwd(DOUT.data_ptr(), B, HW, C, DX.data_ptr(), _stream())
    _count()
    return DX


def ce_fwd(logits: Tensor, C: int, target: Tensor, ignore_index: int, smoothing: float, mix: Optional[Tensor] = None,
           logit_scale: Optional[Tensor] = None):
    """logits: bf16 [B, ld] (C valid columns).  Returns (loss fp32 [1], lse fp32 [B], n_valid fp32 [1])."""
    B = logits.shape[0]
    lse = torch.empty(B, device=logits.device, dtype=torch.float32)
    out = torch.empty(2, device=logits.device, dtype=torch.float32)
    _lib().cvb_ce_fwd(logits.data_ptr(), logits.stride(0), B, C, target.data_ptr(), int(ignore_index), float(smoothing), lse.data_ptr(),
                      out[0:1].data_ptr(), out[1:2].data_ptr(), _p(mix), _p(logit_scale), _stream())
    _count()
    return out[0:1], lse, out[1:2]


def ce_bwd(logits: Tensor, C: int, target: Tensor, ignore_index: int, smoothing: float, lse: Tensor, n_valid: Tensor, gout: Optional[Tensor],
           gscale: Optional[Tensor], ldd: int, mix: Optional[Tensor] = None, logit_scale: Optional[Tensor] = None,
           dlogit_scale: Optional[Tensor] = None) -> Tensor:
    B = logits.shape[0]
    d = torch.empty((B, ldd), device=logits.device, dtype=torch.bfloat16)
    _lib().cvb_ce_bwd(logits.data_ptr(), logits.stride(0), B, C, target.data_ptr(), int(ignore_index), float(smoothing), lse.data_ptr(),
                      n_valid.data_ptr(), _p(gout), _p(gscale), d.data_ptr(), ldd, _p(mix), _p(logit_scale), _p(dlogit_scale), _stream())
    _count()
    return d


def pw_wgrad_side(G: Tensor, A: Tensor, N: int, K: int, **kw) -> Tensor:
    """pw_wgrad on the side stream (the caller joins with join_side() before the result is consumed)."""
    return pw_wgrad(G, A, N, K, side=True, **kw)


def unprep_grad(src: Tensor, rows: int, cols: int, lds: int, kind: int, rot: int = 0, side: bool = False, out: Optional[Tensor] = None) -> Tensor:
    lib = _lib()
    dst = torch.empty((rows, cols) if kind != PreparedWeights.KIND_VECTOR_F32 else (rows,), device=src.device, dtype=torch.float32) if out is None else out
    assert dst.is_contiguous() and dst.numel() == rows * (cols if kind != PreparedWeights.KIND_VECTOR_F32 else 1)
    with _SideCtx(side):
        lib.cvb_unprep_grad(src.data_ptr(), dst.data_ptr(), rows, cols, lds, kind, rot, _stream())
        if side:
            _hold(src, dst)
    _count()
    return dst


_WEIGHTS_GENERATION = [0]


def invalidate_prepared_weights() -> None:
    """Tell every PreparedWeights cache that parameters may have changed WITHOUT a Tensor._version bump (raw-pointer kernels such as
    cvb_adamw_step, optimizer updates replayed inside a CUDA graph): the next eval-mode forward refreshes its kernel-layout copies."""
    _WEIGHTS_GENERATION[0] += 1


class PreparedWeights:
    """Kernel-layout copies of a module's fp32 parameters, refreshed by ONE batched launch (cvb_prep_weights).

    The parameters stay ordinary ``nn.Parameter``s owned by PyTorch (state_dict / optimizer / DDP / EMA see nothing
    new, SURVEY.md 8b); these buffers are a cache keyed on the parameters' ``_version`` and storage address.
    """

    # the layout kinds of cvb_prep_weights / cvb_unprep_grad (CVB_PREP_* in the header)
    KIND_ROWMAJOR, KIND_TRANSPOSED, KIND_TAPMAJOR_F32 = L.PREP_ROWMAJOR, L.PREP_TRANSPOSED, L.PREP_TAPMAJOR_F32
    KIND_VECTOR_F32, KIND_PATCH, KIND_PATCH_T = L.PREP_VECTOR_F32, L.PREP_PATCH, L.PREP_PATCH_T

    def __init__(self):
        self._entries = []  # (param, dst, rows, cols, ldd, dst_rows, kind, rot)
        self._table = None
        self._key = None
        self._versions = None
        self._forced_last = False
        self._max_elems = 1

    def add(self, param: Tensor, kind: int, *, rot: int = 0, ldd: Optional[int] = None, dst_rows: Optional[int] = None) -> int:
        p2 = param.reshape(param.shape[0], -1) if param.dim() > 1 else param.reshape(-1, 1)
        rows, cols = p2.shape
        self._entries.append([param, None, rows, cols, ldd, dst_rows, kind, rot])
        self._table = None
        return len(self._entries) - 1

    def _alloc(self, device):
        for e in self._entries:
            param, _, rows, cols, ldd, dst_rows, kind, rot = e
            if kind in (self.KIND_ROWMAJOR, self.KIND_PATCH):
                ldd = ldd or (cols + 7) // 8 * 8
                dst_rows = dst_rows or rows
                dst = torch.empty((dst_rows, ldd), device=device, dtype=torch.bfloat16)
            elif kind in (self.KIND_TRANSPOSED, self.KIND_PATCH_T):
                ldd = ldd or (rows + 7) // 8 * 8
                dst_rows = dst_rows or (cols + 7) // 8 * 8 if kind == self.KIND_PATCH_T else (dst_rows or cols)
                dst = torch.empty((dst_rows, ldd), device=device, dtype=torch.bfloat16)
            elif kind == self.KIND_TAPMAJOR_F32:
                ldd, dst_rows = rows, cols
                dst = torch.empty((cols, rows), device=device, dtype=torch.float32)
            else:
                dst_rows = dst_rows or rows
                ldd = 1
                dst = torch.empty((dst_rows,), device=device, dtype=torch.float32)
            e[1], e[4], e[5] = dst, ldd, dst_rows
            self._max_elems = max(self._max_elems, dst.numel())

    def get(self, idx: int) -> Tensor:
        return self._entries[idx][1]

    def prepare(self, force: bool = True):
        """Refresh all kernel-layout copies.  ``force=False`` skips the launch when no parameter changed."""
        if not self._entries:
            return
        device = self._entries[0][0].device
        key = tuple(e[0].data_ptr() for e in self._entries) + (device,)
        versions = tuple(e[0]._version for e in self._entries)
        if self._table is None or key != self._key:
            if self._entries[0][1] is None or self._entries[0][1].device != device:
                self._alloc(device)
            descs = (cvb_prep_desc * len(self._entries))()
            for i, (param, dst, rows, cols, ldd, dst_rows, kind, rot) in enumerate(self._entries):
                assert param.dtype == torch.float32 and param.is_contiguous(), "parameters must be contiguous fp32"
                descs[i] = cvb_prep_desc(param.data_ptr(), dst.data_ptr(), rows, cols, ldd, dst_rows, kind, rot)
            raw = torch.frombuffer(bytearray(bytes(descs)), dtype=torch.uint8)
            self._table = raw.to(device)
            self._key = key
            self._versions = None
        versions = versions + (_WEIGHTS_GENERATION[0],)
        # eval-mode callers pass force=False: skip only if nothing can have changed -- same versions, same generation, and the previous
        # refresh was not a training-mode one (a training forward refreshes BEFORE that step's optimizer update)
        if not force and versions == self._versions and not self._forced_last:
            return
        _lib().cvb_prep_weights(self._table.data_ptr(), len(self._entries), int(self._max_elems), _stream())
        _count()
        self._versions = versions
        self._forced_last = bool(force)

    def refresh(self):
        """Refresh all kernel-layout copies now, as an eval-mode forward would: later ``prepare(force=False)`` calls skip until a parameter
        changes (engine.EvalStep refreshes eagerly so that its captured forwards contain no refresh)."""
        self.prepare(force=True)
        self._forced_last = False

"""torch.autograd.Functions of the hot-path modules: each forward/backward is a fixed sequence of C-ABI kernel launches.

Design (DESIGN.md section 3): activations are bf16 channels-last matrices [M=B*H*W, C]; a conv writes its PRE-BatchNorm
output once together with fp64 per-channel sum / sum-of-squares; a tiny finalize kernel turns them into scale/shift; the
CONSUMER applies scale/shift(+SiLU) while loading.  The pre-BN tensors are exactly what the backward needs, so nothing is
stored twice.  Module boundaries materialise real tensors so every module stays a drop-in ``nn.Module``.

Reference semantics restated per function; citations are relative to the reference checkout.
"""
from __future__ import annotations

from types import SimpleNamespace

import torch

from . import ops
from .workspace import Arena
from .ops import A_AFF, A_AFF_SILU, A_BNB, A_GN, A_RAW, A_SILU, E_GN_BWD, E_SILU_BWD, E_STORE
from .ops import PreparedWeights as PW

BF16 = torch.bfloat16


# ------------------------------------------------------------------------------------------------------------ helpers
def to_bf16_cl(x: torch.Tensor) -> torch.Tensor:
    """bf16 + channels_last (a no-op between our own modules).  Dtype/layout glue, not compute."""
    if x.dtype != BF16:
        x = x.to(BF16)
    if not x.is_contiguous(memory_format=torch.channels_last):
        x = x.contiguous(memory_format=torch.channels_last)
    return x


def as_2d(x: torch.Tensor) -> torch.Tensor:
    B, C, H, W = x.shape
    return x.permute(0, 2, 3, 1).reshape(B * H * W, C)


def to_4d(y: torch.Tensor, B: int, H: int, W: int) -> torch.Tensor:
    return y.view(B, H, W, y.shape[1]).permute(0, 3, 1, 2)


def bn_cfg(bn_module) -> SimpleNamespace:
    """Reads nn.BatchNorm2d state at call time (momentum may be annealed: cvnets/layers/normalization_layers.py:91-100)."""
    assert bn_module.momentum is not None, "cumulative-average BatchNorm (momentum=None) is not implemented"
    return SimpleNamespace(running_mean=bn_module.running_mean, running_var=bn_module.running_var,
                           nbt=bn_module.num_batches_tracked, momentum=float(bn_module.momentum), eps=float(bn_module.eps),
                           batch_stats=bool(bn_module.training or bn_module.running_mean is None))


def _bn_forward(stats, count, gamma, beta, c):
    if c.batch_stats:
        return ops.bn_finalize(stats, count, gamma, beta, c.eps, c.momentum, c.running_mean, c.running_var, c.nbt)
    return ops.bn_eval_scale_shift(gamma, beta, c.running_mean, c.running_var, c.eps)


class LazyBN:
    """A module output handed to the NEXT hot-path module still PRE-BatchNorm (DESIGN.md "lazy module boundaries").

    The producer skips its ``bn_apply`` pass and returns the pre-BN tensor tagged with this record; the consumer applies
    ``scale * y + shift`` (+ SiLU) as the load mode of its first kernel and, in the backward, its input-gradient kernel emits
    dz (the gradient w.r.t. the BatchNorm output, through the activation) together with the BatchNorm-backward sums
    (sum dz, sum dz*y) into ``stats`` -- so the producer needs no ``bn_bwd_reduce`` pass either.  Only the model assembler wires this
    (both neighbours must be ours); a module called on its own always materialises its output."""
    __slots__ = ("bn", "act", "stats")

    def __init__(self, bn, act):
        self.bn, self.act, self.stats = bn, bool(act), None


def _lazy_modes(lz):
    """(load mode, input-gradient epilogue, their parameters) of a module input: the producer's BatchNorm (+SiLU) when it is lazy, else raw."""
    if lz is None:
        return A_RAW, E_STORE, (None, None)
    return (A_AFF_SILU if lz.act else A_AFF), (E_SILU_BWD if lz.act else ops.E_LIN_BWD), (lz.bn[2], lz.bn[3])


def _bn_out_grad(lz_out, D, dout, y, bn, act):
    """(dz, sums) of a module output y -> BatchNorm [-> SiLU if ``act``] given its gradient ``dout``: dz is the gradient w.r.t. the BatchNorm
    output and sums the BatchNorm-backward sums (sum dz, sum dz*y).  A lazy output's consumer already took dout through the activation and
    wrote the sums."""
    if lz_out is not None:
        assert lz_out.stats is not None, "lazy module output was consumed by a module that does not know the protocol"
        return dout, lz_out.stats
    sums = D.ar.f64(2, y.shape[1])
    dz = ops.bn_bwd_reduce(dout, y, sums, bn, act=act, store_dz=act)
    return (dz if act else dout), sums


def _ws_of(cfg, params):
    """The module's StepWorkspace if gradients are to be written in place (inside TrainStep, every parameter registered), else None."""
    ws = getattr(cfg, "ws", None)
    if ws is None or not ws.active:
        return None
    return ws if all(ws.has(p) for p in params) else None


def _arena(cfg, kind: str, ws, device) -> Arena:
    """Scratch of one forward ("fwd") or backward ("bwd") of the module behind ``cfg``, sized by what its earlier calls carved (the
    record ``cfg.arena_<kind>``): a slice of the step arena when ``ws`` is given, else zeroed per call."""
    rec = vars(cfg).setdefault("arena_" + kind, [0, 0])
    return ws.arena((id(cfg), kind), rec) if ws is not None else Arena(rec, device)


def _fwd_arena(cfg, device, kind: str = "fwd") -> Arena:
    """fp64 statistics accumulators of one forward: one memset per module, or a slice of the step arena (no launch at all).  ``kind``
    "rfwd": a forward recomputed inside the backward, which must not reuse the slice the step's forward already carved."""
    ws = getattr(cfg, "ws", None)
    return _arena(cfg, kind, ws if ws is not None and ws.active else None, device)


class _Dst:
    """Where the parameter gradients of one module backward go.

    Workspace mode (inside ``engine.TrainStep``): straight into the flat gradient buffer -- ``p.grad`` is a view of it -- and the autograd
    function returns ``None`` for the parameters (no AccumulateGrad kernels, no gather for the optimizer / all-reduce).  Otherwise: fresh
    slices of a per-call arena, returned to autograd as usual (what a plain ``loss.backward()`` on the drop-in modules gets)."""

    def __init__(self, cfg, params, device, use_ws: bool):
        self.params = list(params)
        self.ws = _ws_of(cfg, self.params) if use_ws else None
        self.key = (id(cfg), "bwd")
        self.ar = _arena(cfg, "bwd", self.ws, device)
        self.grads = [None] * len(self.params)
        self.late = []

    def mat(self, i: int, rows: int, cols: int) -> torch.Tensor:
        """zeroed fp32 [rows, cols] accumulator that IS the gradient of params[i] (same memory layout)."""
        if self.ws is not None:
            return self.ws.gview(self.params[i]).view(rows, cols)
        v = self.ar.f32(rows, cols)
        self.grads[i] = v.view(self.params[i].shape)
        return v

    def padded(self, i: int, rows: int, cols: int, npad: int) -> torch.Tensor:
        """zeroed fp32 [npad, cols] accumulator whose first ``rows`` rows are the gradient of params[i] ([rows, cols]; the kernel writes
        ``npad`` >= ``rows`` rows).  Padded rows only outside workspace mode: the scratch is sliced, not copied, into the gradient."""
        if npad == rows:
            return self.mat(i, rows, cols)
        assert self.ws is None, "padded gradient rows cannot be written into the flat gradient buffer"
        v = self.ar.f32(npad, cols)
        self.grads[i] = v[:rows].view(self.params[i].shape)
        return v

    def bn_bwd(self, stats, count, gamma, bn, eval_mode: bool, i: int, j: int) -> torch.Tensor:
        """BatchNorm-backward finalize: writes (dgamma, dbeta) as the gradients of params i, j and returns the input-gradient coefficients."""
        out = (self.ws.gview(self.params[i]), self.ws.gview(self.params[j])) if self.ws is not None else None
        dgb, coef = ops.bn_bwd_finalize(stats, count, gamma, bn, eval_mode=eval_mode, out=out)
        if self.ws is None:
            self.grads[i], self.grads[j] = dgb[0], dgb[1]
        return coef

    def unprep(self, i: int, src, rows: int, cols: int, lds: int, kind: int, rot: int = 0, side: bool = False):
        """kernel-layout gradient (rotated / padded / tap-major) -> the parameter's own layout."""
        out = self.ws.gview(self.params[i]).view((rows, cols) if kind != PW.KIND_VECTOR_F32 else (rows,)) if self.ws is not None else None
        g = ops.unprep_grad(src, rows, cols, lds, kind, rot=rot, side=side, out=out)
        if self.ws is None:
            self.grads[i] = g.view(self.params[i].shape)

    def late64(self, i: int, v64: torch.Tensor):
        """fp64 accumulator that is a gradient: converted after the last kernel that accumulates into it."""
        self.late.append((i, v64))

    def finish(self):
        if self.ws is not None:
            self.ws.scatter64(self.key, [(v, self.ws.gview(self.params[i]).view(v.shape)) for i, v in self.late])
            self.ws.unit_done(self.params)
            return (None,) * len(self.params)
        if self.late:
            self.ar.cast()
            for i, v in self.late:
                self.grads[i] = self.ar.as_f32(v).view(self.params[i].shape)
        return tuple(self.grads)


# ==================================================================================================================
# Stem: ConvLayer2d(3 -> C0, k3, s2) + BN + SiLU  (cvnets/models/classification/mobilevit_v2.py:37-45)
# ==================================================================================================================
class StemFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cfg, w, gamma, beta):
        B, _, H, W = x.shape
        C0 = w.shape[0]
        if H % 2 or W % 2:
            raise NotImplementedError("stem: odd H or W (the reference's 3x3/s2/p1 conv gives ceil(H/2)) is not implemented")
        Ho, Wo = H // 2, W // 2
        M = B * Ho * Wo
        xin = x if x.dtype == torch.float32 else x.float()
        ws = getattr(cfg, "ws", None)
        # batch mixing rides in the gather (TrainStep.set_mix), unless the input is the augmentor's output, which is already mixed
        mix = ws.mix if (ws is not None and ws.active and not getattr(x, "_cvb_premixed", False)) else None
        A0 = ops.stem_im2col(xin, mix=mix)
        Ws = cfg.prep.get(cfg.i_w)
        st = _fwd_arena(cfg, x.device).f64(2, C0)
        y = ops.pw_gemm(A0, Ws, C0, col_stats=st if cfg.bn.batch_stats else None)
        bn = _bn_forward(st, M, gamma, beta, cfg.bn)
        ctx.lz_out = cfg.last_lazy = LazyBN(bn, True) if cfg.lazy_out else None
        out = y if cfg.lazy_out else ops.bn_apply(y, bn, act=True)
        ctx.cfg, ctx.dims, ctx.ev = cfg, (B, Ho, Wo, C0, M), (not cfg.bn.batch_stats,)
        ctx.saved = (A0, y, bn, Ws)
        ctx.plist = cfg.plist
        ctx.save_for_backward(gamma)
        return to_4d(out, B, Ho, Wo)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        B, Ho, Wo, C0, M = ctx.dims
        A0, y, bn, Ws = ctx.saved
        (gamma,) = ctx.saved_tensors
        g2 = as_2d(to_bf16_cl(gout))
        D = _Dst(cfg, ctx.plist, g2.device, True)
        dz, sd = _bn_out_grad(ctx.lz_out, D, g2, y, bn, True)
        coef = D.bn_bwd(sd, M, gamma, bn, ctx.ev[0], 1, 2)
        dW = ops.pw_wgrad_side(dz, A0, C0, 32, g_mode=A_BNB, G2=y, g_p=coef, dW=D.ar.f32(C0, 32))
        D.unprep(0, dW, C0, 27, 32, PW.KIND_ROWMAJOR, side=True)
        # the image's gradient exists only when something upstream learns (the RangeAugment sampler parameters)
        dx = ops.stem_dgrad(dz, y, coef, Ws, B, Ho, Wo) if ctx.needs_input_grad[0] else None
        ops.join_side()
        return (dx, None) + D.finish()


# ==================================================================================================================
# RangeAugment (cvnets/neural_augmentor/neural_aug.py:214-236 with DistributionNeuralAugmentor's UniformSamplers) and its loss
# (loss_fn/neural_augmentation.py:178-218).  Kernels and draw layout: csrc/neural_aug.cu.
# ==================================================================================================================
class NeuralAugmentFn(torch.autograd.Function):
    """(x, cfg, *raw) -> (x_aug fp32 [B, 3, H, W], sq fp64 [B, 3] = per-(sample, channel) sum of (x_aug - x_mix)^2).

    ``raw`` are the enabled samplers' (_low, _high) parameters in brightness, contrast, noise order; ``cfg.enabled`` says which.  Inside
    TrainStep the image is first mixed as ``ws.mix`` says (on the fly, in every kernel that reads it), so the augmentor, the stem and the
    PSNR loss all see the mixed image, as the reference's training_engine.py:236-238 does."""

    @staticmethod
    def forward(ctx, x, cfg, *raw):
        B, C, H, W = x.shape
        if C != 3:
            raise NotImplementedError(f"RangeAugment: {C}-channel input (the kernels take RGB images)")
        x = x.float().contiguous()
        ws = _ws_of(cfg, raw)
        mix = ws.mix if ws is not None else None
        key = ops.rng_next(x.device)
        full = [None] * 6
        it = iter(raw)
        for k in range(3):
            if cfg.enabled >> k & 1:
                full[2 * k], full[2 * k + 1] = next(it), next(it)
        fa = _fwd_arena(cfg, x.device)
        tab, mu, coef, sq = fa.f32(4 + 3 * B), fa.f64(2, 3 * B), fa.f32(3 * B, 3), fa.f64(B, 3)
        need_eps = bool(cfg.enabled & 4)
        ops.na_plan(key, B, cfg.enabled, tab)
        ops.na_stats(x, mix, key, need_eps, mu)
        ops.na_compose(tab, mu, full, B, coef)
        y = ops.na_apply(x, mix, key, coef, need_eps, sq)
        ctx.cfg, ctx.saved = cfg, (x, mix, key, tab, mu, coef, full, need_eps)
        ctx.plist = list(raw)
        ctx.set_materialize_grads(False)  # an output without a gradient arrives as None (no zero tensor is filled); the kernel skips its term
        return y, sq

    @staticmethod
    def backward(ctx, g_y, g_sq):
        x, mix, key, tab, mu, coef, full, need_eps = ctx.saved
        B = x.shape[0]
        D = _Dst(ctx.cfg, ctx.plist, x.device, True)
        red = D.ar.f64(3 * B, 3)
        ops.na_bwd_reduce(None if g_y is None else g_y.float().contiguous(), None if g_sq is None else g_sq.contiguous(), x, mix, key, coef, need_eps,
                          red)
        dests, i = [None] * 6, 0
        for j in range(6):
            if full[j] is not None:
                dests[j] = D.mat(i, 1, 1)
                i += 1
        ops.na_param_grad(tab, mu, red, full, B, dests)
        return (None, None) + D.finish()


class NeuralAugLossFn(torch.autograd.Function):
    """(sq fp64 [B, 3], ce 0-dim or None) -> w_na * L_na + w_ce * ce, L_na = alpha / 65025 * mean_b smooth_l1(mse_b - target[step]) (0-dim
    fp32; loss_fn/composite_loss.py with loss_fn/neural_augmentation.py).  ``cfg``: target (device fp32 table), step (device int64 [1]), alpha,
    w_na, w_ce, H, W, scale (device loss scale or None), parts (device fp32 [2] for (ce, L_na), or None)."""

    @staticmethod
    def forward(ctx, sq, ce, cfg):
        loss = torch.empty((), device=sq.device, dtype=torch.float32)
        ops.na_loss_fwd(sq, cfg.H, cfg.W, cfg.target, cfg.step, cfg.alpha, loss, w_na=cfg.w_na, ce=ce, w_ce=cfg.w_ce, parts=cfg.parts)
        ctx.cfg, ctx.has_ce = cfg, ce is not None
        ctx.save_for_backward(sq)
        return loss

    @staticmethod
    def backward(ctx, g):
        (sq,) = ctx.saved_tensors
        c = ctx.cfg
        g_ce = torch.empty((), device=sq.device, dtype=torch.float32) if ctx.has_ce else None
        g_sq = ops.na_loss_bwd(sq, c.H, c.W, c.target, c.step, c.alpha, g.contiguous(), c.scale, w_na=c.w_na, g_ce=g_ce, w_ce=c.w_ce)
        return g_sq, g_ce, None


# ==================================================================================================================
# InvertedResidual (cvnets/modules/mobilenetv2.py:141-246): exp_1x1 -> dw3x3(stride) -> red_1x1 (+x)
# ==================================================================================================================
class InvertedResidualFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cfg, w1, g1, b1, wd, g2, b2, w3, g3, b3):
        B, Cin, H, W = x.shape
        hid, cout, s = cfg.hid, cfg.cout, cfg.stride
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        M, M2 = B * H * W, B * Ho * Wo
        x2 = as_2d(x)
        P = cfg.prep
        fa = _fwd_arena(cfg, x.device)
        st1, st2, st3 = fa.f64(2, hid), fa.f64(2, hid), fa.f64(2, cout)
        bs = [c.batch_stats for c in cfg.bn]  # per layer: individual BatchNorms may be frozen (base_model.py:139-165)
        lz = ctx.lz_in = cfg.lazy_in
        assert lz is None or not cfg.residual, "a lazily normalised input cannot also be the residual"
        am, _, ap = _lazy_modes(lz)
        y1 = ops.pw_gemm(x2, P.get(cfg.i_w1), hid, a_mode=am, a_p=ap, col_stats=st1 if bs[0] else None)
        bn1 = _bn_forward(st1, M, g1, b1, cfg.bn[0])
        y2 = ops.dw_fwd(y1, B, H, W, hid, s, P.get(cfg.i_wd), x_mode=A_AFF_SILU, x_p=(bn1[2], bn1[3]), col_stats=st2 if bs[1] else None,
                        dilation=cfg.dilation)
        bn2 = _bn_forward(st2, M2, g2, b2, cfg.bn[1])
        y3 = ops.pw_gemm(y2, P.get(cfg.i_w3), cout, a_mode=A_AFF_SILU, a_p=(bn2[2], bn2[3]), col_stats=st3 if bs[2] else None)
        bn3 = _bn_forward(st3, M2, g3, b3, cfg.bn[2])
        lazy_out = cfg.lazy_out and not cfg.residual
        ctx.lz_out = cfg.last_lazy = LazyBN(bn3, False) if lazy_out else None
        out = y3 if lazy_out else ops.bn_apply(y3, bn3, act=False, R=x2 if cfg.residual else None)
        ctx.cfg, ctx.dims, ctx.ev = cfg, (B, Cin, H, W, Ho, Wo), tuple(not b for b in bs)  # BN modes snapshotted for backward
        ctx.saved = (x2, y1, bn1, y2, bn2, y3, bn3)
        ctx.plist = cfg.plist
        ctx.save_for_backward(g1, g2, g3)
        return to_4d(out, B, Ho, Wo)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        B, Cin, H, W, Ho, Wo = ctx.dims
        hid, cout, s = cfg.hid, cfg.cout, cfg.stride
        M, M2 = B * H * W, B * Ho * Wo
        x2, y1, bn1, y2, bn2, y3, bn3 = ctx.saved
        g1, g2, g3 = ctx.saved_tensors
        P = cfg.prep
        ev = ctx.ev
        dout = as_2d(to_bf16_cl(gout))
        # parameter order: (w1, g1, b1, wd, g2, b2, w3, g3, b3)
        D = _Dst(cfg, ctx.plist, dout.device, True)
        ar = D.ar
        # red_1x1 + BN3 (no activation): dz3 = dout
        _, sd3 = _bn_out_grad(ctx.lz_out, D, dout, y3, bn3, False)
        sd2, sd1 = ar.f64(2, hid), ar.f64(2, hid)
        c3 = D.bn_bwd(sd3, M2, g3, bn3, ev[2], 7, 8)
        dz2 = ops.pw_gemm(dout, P.get(cfg.i_w3t), hid, K=cout, a_mode=A_BNB, A2=y3, a_p=c3, e_mode=E_SILU_BWD, Y=y2,
                          e_p=(bn2[2], bn2[3]), col_stats=sd2)
        ops.pw_wgrad_side(dout, y2, cout, hid, g_mode=A_BNB, G2=y3, g_p=c3, a_mode=A_AFF_SILU, a_p=(bn2[2], bn2[3]), dW=D.mat(6, cout, hid))
        # depthwise + BN2
        c2 = D.bn_bwd(sd2, M2, g2, bn2, ev[1], 4, 5)
        dz1, dWt = ops.dw_bwd(dz2, y1, B, H, W, hid, s, P.get(cfg.i_wd), g_mode=A_BNB, Y2=y2, g_p=c2, x_mode=A_AFF_SILU,
                              x_p=(bn1[2], bn1[3]), col_stats=sd1, dWt=ar.f32(9, hid), dilation=cfg.dilation)
        D.unprep(3, dWt, hid, 9, hid, PW.KIND_TAPMAJOR_F32)
        # exp_1x1 + BN1
        c1 = D.bn_bwd(sd1, M, g1, bn1, ev[0], 1, 2)
        lz = ctx.lz_in
        am, em, ap = _lazy_modes(lz)
        if lz is not None:  # the producer's BatchNorm (+SiLU) lives in this module's load mode: emit dz and its BN-backward sums for it
            lz.stats = ar.f64(2, Cin)
        dx = ops.pw_gemm(dz1, P.get(cfg.i_w1t), Cin, K=hid, a_mode=A_BNB, A2=y1, a_p=c1, e_mode=em, Y=x2 if lz is not None else None, e_p=ap,
                         R=dout if cfg.residual else None, col_stats=lz.stats if lz is not None else None)
        ops.pw_wgrad_side(dz1, x2, hid, Cin, g_mode=A_BNB, G2=y1, g_p=c1, a_mode=am, a_p=ap, dW=D.mat(0, hid, Cin))
        ops.join_side()
        return (to_4d(dx, B, H, W), None) + D.finish()


# ==================================================================================================================
# MobileViTBlockv2 (cvnets/modules/mobilevit_block.py:605-626) with LinearAttnFFN (cvnets/modules/transformer.py:248-264)
# and LinearSelfAttention (cvnets/layers/linear_attention.py:134-161); unfold/fold live in the attention kernel's indexing.
# Parameter order: [wd0, g0, b0, wl] + n x [ga, ba, wqkv, bqkv, wo, bo, gf, bf, w1, b1, w2, b2] + [gL, bL, wp, gp, bp]
# ==================================================================================================================
class MobileViTBlockv2Fn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cfg, *params):
        B, C, H, W = x.shape
        d, ffn, n = cfg.d, cfg.ffn, cfg.n_blocks
        HW = H * W
        M = B * HW
        P = cfg.prep
        x2 = as_2d(x)
        wd0, g0, b0, wl = params[:4]
        gL, bL, wp, gp, bp = params[4 + 12 * n:]
        bs = [c.batch_stats for c in cfg.bn]
        fa = _fwd_arena(cfg, x.device)
        st0, stp = fa.f64(2, C), fa.f64(2, C)
        samp = [fa.f64(2, B) for _ in range(2 * n + 1)]
        gcount = HW * d
        # local_rep: dw3x3 + BN + SiLU -> 1x1 (C -> d)
        ctx.lz_in = cfg.lazy_in
        am, _, ap = _lazy_modes(cfg.lazy_in)
        y0 = ops.dw_fwd(x2, B, H, W, C, 1, P.get(cfg.i_wd0), x_mode=am, x_p=ap, col_stats=st0 if bs[0] else None, dilation=cfg.dilation)
        bn0 = _bn_forward(st0, M, g0, b0, cfg.bn[0])
        X = ops.pw_gemm(y0, P.get(cfg.i_wl), d, a_mode=A_AFF_SILU, a_p=(bn0[2], bn0[3]), samp_stats=samp[0], rows_per_sample=HW)
        blocks = []
        for i in range(n):
            ga, ba, wqkv, bqkv, wo, bo, gf, bf, w1, b1, w2, b2 = params[4 + 12 * i: 16 + 12 * i]
            ix = cfg.i_blk[i]
            gnA = ops.gn_finalize(samp[2 * i], gcount, cfg.gn_eps)
            qkv = ops.pw_gemm(X, P.get(ix.wqkv), 2 * d + 8, a_mode=A_GN, a_p=(ga, ba), row_stats=(gnA[0], gnA[1]), rows_per_sample=HW,
                              bias=P.get(ix.bqkv))
            O, S, CTX = ops.linattn_fwd(qkv, B, H, W, d)
            X1 = ops.pw_gemm(O, P.get(ix.wo), d, bias=bo, R=X, samp_stats=samp[2 * i + 1], rows_per_sample=HW)
            gnF = ops.gn_finalize(samp[2 * i + 1], gcount, cfg.gn_eps)
            h = ops.pw_gemm(X1, P.get(ix.w1), ffn, a_mode=A_GN, a_p=(gf, bf), row_stats=(gnF[0], gnF[1]), rows_per_sample=HW, bias=b1)
            X2 = ops.pw_gemm(h, P.get(ix.w2), d, a_mode=A_SILU, bias=b2, R=X1, samp_stats=samp[2 * i + 2], rows_per_sample=HW)
            blocks.append((X, gnA, qkv, O, S, CTX, X1, gnF, h))
            X = X2
        gnL = ops.gn_finalize(samp[2 * n], gcount, cfg.gn_eps)
        yp = ops.pw_gemm(X, P.get(cfg.i_wp), C, a_mode=A_GN, a_p=(gL, bL), row_stats=(gnL[0], gnL[1]), rows_per_sample=HW,
                         col_stats=stp if bs[1] else None)
        bnp = _bn_forward(stp, M, gp, bp, cfg.bn[1])
        ctx.lz_out = cfg.last_lazy = LazyBN(bnp, False) if cfg.lazy_out else None
        out = yp if cfg.lazy_out else ops.bn_apply(yp, bnp, act=False)
        ctx.cfg, ctx.dims, ctx.ev = cfg, (B, C, H, W), tuple(not b for b in bs)
        ctx.saved = (x2, y0, bn0, blocks, X, gnL, yp, bnp)
        ctx.plist = cfg.plist
        ctx.save_for_backward(*params)
        return to_4d(out, B, H, W)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        B, C, H, W = ctx.dims
        d, ffn, n = cfg.d, cfg.ffn, cfg.n_blocks
        HW = H * W
        M = B * HW
        P = cfg.prep
        params = ctx.saved_tensors
        x2, y0, bn0, blocks, XL, gnL, yp, bnp = ctx.saved
        wd0, g0, b0, wl = params[:4]
        gL, bL, wp, gp, bp = params[4 + 12 * n:]
        ev = ctx.ev
        dev = x2.device
        gcount = HW * d
        dout = as_2d(to_bf16_cl(gout))
        D = _Dst(cfg, ctx.plist, dev, True)
        ar = D.ar
        # ---- conv_proj (GN -> 1x1 -> BN, no act)
        base = 4 + 12 * n
        _, sdp = _bn_out_grad(ctx.lz_out, D, dout, yp, bnp, False)
        sd0 = ar.f64(2, C)
        cp = D.bn_bwd(sdp, M, gp, bnp, ev[1], base + 3, base + 4)
        cs, ss = ar.f64(2, d), ar.f64(2, B)
        g = ops.pw_gemm(dout, P.get(cfg.i_wpt), d, K=C, a_mode=A_BNB, A2=yp, a_p=cp, e_mode=E_GN_BWD, Y=XL, e_p=(gL, None),
                        row_stats=(gnL[0], gnL[1]), rows_per_sample=HW, col_stats=cs, samp_stats=ss, gn_ws=ar.f64(2, B, d))
        ops.pw_wgrad_side(dout, XL, C, d, g_mode=A_BNB, G2=yp, g_p=cp, a_mode=A_GN, a_p=(gL, bL), row_stats=(gnL[0], gnL[1]),
                          rows_per_sample=HW, dW=D.mat(base + 2, C, d))
        D.late64(base + 0, cs[1])  # dgamma = sum v*xhat
        D.late64(base + 1, cs[0])  # dbeta = sum v
        bsum = ar.f64(d)  # column sums of the residual-stream gradient = bias gradient of the producing conv
        dX = ops.gn_bwd_apply(g, XL, gnL, ss, gcount, B, HW, DRES=None, col_sum=bsum if n > 0 else None)
        # ---- attention/FFN units, last to first
        for i in reversed(range(n)):
            X, gnA, qkv, O, S, CTX, X1, gnF, h = blocks[i]
            ga, ba, wqkv, bqkv, wo, bo, gf, bf, w1, b1, w2, b2 = params[4 + 12 * i: 16 + 12 * i]
            ix = cfg.i_blk[i]
            o = 4 + 12 * i
            # FFN: X2 = X1 + W2 silu(h) + b2 ; h = W1 GN(X1) + b1
            D.late64(o + 11, bsum)  # db2
            ops.pw_wgrad_side(dX, h, d, ffn, a_mode=A_SILU, dW=D.mat(o + 10, d, ffn))
            csh, csf, ssf, bsum1 = ar.f64(2, ffn), ar.f64(2, d), ar.f64(2, B), ar.f64(d)
            dh = ops.pw_gemm(dX, P.get(ix.w2t), ffn, K=d, e_mode=E_SILU_BWD, Y=h, col_stats=csh)
            D.late64(o + 9, csh[0])  # db1 = column sums of dh
            ops.pw_wgrad_side(dh, X1, ffn, d, a_mode=A_GN, a_p=(gf, bf), row_stats=(gnF[0], gnF[1]), rows_per_sample=HW, dW=D.mat(o + 8, ffn, d))
            gF = ops.pw_gemm(dh, P.get(ix.w1t), d, K=ffn, e_mode=E_GN_BWD, Y=X1, e_p=(gf, None), row_stats=(gnF[0], gnF[1]),
                             rows_per_sample=HW, col_stats=csf, samp_stats=ssf, gn_ws=ar.f64(2, B, d))
            D.late64(o + 6, csf[1])
            D.late64(o + 7, csf[0])
            dX1 = ops.gn_bwd_apply(gF, X1, gnF, ssf, gcount, B, HW, DRES=dX, col_sum=bsum1)
            # attention: X1 = X + Wo O + bo ; O = linattn(qkv) ; qkv = Wqkv GN(X) + bqkv
            D.late64(o + 5, bsum1)  # dbo
            ops.pw_wgrad_side(dX1, O, d, d, dW=D.mat(o + 4, d, d))
            dO = ops.pw_gemm(dX1, P.get(ix.wot), d, K=d)
            dbq = ar.f32(2 * d + 8)
            dqkv = ops.linattn_bwd(qkv, dO, S, CTX, B, H, W, d, dbias=dbq)
            dWq = ops.pw_wgrad_side(dqkv, X, 2 * d + 8, d, a_mode=A_GN, a_p=(ga, ba), row_stats=(gnA[0], gnA[1]), rows_per_sample=HW,
                                    dW=ar.f32(2 * d + 8, d))
            D.unprep(o + 2, dWq, 2 * d + 1, d, d, PW.KIND_ROWMAJOR, rot=1, side=True)
            D.unprep(o + 3, dbq, 2 * d + 1, 1, 1, PW.KIND_VECTOR_F32, rot=1)
            csa, ssa, bsum = ar.f64(2, d), ar.f64(2, B), ar.f64(d)
            gA = ops.pw_gemm(dqkv, P.get(ix.wqkvt), d, K=2 * d + 8, e_mode=E_GN_BWD, Y=X, e_p=(ga, None), row_stats=(gnA[0], gnA[1]),
                             rows_per_sample=HW, col_stats=csa, samp_stats=ssa, gn_ws=ar.f64(2, B, d))
            D.late64(o + 0, csa[1])
            D.late64(o + 1, csa[0])
            dX = ops.gn_bwd_apply(gA, X, gnA, ssa, gcount, B, HW, DRES=dX1, col_sum=bsum if i > 0 else None)
        # ---- local_rep: 1x1 (no bias / norm) <- SiLU <- BN0 <- dw3x3
        ops.pw_wgrad_side(dX, y0, d, C, a_mode=A_AFF_SILU, a_p=(bn0[2], bn0[3]), dW=D.mat(3, d, C))
        dz0 = ops.pw_gemm(dX, P.get(cfg.i_wlt), C, K=d, e_mode=E_SILU_BWD, Y=y0, e_p=(bn0[2], bn0[3]), col_stats=sd0)
        c0 = D.bn_bwd(sd0, M, g0, bn0, ev[0], 1, 2)
        lz = ctx.lz_in
        am, _, ap = _lazy_modes(lz)
        if lz is not None:
            lz.stats = ar.f64(2, C)
        dx, dWt = ops.dw_bwd(dz0, x2, B, H, W, C, 1, P.get(cfg.i_wd0), g_mode=A_BNB, Y2=y0, g_p=c0, x_mode=am, x_p=ap,
                             col_stats=lz.stats if lz is not None else None, dWt=ar.f32(9, C), dilation=cfg.dilation)
        D.unprep(0, dWt, C, 9, C, PW.KIND_TAPMAJOR_F32)
        ops.join_side()
        return (to_4d(dx, B, H, W), None) + D.finish()


# ==================================================================================================================
# classifier head: GlobalPool(mean) + LinearLayer (cvnets/layers/global_pool.py:60-71, linear_layer.py:90)
# ==================================================================================================================
class PoolLinearFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, cfg, w, b):
        B, C, H, W = x.shape
        x2 = as_2d(x)
        pooled = ops.global_pool_fwd(x2, B, H * W)
        ncls = w.shape[0]
        npad = (ncls + 7) // 8 * 8
        logits = ops.pw_gemm(pooled, cfg.prep.get(cfg.i_w), npad, bias=cfg.prep.get(cfg.i_b))
        ctx.cfg, ctx.dims = cfg, (B, C, H, W, ncls, npad)
        ctx.saved = (pooled,)
        ctx.plist = cfg.plist
        return logits[:, :ncls]

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        B, C, H, W, ncls, npad = ctx.dims
        (pooled,) = ctx.saved
        if (gout.dtype == BF16 and gout.dim() == 2 and gout.stride() == (npad, 1) and gout.storage_offset() == 0
                and gout.untyped_storage().nbytes() >= B * npad * 2):
            g = gout.as_strided((B, npad), (npad, 1))  # the padded dlogits matrix cvb_ce_bwd wrote (pad columns are zero)
        else:
            g = torch.zeros((B, npad), device=pooled.device, dtype=BF16)
            g[:, :ncls] = gout
        D = _Dst(cfg, ctx.plist, pooled.device, npad == ncls)
        ops.pw_wgrad_side(g, pooled, npad, C, dW=D.padded(0, ncls, C, npad), dbias=D.padded(1, ncls, 1, npad).view(npad))
        dp = ops.pw_gemm(g, cfg.prep.get(cfg.i_wt), C, K=npad)
        dx = ops.global_pool_bwd(dp, B, H * W)
        ops.join_side()
        return (to_4d(dx, B, H, W), None) + D.finish()


# ==================================================================================================================
# Classification loss (loss_fn/classification/cross_entropy.py:74-95): F.cross_entropy(label_smoothing, ignore_index), mean reduction.
# Two launches; the GradScaler's loss scale (a device scalar) multiplies inside the backward kernel.
# ==================================================================================================================
class CrossEntropyFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, logits, target, cfg):
        B, C = logits.shape
        lg = logits
        if lg.dtype != BF16 or lg.stride(1) != 1 or lg.stride(0) % 8:
            lg = logits.to(BF16).contiguous()
        if target.dtype != torch.int64 or target.dim() != 1 or target.shape[0] != B:
            raise ValueError("cross_entropy: target must be an int64 tensor of shape [batch] (class indices)")
        target = target.contiguous()
        loss, lse, nv = ops.ce_fwd(lg, C, target, cfg.ignore_index, cfg.label_smoothing, mix=getattr(cfg, "mix", None))
        ctx.cfg, ctx.saved, ctx.C = cfg, (lg, target, lse, nv), C
        return loss.view(())

    @staticmethod
    def backward(ctx, gout):
        lg, target, lse, nv = ctx.saved
        cfg, C = ctx.cfg, ctx.C
        g = gout if (gout.dtype == torch.float32 and gout.is_contiguous()) else gout.float().contiguous()
        ldd = lg.stride(0) if lg.stride(0) >= C else (C + 7) // 8 * 8
        d = ops.ce_bwd(lg, C, target, cfg.ignore_index, cfg.label_smoothing, lse, nv, g, getattr(cfg, "scale", None), ldd, mix=getattr(cfg, "mix", None))
        return d[:, :C], None, None


# ==================================================================================================================
# Stand-alone layer functions: the hot-path LAYERS used outside the fused modules (SURVEY.md 8a a1, a7, a8, a12-a14; north_star:
# "MultiHeadAttention and MobileViTv2 LinearSelfAttention in cvnets/layers ... drop-in nn.Module").  Same kernels, one layer per
# autograd function, outputs materialised -- the unfused but native path every layer falls back to when it is not inside a fused block.
# ==================================================================================================================
class PointwiseConvFn(torch.autograd.Function):
    """ConvLayer2d, groups = 1: conv (+bias) [-> BatchNorm2d] [-> Swish | GELU] [+ residual] on a [B, Cin, H, W] map
    (cvnets/layers/conv_layer.py:200-226, 254-255).  1x1 convs ARE the GEMM; k x k convs (the ViT / CLIP conv stem, MobileViT-v1's dense
    3x3 convs) go through the gathered patch matrix of cvb_im2col (csrc/conv.cu).  params = (w, bias | None, gamma | None, beta | None)."""

    @staticmethod
    def forward(ctx, x, cfg, residual, w, bias, gamma, beta):
        B, Cin, H, W = x.shape
        cout = cfg.cout
        P = cfg.prep
        if cfg.k == 1 and cfg.stride == 1:
            x2, Ho, Wo = as_2d(x), H, W
        else:
            x2, Ho, Wo = ops.im2col(x, cfg.k, cfg.stride, cfg.pad)
        M = B * Ho * Wo
        R = as_2d(residual) if residual is not None else None
        ob = None
        if cfg.bn is not None:
            st = _fwd_arena(cfg, x.device).f64(2, cout)
            y = ops.pw_gemm(x2, P.get(cfg.i_w), cout, bias=bias, col_stats=st if cfg.bn.batch_stats else None)
            bn = _bn_forward(st, M, gamma, beta, cfg.bn)
            if cfg.act in (None, ops.ACT_SILU):
                out = ops.bn_apply(y, bn, act=cfg.act is not None, R=R)
            else:  # BatchNorm -> GELU (the ViT conv stem under model.activation.name = gelu): two passes, the stem is ~1 % of the model
                if R is not None:
                    raise NotImplementedError("BatchNorm + GELU + residual in one stand-alone ConvLayer2d")
                ob = ops.bn_apply(y, bn, act=False)
                out = ops.act_fwd(ob, cfg.act)
            ctx.saved, ctx.ev = (x2, y, bn, ob), (not cfg.bn.batch_stats,)
        elif cfg.act is not None:
            h = ops.pw_gemm(x2, P.get(cfg.i_w), cout, bias=bias)
            out = ops.act_fwd(h, cfg.act)
            if R is not None:
                raise NotImplementedError("activation + residual in one stand-alone ConvLayer2d")
            ctx.saved = (x2, h)
        else:
            out = ops.pw_gemm(x2, P.get(cfg.i_w), cout, bias=bias, R=R)
            ctx.saved = (x2,)
        ctx.cfg, ctx.dims, ctx.plist, ctx.has_res = cfg, (B, Cin, H, W, Ho, Wo), cfg.plist, residual is not None
        ctx.x_fp32_nchw = x.dtype == torch.float32 and x.is_contiguous()
        ctx.save_for_backward(gamma) if gamma is not None else None
        return to_4d(out, B, Ho, Wo)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        B, Cin, H, W, Ho, Wo = ctx.dims
        M, cout = B * Ho * Wo, cfg.cout
        P = cfg.prep
        dense = not (cfg.k == 1 and cfg.stride == 1)
        dout = as_2d(to_bf16_cl(gout))
        x2 = ctx.saved[0]
        Kc = x2.shape[1]
        D = _Dst(cfg, ctx.plist, dout.device, True)
        has_bias = cfg.has_bias
        db = D.mat(1, 1, cout).view(cout) if has_bias else None
        dW = D.ar.f32(cout, Kc) if dense else D.mat(0, cout, Cin)
        need_dx = ctx.needs_input_grad[0]
        dA = dx = None
        # the ViT / CLIP image stem (fp32 3-channel image, 4x4 stride-4 pad-1 windows): its image gradient, which the RangeAugment augmentor
        # reads, comes straight from (dz, y) as fp32 NCHW (cvb_patch_stem_dgrad) instead of a GEMM, col2im and a conversion
        patch_stem = (need_dx and cfg.bn is not None and ctx.x_fp32_nchw and Cin == 3 and cfg.k == 4 and cfg.stride == 4 and cfg.pad == 1
                      and H % 4 == 0 and W % 4 == 0 and cout % 16 == 0 and cout <= 320)
        if cfg.bn is not None:
            _, y, bn, ob = ctx.saved
            (gamma,) = ctx.saved_tensors
            if ob is not None:
                dout = ops.act_bwd(dout, ob, cfg.act)
            dz, sd = _bn_out_grad(None, D, dout, y, bn, cfg.act == ops.ACT_SILU)
            gi = 2 if has_bias else 1  # (gamma, beta) follow (w[, bias]) in plist
            c = D.bn_bwd(sd, M, gamma, bn, ctx.ev[0], gi, gi + 1)
            if patch_stem:
                dx = ops.patch_stem_dgrad(dz, y, c, P.get(cfg.i_w), B, Ho, Wo)
            elif need_dx:
                dA = ops.pw_gemm(dz, P.get(cfg.i_wt), Kc, K=cout, a_mode=A_BNB, A2=y, a_p=c)
            ops.pw_wgrad_side(dz, x2, cout, Kc, g_mode=A_BNB, G2=y, g_p=c, dW=dW, dbias=db)
        else:
            dh = ops.act_bwd(dout, ctx.saved[1], cfg.act) if cfg.act is not None else dout
            if need_dx:
                dA = ops.pw_gemm(dh, P.get(cfg.i_wt), Kc, K=cout)
            ops.pw_wgrad_side(dh, x2, cout, Kc, dW=dW, dbias=db)
        if dense:
            D.unprep(0, dW, cout, cfg.k * cfg.k * Cin, Kc, PW.KIND_PATCH, rot=cfg.k * cfg.k, side=True)
        ops.join_side()
        if dA is not None:
            dx = to_4d(ops.col2im(dA, B, Cin, H, W, cfg.k, cfg.stride, cfg.pad) if dense else dA, B, H, W)
        grads = D.finish()
        full = [grads[0], None, None, None]
        if has_bias:
            full[1] = grads[1]
        if cfg.bn is not None:
            full[2], full[3] = grads[2 if has_bias else 1], grads[3 if has_bias else 2]
        return (dx, None, gout if ctx.has_res else None) + tuple(full)


class DepthwiseConvFn(torch.autograd.Function):
    """ConvLayer2d with a depthwise 3x3 or 5x5 kernel (groups = channels, stride 1 | 2, no bias) [-> BatchNorm2d] [-> Swish]."""

    @staticmethod
    def forward(ctx, x, cfg, w, gamma, beta):
        B, C, H, W = x.shape
        s = cfg.stride
        Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
        M2 = B * Ho * Wo
        x2 = as_2d(x)
        if cfg.bn is not None:
            st = _fwd_arena(cfg, x.device).f64(2, C)
            y = ops.dw_fwd(x2, B, H, W, C, s, cfg.prep.get(cfg.i_w), col_stats=st if cfg.bn.batch_stats else None, dilation=cfg.dilation,
                           ksize=cfg.k)
            bn = _bn_forward(st, M2, gamma, beta, cfg.bn)
            out = ops.bn_apply(y, bn, act=cfg.act is not None)
            ctx.saved, ctx.ev = (x2, y, bn), (not cfg.bn.batch_stats,)
        else:
            y = ops.dw_fwd(x2, B, H, W, C, s, cfg.prep.get(cfg.i_w), dilation=cfg.dilation, ksize=cfg.k)
            out = ops.act_fwd(y, cfg.act) if cfg.act is not None else y
            ctx.saved = (x2, y)
        ctx.cfg, ctx.dims, ctx.plist = cfg, (B, C, H, W, Ho, Wo), cfg.plist
        ctx.save_for_backward(gamma) if gamma is not None else None
        return to_4d(out, B, Ho, Wo)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        B, C, H, W, Ho, Wo = ctx.dims
        M2 = B * Ho * Wo
        dout = as_2d(to_bf16_cl(gout))
        taps = cfg.k * cfg.k
        D = _Dst(cfg, ctx.plist, dout.device, True)
        if cfg.bn is not None:
            x2, y, bn = ctx.saved
            (gamma,) = ctx.saved_tensors
            dz, sd = _bn_out_grad(None, D, dout, y, bn, cfg.act is not None)
            c = D.bn_bwd(sd, M2, gamma, bn, ctx.ev[0], 1, 2)
            dx, dWt = ops.dw_bwd(dz, x2, B, H, W, C, cfg.stride, cfg.prep.get(cfg.i_w), g_mode=A_BNB, Y2=y, g_p=c, dWt=D.ar.f32(taps, C),
                                 dilation=cfg.dilation, ksize=cfg.k)
        else:
            x2, y = ctx.saved
            dz = ops.act_bwd(dout, y, cfg.act) if cfg.act is not None else dout
            dx, dWt = ops.dw_bwd(dz, x2, B, H, W, C, cfg.stride, cfg.prep.get(cfg.i_w), dWt=D.ar.f32(taps, C), dilation=cfg.dilation,
                                 ksize=cfg.k)
        D.unprep(0, dWt, C, taps, C, PW.KIND_TAPMAJOR_F32)
        grads = D.finish()
        return (to_4d(dx, B, H, W), None, grads[0]) + ((grads[1], grads[2]) if cfg.bn is not None else (None, None))


class GroupNorm1Fn(torch.autograd.Function):
    """LayerNorm2D_NCHW == nn.GroupNorm(1, C) on [B, C, H, W] (cvnets/layers/normalization/layer_norm.py:75-108): statistics over all of
    (C, H, W) per sample in fp32 (fp64 accumulation), per-channel affine."""

    @staticmethod
    def forward(ctx, x, cfg, gamma, beta):
        B, C, H, W = x.shape
        rps = H * W
        x2 = as_2d(x)
        st = _fwd_arena(cfg, x.device).f64(2, B)
        ops.gn_stats(x2, B, rps, st)
        gn = ops.gn_finalize(st, rps * C, cfg.eps)
        out = ops.apply_load_mode(x2, ops.A_GN, C, a_p=(gamma, beta, None), row_stats=(gn[0], gn[1]), rows_per_sample=rps)
        ctx.cfg, ctx.dims, ctx.saved, ctx.plist = cfg, (B, C, H, W), (x2, gn), cfg.plist
        ctx.save_for_backward(gamma)
        return to_4d(out, B, H, W)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        B, C, H, W = ctx.dims
        x2, gn = ctx.saved
        (gamma,) = ctx.saved_tensors
        dout = as_2d(to_bf16_cl(gout))
        D = _Dst(cfg, ctx.plist, dout.device, True)
        dgb, wsp = D.ar.f64(2, C), D.ar.f64(2, B)
        dx = ops.gn_bwd(dout, x2, gn, gamma, float(H * W * C), B, H * W, dgb[0], dgb[1], wsp)
        D.late64(0, dgb[0])
        D.late64(1, dgb[1])
        return (to_4d(dx, B, H, W), None) + D.finish()


class LayerNormFn(torch.autograd.Function):
    """LayerNorm / LayerNormFP32 over the last dimension of a [..., C] tensor (cvnets/layers/normalization/layer_norm.py:14-72, 111-137).
    Statistics and the normalisation are computed in fp32 from the bf16 input for both variants (the FP32 variant's upcast is implicit)."""

    @staticmethod
    def forward(ctx, x, cfg, gamma, beta):
        shape = x.shape
        C = shape[-1]
        x2 = x.reshape(-1, C).to(BF16).contiguous()
        ln = ops.ln_stats(x2, cfg.eps)
        out = ops.apply_load_mode(x2, ops.A_GN, C, a_p=(gamma, beta, None), row_stats=(ln[0], ln[1]), rows_per_sample=1)
        ctx.cfg, ctx.shape, ctx.saved, ctx.plist = cfg, shape, (x2, ln), cfg.plist
        ctx.save_for_backward(gamma)
        return out.view(shape)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        C = ctx.shape[-1]
        x2, ln = ctx.saved
        (gamma,) = ctx.saved_tensors
        dy = gout.reshape(-1, C).to(BF16).contiguous()
        D = _Dst(cfg, ctx.plist, dy.device, True)
        cs = D.ar.f64(2, C)
        dx = ops.ln_bwd(dy, x2, ln, gamma, cs)
        D.late64(0, cs[1])
        D.late64(1, cs[0])
        return (dx.view(ctx.shape), None) + D.finish()


class LinearSelfAttentionFn(torch.autograd.Function):
    """Stand-alone LinearSelfAttention on the unfolded tensor x [B, d, P, N] (cvnets/layers/linear_attention.py:134-215): self-attention, or
    cross-attention against x_prev [B, d, P, M] (query/key from x_prev, value from x).  ``residual`` (optional, [B, d, P, N]) is added in
    the out_proj epilogue.  params = (wqkv, bqkv, wo, bo)."""

    @staticmethod
    def forward(ctx, x, cfg, x_prev, residual, wqkv, bqkv, wo, bo):
        B, d, Pp, N = x.shape
        Pw = cfg.prep
        x2 = as_2d(x)
        R = as_2d(residual) if residual is not None else None
        qkv = ops.pw_gemm(x2, Pw.get(cfg.i_wqkv), 2 * d + 8, bias=Pw.get(cfg.i_bqkv))
        if x_prev is None:
            xp2, qkp = None, None
            O, S, CTX = ops.linattn_fwd(qkv, B, Pp, N, d, patch=0)
        else:
            if x_prev.shape[0] != B or x_prev.shape[1] != d or x_prev.shape[2] != Pp:
                raise ValueError("The number of pixels in a patch for query and key_value should be the same")  # linear_attention.py:172-174
            xp2 = as_2d(x_prev)
            qkp = ops.pw_gemm(xp2, Pw.get(cfg.i_wqkv), 2 * d + 8, bias=Pw.get(cfg.i_bqkv))
            O, S, CTX = ops.linattn_cross_fwd(qkp, qkv, B, Pp, x_prev.shape[3], N, d)
        y = ops.pw_gemm(O, Pw.get(cfg.i_wo), d, bias=bo, R=R)
        ctx.cfg, ctx.dims, ctx.plist = cfg, (B, d, Pp, N, x_prev.shape[3] if x_prev is not None else N), cfg.plist
        ctx.saved = (x2, qkv, xp2, qkp, O, S, CTX)
        ctx.has_res = residual is not None
        return to_4d(y, B, Pp, N)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        B, d, Pp, N, Mp = ctx.dims
        Pw = cfg.prep
        x2, qkv, xp2, qkp, O, S, CTX = ctx.saved
        dy = as_2d(to_bf16_cl(gout))
        D = _Dst(cfg, ctx.plist, dy.device, True)
        ar = D.ar
        ops.pw_wgrad_side(dy, O, d, d, dW=D.mat(2, d, d), dbias=D.mat(3, 1, d).view(d))
        dO = ops.pw_gemm(dy, Pw.get(cfg.i_wot), d, K=d)
        dbq = ar.f32(2 * d + 8)
        dWq = ar.f32(2 * d + 8, d)
        if xp2 is None:
            dqkv = ops.linattn_bwd(qkv, dO, S, CTX, B, Pp, N, d, dbias=dbq, patch=0)
            ops.pw_wgrad_side(dqkv, x2, 2 * d + 8, d, dW=dWq)
            dx = ops.pw_gemm(dqkv, Pw.get(cfg.i_wqkvt), d, K=2 * d + 8)
            dxp = None
        else:
            dqkp, dqkv = ops.linattn_cross_bwd(qkp, qkv, dO, S, CTX, B, Pp, Mp, N, d, dbias=dbq)
            ops.pw_wgrad_side(dqkp, xp2, 2 * d + 8, d, dW=dWq)
            ops.pw_wgrad_side(dqkv, x2, 2 * d + 8, d, dW=dWq)
            dx = ops.pw_gemm(dqkv, Pw.get(cfg.i_wqkvt), d, K=2 * d + 8)
            dxp = to_4d(ops.pw_gemm(dqkp, Pw.get(cfg.i_wqkvt), d, K=2 * d + 8), B, Pp, Mp)
        D.unprep(0, dWq, 2 * d + 1, d, d, PW.KIND_ROWMAJOR, rot=1, side=True)
        D.unprep(1, dbq, 2 * d + 1, 1, 1, PW.KIND_VECTOR_F32, rot=1)
        ops.join_side()
        return (to_4d(dx, B, Pp, N), None, dxp, gout if ctx.has_res else None) + D.finish()


class LinearFn(torch.autograd.Function):
    """LinearLayer: y = x W^T + b on [..., Cin] (cvnets/layers/linear_layer.py:74-96)."""

    @staticmethod
    def forward(ctx, x, cfg, w, b):
        shape = x.shape
        cin, cout, npad = shape[-1], cfg.cout, cfg.npad
        x2 = x.reshape(-1, cin).to(BF16).contiguous()
        y = ops.pw_gemm(x2, cfg.prep.get(cfg.i_w), npad, bias=cfg.prep.get(cfg.i_b) if b is not None else None)
        ctx.cfg, ctx.shape, ctx.saved, ctx.plist = cfg, shape, (x2,), cfg.plist
        return y[:, :cout].view(*shape[:-1], cout)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        cin, cout, npad = ctx.shape[-1], cfg.cout, cfg.npad
        (x2,) = ctx.saved
        M = x2.shape[0]
        g = gout.reshape(M, cout)
        if npad != cout:
            gp = torch.zeros((M, npad), device=g.device, dtype=BF16)
            gp[:, :cout] = g
            g = gp
        else:
            g = g.to(BF16).contiguous()
        has_b = len(ctx.plist) > 1
        D = _Dst(cfg, ctx.plist, g.device, npad == cout)
        ops.pw_wgrad_side(g, x2, npad, cin, dW=D.padded(0, cout, cin, npad), dbias=D.padded(1, cout, 1, npad).view(npad) if has_b else None)
        dx = ops.pw_gemm(g, cfg.prep.get(cfg.i_wt), cin, K=npad)
        ops.join_side()
        grads = D.finish()
        return (dx.view(ctx.shape), None, grads[0], grads[1] if has_b else None)


class GlobalPoolFn(torch.autograd.Function):
    """GlobalPool(mean) on [B, C, H, W] (cvnets/layers/global_pool.py:60-71)."""

    @staticmethod
    def forward(ctx, x, keep_dim):
        B, C, H, W = x.shape
        out = ops.global_pool_fwd(as_2d(x), B, H * W)
        ctx.dims = (B, C, H, W)
        return out.view(B, C, 1, 1) if keep_dim else out

    @staticmethod
    def backward(ctx, gout):
        B, C, H, W = ctx.dims
        g = gout.reshape(B, C).to(BF16).contiguous()
        return to_4d(ops.global_pool_bwd(g, B, H * W), B, H, W), None


class ActFn(torch.autograd.Function):
    """A stand-alone activation module on a channels-last bf16 map (cvnets/layers/activation/*.py): the act_fn_1 / act_fn_2 / scale_act children of
    InvertedResidualSE and SqueezeExcitation (cvnets/modules/mobilenetv2.py:63-92, squeeze_excitation.py:66-76).  kind: ops.ACT_*."""

    @staticmethod
    def forward(ctx, x, kind):
        if x.numel() % 8:
            raise NotImplementedError("activation: tensors with numel % 8 == 0")
        ctx.kind, ctx.x = kind, x
        y = ops.act_fwd(x, kind)
        return y

    @staticmethod
    def backward(ctx, gout):
        x = ctx.x
        g = gout
        if g.dtype != BF16 or g.stride() != x.stride():
            g = torch.empty_like(x).copy_(gout)  # same memory layout as x: the kernel is a flat element-wise pass
        return ops.act_bwd(g, x, ctx.kind), None


class DropoutFn(torch.autograd.Function):
    """nn.Dropout in training mode on a bf16 tensor whose last dimension is a multiple of 8 (cvnets/layers/dropout.py): the mask is a hash of a
    device-resident key (ops.rng_next), regenerated -- not stored -- in the backward."""

    @staticmethod
    def forward(ctx, x, p):
        x2 = x.reshape(-1, x.shape[-1]).to(BF16).contiguous()
        key = ops.rng_next(x.device)
        ctx.p, ctx.key, ctx.shape = p, key, x.shape
        return ops.dropout_fwd(x2, None, p, key).view(x.shape)

    @staticmethod
    def backward(ctx, gout):
        g = gout.reshape(-1, ctx.shape[-1]).to(BF16).contiguous()
        return ops.dropout_bwd(g, ctx.p, ctx.key).view(ctx.shape), None


class StochasticDepthAddFn(torch.autograd.Function):
    """``x + StochasticDepth(p, "row")(y)`` on [B, C, H, W] maps (cvnets/modules/efficientnet.py): one hashed per-sample keep factor
    (0 or 1 / (1 - p)), drawn from a device-resident key and regenerated -- not stored -- in the backward."""

    @staticmethod
    def forward(ctx, y, x, p):
        B, C, H, W = y.shape
        key = ops.rng_next(y.device)
        ctx.p, ctx.key, ctx.dims = p, key, (B, H, W)
        return to_4d(ops.dropout_fwd(as_2d(y), as_2d(x), 0.0, key, p_row=p, rows_per_sample=H * W), B, H, W)

    @staticmethod
    def backward(ctx, gout):
        B, H, W = ctx.dims
        g = as_2d(to_bf16_cl(gout))
        return to_4d(ops.dropout_bwd(g, 0.0, ctx.key, p_row=ctx.p, rows_per_sample=H * W), B, H, W), gout, None


class SeScaleFn(torch.autograd.Function):
    """SqueezeExcitation.forward's ``x * se_layer(x)`` (cvnets/modules/squeeze_excitation.py:82-83): [B, C, H, W] map times a [B, C, 1, 1] scale."""

    @staticmethod
    def forward(ctx, x, s):
        B, C, H, W = x.shape
        s2 = s.reshape(B, C).to(BF16).contiguous()
        x2 = as_2d(x)
        ctx.saved, ctx.dims = (x2, s2), (B, C, H, W)
        return to_4d(ops.se_scale_fwd(x2, s2, B, H * W), B, H, W)

    @staticmethod
    def backward(ctx, gout):
        B, C, H, W = ctx.dims
        x2, s2 = ctx.saved
        dx, ds = ops.se_scale_bwd(as_2d(to_bf16_cl(gout)), x2, s2, B, H * W)
        return to_4d(dx, B, H, W), ds.view(B, C, 1, 1)


class UnfoldFn(torch.autograd.Function):
    """MobileViTBlock.unfolding (cvnets/modules/mobilevit_block.py:186-231): [B, C, H, W] -> [B*P, N, C] tokens (a row permutation)."""

    @staticmethod
    def forward(ctx, x, ph, pw):
        B, C, H, W = x.shape
        if H % ph or W % pw:
            raise NotImplementedError("H, W must be multiples of the patch size (the bilinear resize branch, mobilevit_block.py:191-200, is not implemented)")
        ctx.dims = (B, C, H, W, ph, pw)
        return ops.patch_permute(as_2d(x), B, H, W, ph, pw, False).view(B * ph * pw, (H // ph) * (W // pw), C)

    @staticmethod
    def backward(ctx, g):
        B, C, H, W, ph, pw = ctx.dims
        g2 = g.reshape(-1, C).to(BF16).contiguous()
        return to_4d(ops.patch_permute(g2, B, H, W, ph, pw, True), B, H, W), None, None


class FoldFn(torch.autograd.Function):
    """MobileViTBlock.folding (mobilevit_block.py:233-267): [B*P, N, C] tokens -> [B, C, H, W]."""

    @staticmethod
    def forward(ctx, t, B, H, W, ph, pw):
        C = t.shape[-1]
        t2 = t.reshape(-1, C).to(BF16).contiguous()
        ctx.dims = (B, C, H, W, ph, pw, tuple(t.shape))
        return to_4d(ops.patch_permute(t2, B, H, W, ph, pw, True), B, H, W)

    @staticmethod
    def backward(ctx, g):
        B, C, H, W, ph, pw, shape = ctx.dims
        return ops.patch_permute(as_2d(to_bf16_cl(g)), B, H, W, ph, pw, False).view(shape), None, None, None, None, None


class Concat2Fn(torch.autograd.Function):
    """torch.cat((a, b), dim=1) on channels-last feature maps (the fusion input of MobileViTBlock, mobilevit_block.py:287)."""

    @staticmethod
    def forward(ctx, a, b):
        B, C1, H, W = a.shape
        ctx.dims = (B, C1, b.shape[1], H, W)
        return to_4d(ops.concat2(as_2d(a), as_2d(b)), B, H, W)

    @staticmethod
    def backward(ctx, g):
        B, C1, C2, H, W = ctx.dims
        da, db = ops.split2(as_2d(to_bf16_cl(g)), C1, C2)
        return to_4d(da, B, H, W), to_4d(db, B, H, W)


class VitTokensFn(torch.autograd.Function):
    """ViT token assembly (cvnets/models/classification/vit.py:476-507): tokens = cat(cls, patch_embedding + positional_embedding).
    patch: [B, C, nh, nw] channels-last (== token-major [B*N, C]); pos: [1, 1, n_pos, C]; cls: [1, 1, C] or None.  Returns [B, N(+1), C].
    The table is linearly resampled to the patch count N inside the kernel, as the reference's F.interpolate does
    (cvnets/layers/positional_embedding.py:90-95); at N == n_pos (224 x 224 inputs) the resample is the identity."""

    @staticmethod
    def forward(ctx, patch, cfg, pos, cls):
        B, C, nh, nw = patch.shape
        N, n_pos = nh * nw, pos.shape[-2]
        p2 = as_2d(to_bf16_cl(patch))
        out = ops.vit_tokens_interp_fwd(p2, pos, cls, B, N, C)
        ctx.cfg, ctx.dims, ctx.plist, ctx.has_cls = cfg, (B, C, nh, nw, n_pos), cfg.plist, cls is not None
        return out

    @staticmethod
    def backward(ctx, gout):
        B, C, nh, nw, n_pos = ctx.dims
        N = nh * nw
        g = gout.to(BF16).contiguous()
        D = _Dst(ctx.cfg, ctx.plist, g.device, True)
        dpos = D.mat(0, n_pos, C)
        dcls = D.mat(1, 1, C).view(C) if ctx.has_cls else None
        dpatch = ops.vit_tokens_interp_bwd(g, dpos, dcls, B, N, C)
        grads = D.finish()
        return to_4d(dpatch, B, nh, nw), None, grads[0], grads[1] if ctx.has_cls else None


# ==================================================================================================================
# CLIP edges (BASELINE.json configs[4]): text embedding, end-of-text gather, projection, feature normalisation, contrastive loss
# ==================================================================================================================
class EmbeddingFn(torch.autograd.Function):
    """token embedding + learnable positional embedding (cvnets/text_encoders/transformer.py:328-341).  params = (table [V, C], pos [1,1,S,C] | None)."""

    @staticmethod
    def forward(ctx, tokens, cfg, table, pos):
        out = ops.embedding_fwd(tokens, table, pos)
        ctx.cfg, ctx.plist, ctx.tokens, ctx.shape, ctx.has_pos = cfg, cfg.plist, tokens, tuple(table.shape), pos is not None
        return out

    @staticmethod
    def backward(ctx, g):
        V, C = ctx.shape
        B, S = ctx.tokens.shape
        g = g.to(BF16).contiguous()
        D = _Dst(ctx.cfg, ctx.plist, g.device, True)
        dtable = D.mat(0, V, C)
        dpos = D.mat(1, S, C) if ctx.has_pos else None
        ops.embedding_bwd(g, ctx.tokens, dtable, dpos)
        grads = D.finish()
        return None, None, grads[0], grads[1] if ctx.has_pos else None


class EotGatherFn(torch.autograd.Function):
    """x[arange(B), tokens.argmax(-1)] (transformer.py:413-421): the end-of-text token carries the sequence feature."""

    @staticmethod
    def forward(ctx, x, tokens):
        B, S, C = x.shape
        x = x.to(BF16).contiguous()
        out, idx = ops.eot_gather_fwd(x, tokens)
        ctx.dims, ctx.idx = (B, S, C), idx
        return out

    @staticmethod
    def backward(ctx, g):
        B, S, C = ctx.dims
        g = g.to(BF16).contiguous()
        return ops.eot_gather_bwd(g, ctx.idx, B, S, C), None


class ProjectionFn(torch.autograd.Function):
    """y = x @ P with a parameter stored [in, out] (TextTransformer.projection_layer, transformer.py:159-161, 422; SimpleImageProjectionHead.proj)."""

    @staticmethod
    def forward(ctx, x, cfg, P):
        x2 = x if (x.dtype == BF16 and x.stride(-1) == 1 and x.stride(0) % 8 == 0) else x.to(BF16).contiguous()
        y = ops.pw_gemm(x2, cfg.prep.get(cfg.i_pt), P.shape[1])
        ctx.cfg, ctx.plist, ctx.saved, ctx.shape = cfg, cfg.plist, (x2,), tuple(P.shape)
        return y

    @staticmethod
    def backward(ctx, g):
        din, dout = ctx.shape
        (x2,) = ctx.saved
        g = g.to(BF16).contiguous()
        D = _Dst(ctx.cfg, ctx.plist, g.device, True)
        ops.pw_wgrad_side(x2, g, din, dout, dW=D.mat(0, din, dout))
        dx = ops.pw_gemm(g, ctx.cfg.prep.get(ctx.cfg.i_p), din, K=dout)
        ops.join_side()
        return (dx, None) + D.finish()


class L2NormFn(torch.autograd.Function):
    """F.normalize(x, dim=-1) (transformer.py:423-425)."""

    @staticmethod
    def forward(ctx, x):
        x = x.to(BF16).contiguous()
        y, inv = ops.l2norm_fwd(x)
        # y is also the OUTPUT: keeping that very object on ctx would close a reference cycle (output -> grad_fn -> ctx -> output) that keeps the
        # whole step's autograd graph -- and the leaf accumulators with the stream they were created on -- alive into the next step
        ctx.saved = (y.detach(), inv)
        return y

    @staticmethod
    def backward(ctx, g):
        y, inv = ctx.saved
        g = g.to(BF16).contiguous()
        return ops.l2norm_bwd(g, y, inv)


def _padded_rows(G: int, G8: int, d: int, device) -> torch.Tensor:
    """bf16 [G8, d] whose rows G..G8 are zero (one memset node); rows 0..G are the caller's to fill."""
    t = torch.empty((G8, d), device=device, dtype=BF16)
    if G8 > G:
        ops._lib().cvb_memset_zero(t[G:].data_ptr(), (G8 - G) * d * 2, ops._stream())
    return t


class ClipLossFn(torch.autograd.Function):
    """ContrastiveLossClip._forward_clip (loss_fn/multi_modal_img_text/contrastive_loss_clip.py:56-97) with gather_all_features
    (utils/third_party/ddp_functional_utils.py:334-357): logits_per_image = s * img @ all_text^T, logits_per_text = s * text @ all_img^T,
    s = clamp(exp(logit_scale), 0, 100); loss = (CE(logits_per_image, arange + N*rank) + CE(logits_per_text, .)) / 2.
    Data parallel: the features are all-gathered over NCCL in the forward and their gradients reduce-scattered in the backward (every rank
    must bring the same batch N, as the reference's gather does).

    Any global batch G = world * N: when G is not a multiple of 8 the gathered operands are [G8, d] buffers (G8 = G rounded up to 8) whose
    last rows are zero, so the logits GEMMs run at N = G8; the loss kernels read C = G columns of the [N, G8] logits and write zeros into the
    gradient's pad columns, so the pad adds nothing to the input gradients, and the weight gradients' pad rows are dropped (a view) before the
    reduce-scatter.  The feature dimension d must be a multiple of 8."""

    @staticmethod
    def forward(ctx, img, txt, logit_scale, cfg):
        import torch.distributed as dist
        N, d = img.shape
        if d % 8:
            raise NotImplementedError(f"contrastive loss: the feature dim ({d}) must be a multiple of 8")
        img = img.to(BF16).contiguous()
        txt = txt.to(BF16).contiguous()
        world, rank = cfg.world, cfg.rank
        G = world * N
        G8 = (G + 7) // 8 * 8
        if world > 1 or G8 != G:
            I_all, T_all = _padded_rows(G, G8, d, img.device), _padded_rows(G, G8, d, img.device)
            if world > 1:
                w1 = dist.all_gather_into_tensor(I_all[:G], img, group=cfg.group, async_op=True)
                w2 = dist.all_gather_into_tensor(T_all[:G], txt, group=cfg.group, async_op=True)
                w1.wait()
                w2.wait()
            else:
                I_all[:G].copy_(img)
                T_all[:G].copy_(txt)
        else:
            I_all, T_all = img, txt
        # one labels tensor per (N, rank), kept: a CUDA graph captured at one batch reads its own labels while other batches run
        cache = cfg.__dict__.setdefault("_labels", {})
        labels = cache.get((N, rank))
        if labels is None:
            labels = cache[(N, rank)] = torch.arange(N, device=img.device, dtype=torch.int64) + N * rank
        Li = ops.pw_gemm(img, T_all, G8)
        Lt = ops.pw_gemm(txt, I_all, G8)
        li, lse_i, nv_i = ops.ce_fwd(Li, G, labels, -1, 0.0, logit_scale=logit_scale)
        lt, lse_t, nv_t = ops.ce_fwd(Lt, G, labels, -1, 0.0, logit_scale=logit_scale)
        ctx.cfg, ctx.plist, ctx.dims = cfg, [logit_scale], (N, d, G)
        ctx.saved = (img, txt, I_all, T_all, Li, Lt, labels, lse_i, nv_i, lse_t, nv_t, logit_scale)
        return ((li + lt) * 0.5).view(())

    @staticmethod
    def backward(ctx, gout):
        import torch.distributed as dist
        cfg = ctx.cfg
        N, d, G = ctx.dims
        img, txt, I_all, T_all, Li, Lt, labels, lse_i, nv_i, lse_t, nv_t, p = ctx.saved
        g = (gout.float() * 0.5).contiguous()
        D = _Dst(cfg, ctx.plist, img.device, True)
        dp = D.mat(0, 1, 1)
        scale = getattr(cfg, "scale", None)
        G8 = I_all.shape[0]
        dLi = ops.ce_bwd(Li, G, labels, -1, 0.0, lse_i, nv_i, g, scale, G8, logit_scale=p, dlogit_scale=dp)
        dLt = ops.ce_bwd(Lt, G, labels, -1, 0.0, lse_t, nv_t, g, scale, G8, logit_scale=p, dlogit_scale=dp)
        dI = ops.pw_gemm(dLi, ops.transpose_bf16(T_all), d, K=G8)    # through the local rows of logits_per_image
        dT = ops.pw_gemm(dLt, ops.transpose_bf16(I_all), d, K=G8)
        dT_all = ops.pw_wgrad(dLi, img, G8, d)[:G]                    # fp32 [G, d]: through the gathered operand; pad rows dropped
        dI_all = ops.pw_wgrad(dLt, txt, G8, d)[:G]
        if cfg.world > 1:
            dT_part = torch.empty((N, d), device=img.device, dtype=torch.float32)
            dI_part = torch.empty((N, d), device=img.device, dtype=torch.float32)
            w1 = dist.reduce_scatter_tensor(dT_part, dT_all, op=dist.ReduceOp.SUM, group=cfg.group, async_op=True)
            w2 = dist.reduce_scatter_tensor(dI_part, dI_all, op=dist.ReduceOp.SUM, group=cfg.group, async_op=True)
            w1.wait()
            w2.wait()
        else:
            dT_part, dI_part = dT_all, dI_all
        dimg, dtxt = ops.add_bf16_f32(dI, dI_part), ops.add_bf16_f32(dT, dT_part)
        grads = D.finish()
        return dimg, dtxt, (grads[0].view(()) if grads[0] is not None else None), None


# ==================================================================================================================
# Transformer rows (SURVEY.md 8a a10-a12): MultiHeadAttention (cvnets/layers/multi_head_attention.py:135-239) and the pre-norm
# TransformerEncoder (cvnets/modules/transformer.py:129-156) on token matrices [M = N*S, C] (bf16).  LayerNorm is the GroupNorm
# load mode of the consuming GEMM with rows_per_sample = 1 (per-token statistics); its backward is the one-pass
# cvb_ln_bwd kernel behind a plain dX GEMM.  dropout / stochastic depth p = 0 (the module raises otherwise).
# ==================================================================================================================
def _masks(cfg_masks, N, S, device):
    """(attn_mask fp32 [N,S,S] or None, key_padding_mask uint8 [N,S] or None) in the layout cvb_mha_* reads."""
    amask, kpm = cfg_masks
    if amask is not None:
        if list(amask.shape) != [N, S, S]:
            raise ValueError(f"Shape of attention mask should be [{N}, {S}, {S}]. Got: {list(amask.shape)}")  # multi_head_attention.py:199-205
        amask = amask.to(device=device, dtype=torch.float32).contiguous()
    if kpm is not None:
        if kpm.dim() != 2 or list(kpm.shape) != [N, S]:
            raise ValueError(f"Key_padding_mask should be 2-dimension with shape [{N}, {S}]. Got: {list(kpm.shape)}")  # :213-219
        kpm = kpm.to(device=device).to(torch.uint8).contiguous()
    return amask, kpm


class MultiHeadAttentionFn(torch.autograd.Function):
    """Stand-alone self-attention: qkv_proj GEMM (+bias) -> attention core -> out_proj GEMM (+bias)."""

    @staticmethod
    def forward(ctx, x, cfg, wqkv, bqkv, wo, bo):
        N, S, C = x.shape
        P = cfg.prep
        x2 = x.reshape(N * S, C)
        amask, kpm = _masks(cfg.masks, N, S, x.device)
        qkv = ops.pw_gemm(x2, P.get(cfg.i_wqkv), 3 * C, bias=bqkv)
        O, LSE = ops.mha_fwd(qkv, N, S, cfg.heads, cfg.head_dim, cfg.scale, amask, kpm)
        y = ops.pw_gemm(O, P.get(cfg.i_wo), cfg.out_dim, bias=bo)
        ctx.cfg, ctx.dims = cfg, (N, S, C)
        ctx.saved = (x2, qkv, O, LSE, amask, kpm)
        return y.view(N, S, cfg.out_dim)

    @staticmethod
    def backward(ctx, gout):
        cfg = ctx.cfg
        N, S, C = ctx.dims
        P = cfg.prep
        x2, qkv, O, LSE, amask, kpm = ctx.saved
        dy = gout.reshape(N * S, cfg.out_dim).to(BF16).contiguous()
        dbo = torch.zeros(cfg.out_dim, device=dy.device, dtype=torch.float32)
        dWo = ops.pw_wgrad_side(dy, O, cfg.out_dim, C, dbias=dbo)
        dO = ops.pw_gemm(dy, P.get(cfg.i_wot), C, K=cfg.out_dim)
        dqkv = ops.mha_bwd(qkv, O, dO, LSE, N, S, cfg.heads, cfg.head_dim, cfg.scale, amask, kpm)
        dbq = torch.zeros(3 * C, device=dy.device, dtype=torch.float32)
        dWq = ops.pw_wgrad_side(dqkv, x2, 3 * C, C, dbias=dbq)
        dx = ops.pw_gemm(dqkv, P.get(cfg.i_wqkvt), C, K=3 * C)
        ops.join_side()
        return dx.view(N, S, C), None, dWq, dbq, dWo, dbo


def _encoder_forward(x2, N, S, cfg, amask, kpm, drop, keys=None, arena="fwd"):
    """One TransformerEncoder forward on the token matrix x2 [M = N*S, C] -> (output [M, C], what its backward needs).

    ``drop``: (p, p_ffn, p_row) in training with dropout / stochastic depth > 0, else None.  ``keys``: the mask keys an earlier forward of the
    same layer drew, to replay it bit for bit (a recompute), else new keys are drawn from the device generator.  ``arena``: the key of the
    call's statistics scratch (a recompute inside the backward carves a slice of its own)."""
    M, C = x2.shape
    ffn = cfg.ffn
    P = cfg.prep
    ln1 = ops.ln_stats(x2, cfg.eps)
    # wide layers (ViT / CLIP: K = 768 under 18-24 N tiles): the LayerNorm prologue is applied ONCE by a pre-pass (ops.WIDE_K / WIDE_N policy, which
    # pw_gemm would apply internally) and the normalised tokens are KEPT for the weight gradient of the same projection, which would otherwise
    # re-normalise them (one extra pass over the tokens per weight-gradient block)
    keep_n = C >= ops.WIDE_K and 3 * C >= ops.WIDE_N_WGRAD and ffn >= ops.WIDE_N_WGRAD
    g1, b1, _, bqkv, _, bo, g2, b2, _, bb1, _, bb2 = cfg.plist

    def ln_proj(X, ln, gamma, beta, weight, N, bias):
        """(LayerNorm(X) @ weight^T + bias, the kept normalised tokens or None)."""
        if not keep_n:
            return ops.pw_gemm(X, weight, N, a_mode=A_GN, a_p=(gamma, beta), row_stats=(ln[0], ln[1]), rows_per_sample=1, bias=bias), None
        xn = ops.apply_load_mode(X, A_GN, C, a_p=(gamma, beta), row_stats=(ln[0], ln[1]), rows_per_sample=1)
        return ops.pw_gemm(xn, weight, N, bias=bias), xn

    qkv, xn1 = ln_proj(x2, ln1, g1, b1, P.get(cfg.i_wqkv), 3 * C, bqkv)
    O, LSE = ops.mha_fwd(qkv, N, S, cfg.heads, cfg.head_dim, cfg.scale, amask, kpm)
    if drop is None:
        samp = _fwd_arena(cfg, x2.device, arena).f64(2, M)
        X1 = ops.pw_gemm(O, P.get(cfg.i_wo), C, bias=bo, R=x2, samp_stats=samp, rows_per_sample=1)
        ln2 = ops.gn_finalize(samp, C, cfg.eps)
    else:
        # the residual adds leave the GEMM epilogues: x + DropPath(Dropout(branch)) is one element-wise pass with hashed masks
        p, p_ffn, p_row = drop
        if keys is None:
            keys = (ops.rng_next(x2.device), ops.rng_next(x2.device), ops.rng_next(x2.device) if p_ffn > 0 else None)
        k1, k2, k3 = keys
        A = ops.pw_gemm(O, P.get(cfg.i_wo), C, bias=bo)
        X1 = ops.dropout_fwd(A, x2, p, k1, p_row=p_row, rows_per_sample=S)
        ln2 = ops.ln_stats(X1, cfg.eps)
    h, xn2 = ln_proj(X1, ln2, g2, b2, P.get(cfg.i_w1), ffn, bb1)
    if drop is None:
        if cfg.act == ops.ACT_SILU:
            ha = None
            X2 = ops.pw_gemm(h, P.get(cfg.i_w2), C, a_mode=A_SILU, bias=bb2, R=X1)
        else:
            ha = ops.act_fwd(h, cfg.act)
            X2 = ops.pw_gemm(ha, P.get(cfg.i_w2), C, bias=bb2, R=X1)
    else:
        ha = ops.act_fwd(h, cfg.act)
        if k3 is not None:
            ha = ops.dropout_fwd(ha, None, p_ffn, k3)
        Fo = ops.pw_gemm(ha, P.get(cfg.i_w2), C, bias=bb2)
        X2 = ops.dropout_fwd(Fo, X1, p, k2, p_row=p_row, rows_per_sample=S)
    return X2, SimpleNamespace(N=N, S=S, x2=x2, ln1=ln1, qkv=qkv, O=O, LSE=LSE, X1=X1, ln2=ln2, h=h, ha=ha, xn1=xn1, xn2=xn2,
                               amask=amask, kpm=kpm, drop=drop, keys=keys)


def _encoder_backward(st, dY, cfg, plist):
    """Backward of one ``_encoder_forward`` (``st``: what it returned) for the output gradient dY bf16 [M, C] -> (input gradient [M, C], the
    parameter gradients as ``_Dst.finish`` returns them).  ``plist``: the layer's parameters in TransformerEncoder._bind order."""
    N, S = st.N, st.S
    M, C = dY.shape
    ffn = cfg.ffn
    P = cfg.prep
    x2, ln1, qkv, O, LSE, X1, ln2, h, ha, amask, kpm = st.x2, st.ln1, st.qkv, st.O, st.LSE, st.X1, st.ln2, st.h, st.ha, st.amask, st.kpm
    g1, b1, g2, b2 = plist[0], plist[1], plist[6], plist[7]
    dev = x2.device
    # parameter order: (g1, b1, wqkv, bqkv, wo, bo, g2, b2, w1, bb1, w2, bb2)
    D = _Dst(cfg, plist, dev, True)
    ar = D.ar
    vec = lambda i, n: D.mat(i, 1, n).view(n)  # noqa: E731

    def ln_wgrad(G, xn, X, ln, gamma, beta, N, dW, dbias):
        """Weight gradient of the forward's ln_proj: on the kept normalised tokens, else through the LayerNorm load mode on X."""
        if xn is not None:
            return ops.pw_wgrad_side(G, xn, N, C, dW=dW, dbias=dbias)
        return ops.pw_wgrad_side(G, X, N, C, a_mode=A_GN, a_p=(gamma, beta), row_stats=(ln[0], ln[1]), rows_per_sample=1, dW=dW, dbias=dbias)

    # ---- FFN
    db2, db1 = vec(11, C), vec(9, ffn)
    drop = st.drop
    if drop is not None:
        p, p_ffn, p_row = drop
        k1, k2, k3 = st.keys
        dF = ops.dropout_bwd(dY, p, k2, p_row=p_row, rows_per_sample=S)  # gradient of the FFN branch; the residual path keeps dY
        ops.pw_wgrad_side(dF, ha, C, ffn, dW=D.mat(10, C, ffn), dbias=db2)
        dha = ops.pw_gemm(dF, P.get(cfg.i_w2t), ffn, K=C)
        if k3 is not None:
            dha = ops.dropout_bwd(dha, p_ffn, k3)
        dh = ops.act_bwd(dha, h, cfg.act)
    elif cfg.act == ops.ACT_SILU:
        ops.pw_wgrad_side(dY, h, C, ffn, a_mode=A_SILU, dW=D.mat(10, C, ffn), dbias=db2)
        dh = ops.pw_gemm(dY, P.get(cfg.i_w2t), ffn, K=C, e_mode=E_SILU_BWD, Y=h)
    else:
        ops.pw_wgrad_side(dY, ha, C, ffn, dW=D.mat(10, C, ffn), dbias=db2)
        dh = ops.act_bwd(ops.pw_gemm(dY, P.get(cfg.i_w2t), ffn, K=C), h, cfg.act)
    ln_wgrad(dh, st.xn2, X1, ln2, g2, b2, ffn, D.mat(8, ffn, C), db1)
    csf = ar.f64(2, C)
    vF = ops.pw_gemm(dh, P.get(cfg.i_w1t), C, K=ffn)
    if drop is None:
        bsum1 = ar.f64(C)
        dX1 = ops.ln_bwd(vF, X1, ln2, g2, csf, DRES=dY, col_sum=bsum1)  # bsum1 = column sums of dX1 = d(out_proj bias)
        D.late64(5, bsum1)
        dA = dX1
        dbo = None
    else:
        dX1 = ops.ln_bwd(vF, X1, ln2, g2, csf, DRES=dY)
        dA = ops.dropout_bwd(dX1, p, k1, p_row=p_row, rows_per_sample=S)  # gradient of the attention branch (out_proj output)
        dbo = vec(5, C)
    D.late64(6, csf[1])
    D.late64(7, csf[0])
    # ---- attention
    ops.pw_wgrad_side(dA, O, C, C, dW=D.mat(4, C, C), dbias=dbo)
    dO = ops.pw_gemm(dA, P.get(cfg.i_wot), C, K=C)
    dqkv = ops.mha_bwd(qkv, O, dO, LSE, N, S, cfg.heads, cfg.head_dim, cfg.scale, amask, kpm)
    ln_wgrad(dqkv, st.xn1, x2, ln1, g1, b1, 3 * C, D.mat(2, 3 * C, C), vec(3, 3 * C))
    csa = ar.f64(2, C)
    vA = ops.pw_gemm(dqkv, P.get(cfg.i_wqkvt), C, K=3 * C)
    dx = ops.ln_bwd(vA, x2, ln1, g1, csa, DRES=dX1)
    D.late64(0, csa[1])
    D.late64(1, csa[0])
    ops.join_side()
    return dx, D.finish()


class TransformerEncoderFn(torch.autograd.Function):
    """x = x + MHA(LN1(x));  x = x + W2 act(W1 LN2(x) + b1) + b2   (transformer.py:139-156)."""

    @staticmethod
    def forward(ctx, x, cfg, *params):
        N, S, C = x.shape
        amask, kpm = _masks(cfg.masks, N, S, x.device)
        X2, ctx.st = _encoder_forward(x.reshape(N * S, C), N, S, cfg, amask, kpm, getattr(cfg, "drop", None))
        ctx.cfg, ctx.plist = cfg, cfg.plist
        return X2.view(N, S, C)

    @staticmethod
    def backward(ctx, gout):
        N, S, C = gout.shape
        dx, grads = _encoder_backward(ctx.st, gout.reshape(N * S, C).to(BF16).contiguous(), ctx.cfg, ctx.plist)
        return (dx.view(N, S, C), None) + grads


class EncoderRunFn(torch.autograd.Function):
    """A run of TransformerEncoder layers with recomputing gradient checkpointing (what torch.utils.checkpoint does for the reference,
    vit.py:526-533, text_encoders/transformer.py:390-401): the forward keeps only the run's input and each layer's mask keys, the backward
    re-runs the run's forward from them -- bit for bit the same activations, every forward kernel being deterministic -- and then each
    layer's backward, last layer first.  torch's checkpoint would restore torch's RNG state, not the library's device-side generator, so the
    dropout / stochastic-depth masks are replayed from the saved keys instead.  ``run.cfgs``: the layers' cfgs as TransformerEncoder.prepare
    left them; ``params``: their parameter lists, concatenated."""

    @staticmethod
    def forward(ctx, x, run, *params):
        N, S, C = x.shape
        x2 = y = x.reshape(N * S, C)
        layers = []
        for cfg in run.cfgs:
            amask, kpm = _masks(cfg.masks, N, S, x.device)
            drop = getattr(cfg, "drop", None)
            y, st = _encoder_forward(y, N, S, cfg, amask, kpm, drop)
            layers.append((cfg, cfg.plist, amask, kpm, drop, st.keys))
            del st
        ctx.x2, ctx.layers = x2, layers
        return y.view(N, S, C)

    @staticmethod
    def backward(ctx, gout):
        N, S, C = gout.shape
        y, sts = ctx.x2, []
        for cfg, _, amask, kpm, drop, keys in ctx.layers:
            y, st = _encoder_forward(y, N, S, cfg, amask, kpm, drop, keys=keys, arena="rfwd")
            sts.append(st)
        del y
        dY = gout.reshape(N * S, C).to(BF16).contiguous()
        grads = []
        for cfg, plist, *_ in reversed(ctx.layers):
            dY, g = _encoder_backward(sts.pop(), dY, cfg, plist)  # the layer's activations are released as soon as its backward is issued
            grads.append(g)
        return (dY.view(N, S, C), None) + tuple(gp for g in reversed(grads) for gp in g)

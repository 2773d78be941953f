"""EfficientNet at training-size grids (-m gpu): the kernels it adds (5x5 depthwise walk kernels, squeeze-excitation scaling, stochastic
depth, the SGD step) at the batch sizes and widths b0 .. b7 train with, every mode end to end, and the b0 SGD step bit for bit.

Kernel level, as test_reproducible_gpu.py: inputs are rounded to bf16, each call is compared with an fp64 torch restatement of the same
operation, and every call whose grid loops over work (a CTA's batch loop, a grid-capped element loop) runs twice and must be torch.equal.
The batch sizes come from the SM count through a restatement of the host-side grid formula, so each CTA runs several images unevenly.

Widths past 2048 channels (the b2 .. b7 squeeze-excitation units, depthwise convs and BatchNorms) run on a second grid dimension of
2048-channel chunks; they are called directly at C = 2056 .. 3840.

Model level: b0 .. b7 train-mode forward / backward at 64^2 against the fp32 restatement (tests/efficientnet_ref.py), with the
autocast-relative bounds of test_efficientnet_gpu.py, and eval-mode logits at each recipe's resolution.  Step level: three SGD-Nesterov
TrainStep steps of b0 with stochastic depth, eager twice, without programmatic dependent launch, without the weight-gradient side stream
and replayed from a CUDA graph, all in the same bits."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import efficientnet_ref as E  # noqa: E402
from oracle import cvnets_oracle as O  # noqa: E402
from test_kernels_gpu import bf, close, close_stat, dsilu, load_ref, rnd  # noqa: E402
from test_kernels_edges_gpu import same  # noqa: E402
from test_reproducible_gpu import passes, twice, zeros64  # noqa: E402

pytestmark = pytest.mark.gpu

F64 = torch.float64


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


def rel_l2(a, b):
    a, b = a.detach().double(), b.detach().double()
    return float((a - b).norm() / (b.norm() + 1e-30))


# ------------------------------------------------------------------------------------------- 5x5 depthwise walk kernels, batch loop
def dw_grid(H, W, C, s, K, sms, bwd):
    """the walk kernels' grid (dwconv.cu, cvb_dw_fwd / cvb_dw_bwd): TW x TH output tiles x 64-channel blocks per image, and the batch split
    gz = ceil(8 #SM / per_img) forward, ceil(4 #SM / per_img) backward.  The 5x5 tiles are 8 rows high at both strides."""
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    TW = (16 if Wo > 8 else 8) if bwd else (16 if (s == 1 and Wo > 8) else 8)
    TH = (16 if Ho > 8 else 8) if (s == 1 and K == 3) else 8
    per_img = math.ceil(Ho / TH) * math.ceil(Wo / TW) * math.ceil(C / 64)
    return math.ceil((4 if bwd else 8) * sms / per_img)


def dw_batch(gz):
    """B = 3 gz + 1: every CTA's batch loop runs three images, the first CTA of each tile a fourth"""
    B = 3 * gz + 1
    passes(B, gz)
    return B


def dwk_ref_fwd(xa, wk, s, K):
    """xa: activated input [B, H, W, C] fp64, wk: [K*K, C] (tap u * K + v) -> [B, Ho, Wo, C]; pad (K - 1) / 2, stride s"""
    B, H, W, C = xa.shape
    P = (K - 1) // 2
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    xp = F.pad(xa, (0, 0, P, P, P, P))
    y = torch.zeros(B, Ho, Wo, C, device=xa.device, dtype=F64)
    for u in range(K):
        for v in range(K):
            y += wk[K * u + v] * xp[:, u:u + s * (Ho - 1) + 1:s, v:v + s * (Wo - 1) + 1:s]
    return y


def dwk_ref_bwd(xa, dy, wk, s, K):
    """adjoint of dwk_ref_fwd: (d xa [B, H, W, C], dW [K*K, C])"""
    B, H, W, C = xa.shape
    P = (K - 1) // 2
    Ho, Wo = dy.shape[1:3]
    xp = F.pad(xa, (0, 0, P, P, P, P))
    dxp = torch.zeros_like(xp)
    dw = torch.empty(K * K, C, device=xa.device, dtype=F64)
    for u in range(K):
        for v in range(K):
            sl = (slice(None), slice(u, u + s * (Ho - 1) + 1, s), slice(v, v + s * (Wo - 1) + 1, s))
            dw[K * u + v] = (xp[sl] * dy).sum((0, 1, 2))
            dxp[sl] += wk[K * u + v] * dy
    return dxp[:, P:P + H, P:P + W], dw


def _dw5_params(C, seed):
    Wt = bf(rnd(25, C, scale=0.2, seed=seed)).float()
    xp = (1 + 0.2 * rnd(C, seed=seed + 1), 0.3 * rnd(C, seed=seed + 2))
    gp = (1 + 0.2 * rnd(C, seed=seed + 3), 0.3 * rnd(C, seed=seed + 4), 0.1 * rnd(C, seed=seed + 5))
    return Wt, xp, gp


def _check_dw5_fwd(ops, B, H, C, s, x_mode, seed):
    W = H
    X = bf(rnd(B * H * W, C, seed=seed))
    Wt, xp, _ = _dw5_params(C, seed + 10)

    def run():
        col = zeros64(2, C)
        Y = ops.dw_fwd(X, B, H, W, C, s, Wt, x_mode=x_mode, x_p=xp, col_stats=col, ksize=5)
        return Y, col

    Y, col = twice(run, ("Y", "col_stats"))
    xa = load_ref(x_mode, X, xp + (None,)).double().view(B, H, W, C)
    ref = dwk_ref_fwd(xa, Wt.double(), s, 5).view(-1, C)
    close(Y, ref, what="dw5 fwd")
    o = Y.double()
    close_stat(col[0], o.sum(0), "col_sum")
    close_stat(col[1], (o * o).sum(0), "col_sq")


def _check_dw5_bwd(ops, B, H, C, s, g_mode, x_mode, seed):
    W = H
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    X = bf(rnd(B * H * W, C, seed=seed))
    DZ, Y2 = bf(rnd(B * Ho * Wo, C, seed=seed + 1)), bf(rnd(B * Ho * Wo, C, seed=seed + 2))
    Wt, xp, gp = _dw5_params(C, seed + 10)

    def run():
        col = zeros64(2, C)
        DX, dWt = ops.dw_bwd(DZ, X, B, H, W, C, s, Wt, g_mode=g_mode, Y2=Y2 if g_mode == ops.A_BNB else None, g_p=gp, x_mode=x_mode, x_p=xp,
                             col_stats=col if x_mode != ops.A_RAW else None, ksize=5)
        return DX, dWt, col

    DX, dWt, col = twice(run, ("dX", "dW", "col_stats"))
    dy = load_ref(g_mode, DZ, gp, Y2).double().view(B, Ho, Wo, C)
    xa = load_ref(x_mode, X, xp + (None,)).double().view(B, H, W, C)
    da, dw = dwk_ref_bwd(xa, dy, Wt.double(), s, 5)
    da = da.reshape(-1, C)
    if x_mode == ops.A_AFF_SILU:
        da = da * dsilu(xp[0].double() * X.double() + xp[1].double())
    close(DX, da, what="dX")
    close(dWt, dw, rtol=3e-3, atol=3e-3 * float(dw.abs().max()) + 1e-5, what="dW")
    if x_mode != ops.A_RAW:
        # interior tiles' statistics come from the fp32 values, edge tiles' from the stored ones (test_dw_bwd)
        close_stat(col[0], da.sum(0), "sum dz", rtol=6e-3)
        close_stat(col[1], (da * X.double()).sum(0), "sum dz*x", rtol=6e-3)


# every 5x5 layer of EfficientNet-b0 at 224^2: (H_in, C, stride)
DW5_LAYERS = [(56, 144, 2), (28, 240, 1), (14, 480, 1), (14, 672, 1), (14, 672, 2), (7, 1152, 1)]


@pytest.mark.parametrize("H,C,s", DW5_LAYERS)
@pytest.mark.parametrize("x_mode", [0, 1, 2])
def test_dw5_fwd_batch_loop(ops, sms, H, C, s, x_mode):
    B = dw_batch(dw_grid(H, H, C, s, 5, sms, bwd=False))
    _check_dw5_fwd(ops, B, H, C, s, x_mode, seed=2000 + H + C + s)


@pytest.mark.parametrize("H,C,s", DW5_LAYERS)
@pytest.mark.parametrize("g_mode,x_mode", [(0, 0), (5, 0), (0, 1), (5, 1), (0, 2), (5, 2)])
def test_dw5_bwd_batch_loop(ops, sms, H, C, s, g_mode, x_mode):
    B = dw_batch(dw_grid(H, H, C, s, 5, sms, bwd=True))
    _check_dw5_bwd(ops, B, H, C, s, g_mode, x_mode, seed=2100 + H + C + s)


# stride 2 on odd maps at the b1 .. b3 recipe sizes: b1 layer_5 (15 -> 8), b2 layer_3 / layer_5 (65 -> 33, 17 -> 9), b3 layer_3 (75 -> 38)
@pytest.mark.parametrize("H,C", [(15, 672), (65, 144), (17, 720), (75, 192)])
def test_dw5_fwd_stride2_odd_batch_loop(ops, sms, H, C):
    B = dw_batch(dw_grid(H, H, C, 2, 5, sms, bwd=False))
    _check_dw5_fwd(ops, B, H, C, 2, 2, seed=2200 + H + C)


def test_dw5_bwd_stride2_odd_still_rejected(ops):
    """the stride-2 backward on odd maps is not implemented (DESIGN.md section 7): a clear error, not a wrong gradient"""
    from ml_cvnets_b200 import _lib as L
    B, H, C = 2, 15, 64
    x = torch.zeros(B * H * H, C, device="cuda", dtype=torch.bfloat16)
    with pytest.raises(L.CvbError):
        ops.dw_bwd(torch.zeros(B * 8 * 8, C, device="cuda", dtype=torch.bfloat16), x, B, H, H, C, 2, torch.zeros(25, C, device="cuda"), ksize=5)


# ------------------------------------------------------------------------------------------- squeeze-excitation scaling
def _check_se(ops, B, HW, C, seed):
    X = bf(rnd(B * HW, C, seed=seed))
    S = bf(torch.sigmoid(rnd(B, C, seed=seed + 1)))
    DY = bf(rnd(B * HW, C, seed=seed + 2))

    def run():
        Y = ops.se_scale_fwd(X, S, B, HW)
        DX, DS = ops.se_scale_bwd(DY, X, S, B, HW)
        return Y, DX, DS

    Y, DX, DS = twice(run, ("Y", "dX", "dS"))
    s = S.float().repeat_interleave(HW, 0)
    # a bf16 x bf16 product is exact in fp32: the kernel's one rounding to bf16 is torch's
    same(Y, (X.float() * s).to(torch.bfloat16), "Y = X * S")
    same(DX, (DY.float() * s).to(torch.bfloat16), "dX = dY * S")
    ref = (DY.double() * X.double()).view(B, HW, C).sum(1)
    close(DS, ref, rtol=1e-4, atol=1e-5 * float(ref.abs().max()) + 1e-6, what="dS", rel_l2=1e-5)


def se_strips(B, HW, sms):
    """cvb_se_scale_* grid (se.cu, se_geometry): strips of >= 32 pixels, ~4 #SM CTAs over B samples"""
    s = math.ceil(4 * sms / B)
    rpc = max(32, math.ceil(HW / s))
    return math.ceil(HW / rpc)


# the b0 squeeze-excitation inputs (the depthwise output map): layer_1 (32 @ 112^2), layer_2.0 (96 @ 56^2) .. layer_5 (1152 @ 7^2); 144, 240,
# 480 and 672 are not multiples of 64
SE_SHAPES = [(112, 32, 16), (56, 96, 48), (56, 144, 64), (28, 144, 64), (28, 240, 64), (14, 240, 64), (14, 480, 128), (14, 672, 128),
             (7, 672, 256), (7, 1152, 256)]


@pytest.mark.parametrize("H,C,B", SE_SHAPES)
def test_se_scale_b0_shapes(ops, sms, H, C, B):
    """DS of each (sample, channel) is the sum of several CTAs' strips (fp64 scratch), and of the pixel lanes inside a CTA: bitwise twice"""
    HW = H * H
    assert se_strips(B, HW, sms) >= 2
    _check_se(ops, B, HW, C, seed=2300 + H + C)


# ------------------------------------------------------------------------------------------- widths past 2048 channels
WIDE = [2056, 2112, 2304, 3456, 3840]


@pytest.mark.parametrize("C", WIDE)
def test_se_scale_wide(ops, C):
    _check_se(ops, 6, 100, C, seed=2400 + C)


@pytest.mark.parametrize("C", WIDE)
def test_global_pool_fwd_wide(ops, C):
    B, HW = 5, 81
    X = bf(rnd(B * HW, C, seed=2500 + C) + 0.2)
    p = twice(lambda: (ops.global_pool_fwd(X, B, HW),), ("pool",))[0]
    close(p, X.double().view(B, HW, C).mean(1), what="pool fwd")


@pytest.mark.parametrize("C", WIDE)
def test_bn_bwd_reduce_wide(ops, C):
    M = 3001
    D, Y = bf(rnd(M, C, seed=2600 + C)), bf(rnd(M, C, seed=2601 + C) * 1.5 + 0.3)
    bn = torch.stack([rnd(C, seed=2602), rnd(C, seed=2603).abs() + 0.5, 1 + 0.2 * rnd(C, seed=2604), 0.3 * rnd(C, seed=2605)])

    def run():
        st, st2 = zeros64(2, C), zeros64(2, C)
        ops.bn_bwd_reduce(D, Y, st)
        dz = ops.bn_bwd_reduce(D, Y, st2, bn, act=True, store_dz=True)
        return st, st2, dz

    st, st2, dz = twice(run, ("stats", "stats (act)", "dz"))
    d, y = D.double(), Y.double()
    close_stat(st[0], d.sum(0), "sum dz")
    close_stat(st[1], (d * y).sum(0), "sum dz*y")
    close(dz, d * dsilu(y * bn[2].double() + bn[3].double()), what="dz")
    close_stat(st2[0], dz.double().sum(0), "sum dz (act)")
    close_stat(st2[1], (dz.double() * y).sum(0), "sum dz*y (act)")


@pytest.mark.parametrize("K,N", [(3456, 144), (3840, 160), (3072, 128)])
def test_pw_gemm_se_reduce_wide_k(ops, K, N):
    """the b5 .. b7 squeeze-excitation reduce convs (pooled [B, K] -> N squeeze channels, bias): K too large for the mma.sync kernel's
    resident weight panel at a narrow N, so the wgmma kernel streams the weights"""
    B = 16
    A = bf(rnd(B, K, seed=2700 + K))
    W = bf(rnd(N, K, scale=K ** -0.5, seed=2701 + K))
    bias = rnd(N, seed=2702 + K)
    out = ops.pw_gemm(A, W, N, bias=bias)
    close(out, A.double() @ W.double().t() + bias.double(), what="se reduce")


# ------------------------------------------------------------------------------------------- SGD past its grid cap
class _SgdTail:
    """flat fp32 buffers for cvb_grad_norm + cvb_sgd_step"""

    def __init__(self, lib, n, wd, *, momentum, nesterov, lr=0.1, max_norm=10.0, growth_interval=2, ema=0.1, seed=0):
        self.lib, self.n = lib, n
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.p = torch.randn(n, device="cuda", generator=g)
        self.buf = torch.zeros(n, device="cuda")
        self.wd = wd
        self.ema = self.p.clone()
        self.ema_m = float(ema)
        self.stats = torch.zeros(4, device="cuda")
        self.partials = torch.zeros(2 * lib.cvb_grad_norm_blocks(n), device="cuda")
        self.scale = torch.tensor([65536.0, 0.0], device="cuda")
        self.step_count = torch.zeros(1, device="cuda")
        self.hp = torch.tensor([lr], device="cuda")
        self.momentum, self.nesterov = float(momentum), int(nesterov)
        self.max_norm, self.gi = float(max_norm), int(growth_interval)

    def step(self, grads):
        st = torch.cuda.current_stream().cuda_stream
        self.lib.cvb_grad_norm(grads.data_ptr(), self.n, self.scale.data_ptr(), 1.0, self.stats.data_ptr(), self.partials.data_ptr(), st)
        self.lib.cvb_sgd_step(self.p.data_ptr(), grads.data_ptr(), self.buf.data_ptr(), self.wd.data_ptr(), self.n, self.hp.data_ptr(),
                              self.momentum, self.nesterov, self.max_norm, self.stats.data_ptr(), self.scale.data_ptr(),
                              self.step_count.data_ptr(), 2.0, 0.5, self.gi, self.ema.data_ptr(), self.ema_m, self.partials.data_ptr(), st)

    def state(self):
        return [t.clone() for t in (self.p, self.buf, self.stats, self.scale, self.step_count, self.partials, self.ema)]


class _RefSgd:
    """GradScaler.unscale_ -> clip_grad_norm_ -> torch.optim.SGD(foreach=False) per weight-decay group -> GradScaler.update, and the EMA, in fp64"""

    def __init__(self, p0, wd, *, momentum, nesterov, lr=0.1, max_norm=10.0, growth_interval=2, ema=0.1):
        f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))  # noqa: E731  (the kernel receives fp32 hyper-parameters)
        self.wds = torch.unique(wd).tolist()
        self.groups = [(wd == w).nonzero().squeeze(1) for w in self.wds]
        self.params = [torch.nn.Parameter(p0.double()[idx].clone()) for idx in self.groups]
        self.opt = torch.optim.SGD([{"params": [p], "weight_decay": w} for p, w in zip(self.params, self.wds)], lr=f32(lr), momentum=f32(momentum),
                                   nesterov=nesterov, foreach=False)
        self.n = p0.numel()
        self.scale, self.tracker, self.gi, self.max_norm = 65536.0, 0, growth_interval, max_norm
        self.ema, self.ema_m = p0.double().clone(), f32(ema)
        self.clipped = []

    def _gather(self, get):
        out = torch.zeros(self.n, device="cuda", dtype=F64)
        for idx, p in zip(self.groups, self.params):
            v = get(p)
            if v is not None:
                out[idx] = v
        return out

    def flat(self):
        return self._gather(lambda p: p.detach())

    def momentum_buffer(self):
        return self._gather(lambda p: self.opt.state.get(p, {}).get("momentum_buffer"))

    def step(self, grads):
        g = grads.double() / self.scale
        if bool(torch.isfinite(g).all()):
            coef = min(1.0, self.max_norm / (float(g.norm()) + 1e-6))
            self.clipped.append(coef < 1.0)
            for idx, p in zip(self.groups, self.params):
                p.grad = g[idx] * coef
            self.opt.step()
            self.tracker += 1
            if self.tracker >= self.gi:
                self.scale, self.tracker = self.scale * 2.0, 0
        else:
            self.scale, self.tracker = self.scale * 0.5, 0
        self.ema = self.ema * (1 - self.ema_m) + self.ema_m * self.flat()


def _sgd_n(sms):
    """cvb_sgd_step runs min(ceil(n / 256), 8 #SM) blocks of 256 (optim.cu): three passes and a remainder"""
    cap = 8 * sms * 256
    n = 3 * cap + 5 * 256 + 3
    passes(n, cap)
    return n


@pytest.mark.parametrize("momentum,nesterov", [(0.9, True), (0.9, False), (0.0, False)], ids=["nesterov", "momentum", "plain"])
def test_grad_norm_sgd_step_past_grid_cap(ops, sms, momentum, nesterov):
    """weight decay with zeros (the no_decay_bn_filter_bias group), EMA, clipping active then inactive, an inf and a NaN step (skipped: scale
    backed off, EMA still moving) and loss-scale growth every second finite step; the whole sequence twice, bitwise"""
    from ml_cvnets_b200 import _lib as L
    lib = L.load()
    n = _sgd_n(sms)
    idx = torch.arange(n, device="cuda")
    wd = torch.where(idx % 3 == 0, torch.tensor(4e-5, device="cuda"), torch.where(idx % 3 == 1, torch.tensor(1e-2, device="cuda"),
                                                                                    torch.tensor(0.0, device="cuda")))
    # loss scale at each step: growth_interval 2 doubles it after two finite steps, each non-finite step halves it
    scales = [65536.0, 65536.0, 32768.0, 32768.0, 16384.0, 16384.0, 32768.0]
    mags = [0.05, 0.05, 0.05, 0.05, 0.002, 0.05, 0.002]  # unscaled norms ~ 0.05 sqrt(n) > max_norm (clipped) and ~ 0.002 sqrt(n) < max_norm
    gen = torch.Generator(device="cuda").manual_seed(2801)
    grads = []
    for it, (sc, mg) in enumerate(zip(scales, mags)):
        g = torch.randn(n, device="cuda", generator=gen) * sc * mg
        if it == 1:
            g[n - 1000] = float("inf")  # inside the last block's range of the grid-stride loop
        if it == 3:
            g[n - 1] = float("nan")  # the n % 4 scalars after grad_norm's last float4
        grads.append(g)
    kw = dict(momentum=momentum, nesterov=nesterov)

    def run():
        tail = _SgdTail(lib, n, wd, seed=2802, **kw)
        for g in grads:
            tail.step(g)
        return tail.state()

    twice(run, ("params", "momentum", "stats", "scale", "step", "partials", "ema"))
    tail = _SgdTail(lib, n, wd, seed=2802, **kw)
    ref = _RefSgd(tail.p, wd, **kw)
    for it, g in enumerate(grads):
        tail.step(g)
        ref.step(g)
        torch.cuda.synchronize()
        rp = ref.flat()
        err = float((tail.p.double() - rp).abs().max())
        assert err <= 2e-6 + 1e-5 * float(rp.abs().max()), f"step {it}: params max abs diff {err}"
        if momentum > 0:
            rb = ref.momentum_buffer()
            e = float((tail.buf.double() - rb).abs().max())
            assert e <= 1e-5 * float(rb.abs().max()) + 1e-9, f"step {it}: momentum buffer max abs diff {e}"
        e = float((tail.ema.double() - ref.ema).abs().max())
        assert e <= 2e-6 + 1e-5 * float(ref.ema.abs().max()), f"step {it}: EMA max abs diff {e}"
        assert float(tail.scale[0]) == ref.scale and int(tail.scale[1]) == ref.tracker, (it, tail.scale.tolist(), ref.scale, ref.tracker)
        assert float(tail.stats[1]) == (1.0 if it in (1, 3) else 0.0), (it, float(tail.stats[1]))
    assert ref.clipped == [True, True, False, True, False], ref.clipped
    assert float(tail.step_count) == 5.0 and float(tail.scale[0]) == 32768.0


def test_train_step_sgd_clipped_vs_torch(pkg):
    """One TrainStep(optimizer="sgd", max_norm=...) step of EfficientNet-b0 with an active clip: the parameter update is clip_grad_norm_ +
    torch.optim.SGD (Nesterov, the no-decay group for BatchNorm / bias) applied in fp64 to the gradients the step computed"""
    torch.manual_seed(0)
    model = pkg.EfficientNet(pkg.default_effnet_opts("b0", n_classes=16)).cuda()
    lr, mu, wdv, max_norm = 0.1, 0.9, 4e-5, 0.5
    ts = pkg.TrainStep(model, optimizer="sgd", lr=lr, momentum=mu, nesterov=True, weight_decay=wdv, max_norm=max_norm, label_smoothing=0.1)
    g = torch.Generator(device="cuda").manual_seed(2901)
    x = torch.randn(8, 3, 64, 64, device="cuda", generator=g)
    y = torch.randint(0, 16, (8,), device="cuda", generator=g)
    p0, scale0 = ts.opt.flat_p.clone(), float(ts.opt.scale[0])
    ts.step(x, y)
    torch.cuda.synchronize()
    gr = ts.opt.flat_g.double() / scale0
    assert bool(torch.isfinite(gr).all())
    coef = max_norm / (float(gr.norm()) + 1e-6)
    assert coef < 1.0, "the clip must be active for this test"
    f32 = lambda v: float(torch.tensor(v, dtype=torch.float32))  # noqa: E731
    wd = ts.opt.wd
    assert float(wd.min()) == 0.0 and f32(wdv) == float(wd.max())
    groups = [(wd == w).nonzero().squeeze(1) for w in torch.unique(wd).tolist()]
    params = [torch.nn.Parameter(p0.double()[i].clone()) for i in groups]
    opt = torch.optim.SGD([{"params": [p], "weight_decay": float(wd[i[0]])} for p, i in zip(params, groups)], lr=f32(lr), momentum=f32(mu),
                          nesterov=True, foreach=False)
    for p, i in zip(params, groups):
        p.grad = gr[i] * coef
    opt.step()
    want = torch.zeros_like(gr)
    for p, i in zip(params, groups):
        want[i] = p.detach()
    err = float((ts.opt.flat_p.double() - want).abs().max())
    assert err <= 2e-6 + 1e-5 * float(want.abs().max()), err
    assert rel_l2(ts.opt.flat_p - p0, want - p0.double()) <= 1e-4


# ------------------------------------------------------------------------------------------- stochastic depth at b0 sizes
@pytest.mark.parametrize("rps,C", [(3136, 24), (784, 40), (196, 112)])
def test_stochastic_depth_b0_sizes(ops, rps, C):
    """Y = X + factor * V with one factor per sample (0 or 1 / (1 - p); p = 0.2 makes it 1.25, exact in bf16), over B = 256 samples of a b0
    map; the backward regenerates the same mask.  Outputs are exactly X or bf16(X + 1.25 V), gradients exactly 0 or bf16(1.25 dY)."""
    B, p = 256, 0.2
    M = B * rps
    V, X, DY = bf(rnd(M, C, seed=3000 + rps)), bf(rnd(M, C, seed=3001 + rps)), bf(rnd(M, C, seed=3002 + rps))
    key = torch.tensor([0x5DEECE66D + rps], device="cuda", dtype=torch.int64)

    def run():
        Y = ops.dropout_fwd(V, X, 0.0, key, p_row=p, rows_per_sample=rps)
        DV = ops.dropout_bwd(DY, 0.0, key, p_row=p, rows_per_sample=rps)
        fac = ops.dropout_fwd(torch.ones_like(V), None, 0.0, key, p_row=p, rows_per_sample=rps)
        return Y, DV, fac

    Y, DV, fac = twice(run, ("Y", "dV", "factor"))
    f = fac.float().view(B, rps * C)
    assert torch.equal(f, f[:, :1].expand_as(f)), "the factor varies inside a sample"
    assert set(f[:, 0].unique().tolist()) <= {0.0, 1.25}
    keep = f[:, 0] != 0
    assert 0.6 * B < int(keep.sum()) < B, int(keep.sum())
    k = keep.repeat_interleave(rps)[:, None]
    same(Y, torch.where(k, (X.double() + 1.25 * V.double()).float().to(torch.bfloat16), X), "Y")
    same(DV, torch.where(k, (1.25 * DY.double()).float().to(torch.bfloat16), torch.zeros_like(DY)), "dV")


# ------------------------------------------------------------------------------------------- every mode
MODES = ["b0", "b1", "b2", "b3", "b4", "b5", "b6", "b7"]
RECIPE_RES = {"b0": 224, "b1": 240, "b2": 260, "b3": 300, "b4": 380, "b5": 456, "b6": 528, "b7": 600}


def _model(pkg, mode, seed):
    shapes = E.efficientnet_shapes(mode)
    m = pkg.EfficientNet(pkg.default_effnet_opts(mode))
    m.load_state_dict(O.seeded_fill_(dict(shapes), seed), strict=True)
    return m.cuda(), shapes


@pytest.mark.parametrize("mode", MODES)
def test_efficientnet_modes_train(pkg, mode):
    """train-mode forward / backward at 64^2, batch 2, against the fp32 restatement; bounds relative to the same restatement under bf16
    autocast (the last stage's BatchNorms see 8 values per channel)"""
    seed, B, res = 40 + MODES.index(mode), 2, 64
    m, shapes = _model(pkg, mode, seed)
    m.train()
    x = O.seeded_input((B, 3, res, res), seed + 100).cuda()
    gy = O.seeded_input((B, 1000), seed + 200).cuda()
    y = m(x)
    y.backward(gy.to(y.dtype))
    P = O.clone_params(O.seeded_fill_(dict(shapes), seed), device="cuda")
    yr = E.efficientnet_forward(P, x, mode=mode)
    yr.backward(gy)
    Pa = O.clone_params(O.seeded_fill_(dict(shapes), seed), device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        ya = E.efficientnet_forward(Pa, x, mode=mode)
    ya.float().backward(gy)
    torch.cuda.synchronize()
    e, ea = rel_l2(y, yr), rel_l2(ya, yr)
    assert e <= max(2e-2, 3.0 * ea), f"logits rel-L2 {e:.4g} (autocast {ea:.3g})"
    bad = []
    for k, prm in m.named_parameters():
        gr, ga = P[k].grad, Pa[k].grad
        if float(gr.norm()) < 1e-3 * float(gy.norm()):  # analytically ~0 (a BatchNorm bias feeding another normalisation)
            continue
        e, ea = rel_l2(prm.grad, gr), rel_l2(ga, gr)
        if e > max(5e-2, 3.0 * ea):
            bad.append((k, round(e, 4), round(ea, 4)))
    assert not bad, f"{len(bad)} parameter gradients outside 3x the autocast error: {bad[:8]}"


@pytest.mark.parametrize("mode", MODES)
def test_efficientnet_modes_eval_recipe_res(pkg, mode):
    """eval-mode logits at each recipe's training resolution (b0 224 .. b7 600), batch 2"""
    seed, B, res = 60 + MODES.index(mode), 2, RECIPE_RES[mode]
    m, shapes = _model(pkg, mode, seed)
    m.eval()
    x = O.seeded_input((B, 3, res, res), seed + 100).cuda()
    P = O.clone_params(O.seeded_fill_(dict(shapes), seed), device="cuda")
    with torch.no_grad():
        y = m(x)
        yr = E.efficientnet_forward(P, x, mode=mode, training=False)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ya = E.efficientnet_forward(P, x, mode=mode, training=False)
    e, ea = rel_l2(y, yr), rel_l2(ya, yr)
    assert e <= max(2e-2, 3.0 * ea), f"logits rel-L2 {e:.4g} (autocast {ea:.3g})"


# ------------------------------------------------------------------------------------------- step level: b0 SGD-Nesterov, bitwise
def _effnet_state(ts, model):
    st = {f"param {k}": p.detach().clone() for k, p in model.named_parameters()}
    st.update({f"buffer {k}": b.detach().clone() for k, b in model.named_buffers()})
    o = ts.opt
    st.update({"momentum": o.momentum_buffer.clone(), "ema": o.ema.clone(), "scale": o.scale.clone(), "step": o.step_count.clone()})
    return st


def _effnet_train(pkg, ops, xs, ys, *, pdl=True, side=True, graph=False):
    lr = 0.1
    prev_pdl, prev_side = ops.set_pdl_enabled(pdl), ops._SIDE["on"]
    ops._SIDE["on"] = side
    try:
        model = pkg.EfficientNet(pkg.default_effnet_opts("b0", **{"model.classification.efficientnet.stochastic_depth_prob": 0.2}))
        model.load_state_dict(O.seeded_fill_(E.efficientnet_shapes("b0"), 77), strict=True)
        model = model.cuda().train()
        ts = pkg.TrainStep(model, optimizer="sgd", lr=0.0 if graph else lr, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None,
                           label_smoothing=0.1, ema_momentum=0.0005)
        ops.rng_seed(7)
        rng = ops._RNG[ops._rng_device("cuda")]
        rng0 = rng.clone()
        if graph:
            sd0 = {k: v.clone() for k, v in model.state_dict().items()}
            ts.capture(xs[0], ys[0])
            # undo what the warm-up steps changed: BatchNorm statistics and counters, momentum, EMA, step count, loss scale, mask counter
            model.load_state_dict(sd0)
            ts.opt.momentum_buffer.zero_()
            ts.opt.ema.copy_(ts.opt.flat_p)
            ts.opt.step_count.zero_()
            ts.opt.scale.copy_(torch.tensor([65536.0, 0.0]))
            rng.copy_(rng0)
            ts.set_lr(lr)
        losses = [ts.step(x, y).detach().clone() for x, y in zip(xs, ys)]
        torch.cuda.synchronize()
        return losses, _effnet_state(ts, model)
    finally:
        ops.set_pdl_enabled(prev_pdl)
        ops._SIDE["on"] = prev_side


def test_train_step_sgd_bitwise_across_launch_paths(pkg, ops):
    """EfficientNet-b0, batch 32 at 128^2, stochastic depth 0.2, three SGD-Nesterov steps with EMA and label smoothing: eager twice, without
    programmatic dependent launch, with the weight gradients on the main stream and replayed from a CUDA graph all end in the same bits"""
    B, res = 32, 128
    xs = [O.seeded_input((B, 3, res, res), 300 + i).cuda() for i in range(3)]
    ys = [(torch.arange(B, device="cuda") * (11 + i)) % 1000 for i in range(3)]
    ref_l, ref_s = _effnet_train(pkg, ops, xs, ys)
    assert all(bool(torch.isfinite(v)) for v in ref_l)
    for what, kw in (("eager rerun", {}), ("PDL off", {"pdl": False}), ("side stream off", {"side": False}), ("graph replay", {"graph": True})):
        losses, st = _effnet_train(pkg, ops, xs, ys, **kw)
        for i, (a, b) in enumerate(zip(losses, ref_l)):
            same(a, b, f"{what}: loss of step {i}")
        assert st.keys() == ref_s.keys()
        bad = [k for k in ref_s if not torch.equal(st[k], ref_s[k])]
        assert not bad, f"{what}: {len(bad)} of {len(ref_s)} state tensors differ from the first eager run, e.g. {bad[:6]}"
    assert float(ref_s["step"]) == 3.0

"""Bitwise run-to-run reproducibility (-m gpu), at the grid sizes training uses.

A MobileViTv2 training step is meant to be bitwise reproducible: every reduction that several CTAs add into sums fp32 partials in fp64, and
weight gradients meet in an fp64 scratch (DetScratch in csrc/common.cuh).  One last-bit difference flips a bf16 rounding somewhere in the
network, and AdamW turns the noise gradients of analytically-zero parameters into +-lr steps, so "close" is not enough: two runs must be
torch.equal.

Step level: the same three TrainStep steps eager twice, with programmatic dependent launch off, with the weight-gradient side stream off and
replayed from a captured graph; the dilated (output_stride 8 / 16) backbone's end points and gradients.

Kernel level: each persistent or grid-capped kernel is called at a size where its CTAs loop over at least three units of work, unevenly
(the state carried from one pass to the next -- double-buffered TMA sets, mbarrier parities, accumulators kept across images or rows -- is
what the small shapes of test_kernels_gpu.py never reach).  The size comes from the SM count through a restatement of the host-side grid
formula.  Every such call runs twice on identical inputs (torch.equal on every output and accumulator) and is compared with an fp64 torch
restatement on the same bf16-rounded inputs.  The entry points DESIGN.md lists as still using fp32 atomics are in NONDETERMINISTIC: they get
the fp64 comparison past their grid caps, but no torch.equal."""
import math
import os
import sys

import pytest
import torch
import torch.nn.functional as F

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from test_kernels_gpu import BF, bf, close, close_stat, dsilu, load_ref, rnd  # noqa: E402
from test_kernels_edges_gpu import same  # noqa: E402

pytestmark = pytest.mark.gpu

F64 = torch.float64

# entry points that still add fp32 partials with fp32 atomics (DESIGN.md section 6): their results depend on arrival order in the last bits
NONDETERMINISTIC = {
    "cvb_ln_bwd": "dgamma / dbeta of the ViT / CLIP LayerNorm backward are fp32 atomics of per-CTA partials",
    "cvb_mha_bwd": "the register-resident (S <= 256) attention backward sums dQ with shared-memory float atomics",
    "cvb_embedding_bwd": "token-embedding gradients add repeated token ids with fp32 atomics",
    "cvb_ce_bwd": "the CLIP logit-scale gradient dlogit_scale is an fp32 atomic sum over rows (dlogits themselves have one writer)",
}


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


def twice(fn, names):
    """fn() twice on identical inputs: every returned tensor bitwise equal (NaN == NaN); returns the first run's outputs"""
    a = [t.clone() for t in fn()]
    torch.cuda.synchronize()
    b = fn()
    torch.cuda.synchronize()
    assert len(a) == len(b) == len(names)
    for x, y, n in zip(a, b, names):
        same(y, x, f"{n}: second run")
    return a


def passes(units, ctas):
    """the work/grid split the tests need: >= 3 units per CTA, and a remainder so that CTAs get unequal counts"""
    assert units >= 3 * ctas and units % ctas != 0, (units, ctas)


def zeros64(*shape):
    return torch.zeros(*shape, device="cuda", dtype=F64)


# ------------------------------------------------------------------------------------------- step level: MobileViTv2 TrainStep
def _state(ts, model):
    st = {f"param {k}": p.detach().clone() for k, p in model.named_parameters()}
    st.update({f"buffer {k}": b.detach().clone() for k, b in model.named_buffers()})
    o = ts.opt
    st.update({"exp_avg": o.exp_avg.clone(), "exp_avg_sq": o.exp_avg_sq.clone(), "scale": o.scale.clone(), "step": o.step_count.clone()})
    return st


def _train(pkg, ops, xs, ys, *, pdl=True, side=True, graph=False, width=1.0):
    from test_engine_gpu import _small_model
    lr = 2e-3
    prev_pdl, prev_side = ops.set_pdl_enabled(pdl), ops._SIDE["on"]
    ops._SIDE["on"] = side
    try:
        model = _small_model(pkg, width=width)
        # weight decay is set from the start: at lr = 0 the capture's warm-up steps leave the weights bit-for-bit unchanged (p * (1 - 0 * wd) - 0 * u)
        ts = pkg.TrainStep(model, lr=0.0 if graph else lr, weight_decay=0.05, max_norm=10.0, label_smoothing=0.1)
        if graph:
            sd0 = {k: v.clone() for k, v in model.state_dict().items()}
            ts.capture(xs[0], ys[0])
            # undo what the warm-up steps changed: BatchNorm running statistics and counters, moments, step count, loss scale
            model.load_state_dict(sd0)
            ts.opt.exp_avg.zero_()
            ts.opt.exp_avg_sq.zero_()
            ts.opt.step_count.zero_()
            ts.opt.scale.copy_(torch.tensor([65536.0, 0.0]))
            ts.set_lr(lr)
        losses = [ts.step(x, y).detach().clone() for x, y in zip(xs, ys)]
        torch.cuda.synchronize()
        return losses, _state(ts, model)
    finally:
        ops.set_pdl_enabled(prev_pdl)
        ops._SIDE["on"] = prev_side


def test_train_step_bitwise_across_launch_paths(pkg, ops):
    """MobileViTv2-1.0, batch 32 at 256x256, three AdamW steps with clipping and label smoothing: eager twice, eager without programmatic
    dependent launch, eager with the weight gradients on the main stream, and a replayed CUDA graph all end in the same bits.  A PDL-only
    difference would mean a kernel reads its producer's output before griddepcontrol.wait; a graph-only one, state surviving the warm-up."""
    from oracle import cvnets_oracle as O
    B, res = 32, 256
    xs = [O.seeded_input((B, 3, res, res), 200 + i).cuda() for i in range(3)]
    ys = [(torch.arange(B, device="cuda") * (7 + i)) % 1000 for i in range(3)]
    ref_l, ref_s = _train(pkg, ops, xs, ys)
    for what, kw in (("eager rerun", {}), ("PDL off", {"pdl": False}), ("side stream off", {"side": False}), ("graph replay", {"graph": True})):
        losses, st = _train(pkg, ops, xs, ys, **kw)
        for i, (a, b) in enumerate(zip(losses, ref_l)):
            same(a, b, f"{what}: loss of step {i}")
        assert st.keys() == ref_s.keys()
        bad = [k for k in ref_s if not torch.equal(st[k], ref_s[k])]
        assert not bad, f"{what}: {len(bad)} of {len(ref_s)} state tensors differ from the first eager run, e.g. {bad[:6]}"
    assert float(ref_s["step"]) == 3.0


# ------------------------------------------------------------------------------------------- step level: dilated backbone
@pytest.mark.parametrize("output_stride", [8, 16])
def test_dilated_backbone_bitwise(pkg, output_stride):
    """output_stride 8 / 16 (segmentation backbones): layer_4 / layer_5 run the dilated depthwise kernels.  extract_end_points_all forward and a
    seeded backward, twice: end points and every parameter gradient bitwise equal."""
    from oracle import cvnets_oracle as O
    B, res, width = 16, 256, 1.0
    x = O.seeded_input((B, 3, res, res), 31).cuda()

    def run():
        model = pkg.MobileViTv2(pkg.default_opts(width_multiplier=width), output_stride=output_stride)
        model.load_state_dict(O.seeded_fill_(O.mobilevit_v2_shapes(width), 11), strict=True)
        model = model.cuda().train()
        ends = model.extract_end_points_all(x)
        g = torch.Generator(device="cuda").manual_seed(32)
        loss = sum((ends[k].float() * torch.randn(ends[k].shape, device="cuda", generator=g)).sum() for k in sorted(ends))
        loss.backward()
        torch.cuda.synchronize()
        # the classifier is not on the end-point path: no gradient
        return {k: v.detach().clone() for k, v in ends.items()}, {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}

    e1, g1 = run()
    e2, g2 = run()
    assert g1.keys() == g2.keys() and len(g1) > 100
    for k in e1:
        same(e2[k], e1[k], f"end point {k}")
    diff = {k: int((g1[k] != g2[k]).sum()) for k in g1}
    bad = {k: n for k, n in diff.items() if n}
    assert not bad, f"{len(bad)} parameter gradients differ between two runs ({sum(bad.values())} elements): {bad}"


# ------------------------------------------------------------------------------------------- depthwise 3x3, fp64 restatement
def dw_ref_fwd(xa, w9, s, d):
    """xa: activated input [B, H, W, C] fp64, w9: [9, C] (tap u * 3 + v) -> [B, Ho, Wo, C]; pad = d, stride s, dilation d"""
    B, H, W, C = xa.shape
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    xp = F.pad(xa, (0, 0, d, d, d, d))
    y = torch.zeros(B, Ho, Wo, C, device=xa.device, dtype=F64)
    for u in range(3):
        for v in range(3):
            y += w9[3 * u + v] * xp[:, u * d:u * d + s * (Ho - 1) + 1:s, v * d:v * d + s * (Wo - 1) + 1:s]
    return y


def dw_ref_bwd(xa, dy, w9, s, d):
    """adjoint of dw_ref_fwd: (d xa [B, H, W, C], dW [9, C])"""
    B, H, W, C = xa.shape
    Ho, Wo = dy.shape[1:3]
    xp = F.pad(xa, (0, 0, d, d, d, d))
    dxp = torch.zeros_like(xp)
    dw = torch.empty(9, C, device=xa.device, dtype=F64)
    for u in range(3):
        for v in range(3):
            sl = (slice(None), slice(u * d, u * d + s * (Ho - 1) + 1, s), slice(v * d, v * d + s * (Wo - 1) + 1, s))
            dw[3 * u + v] = (xp[sl] * dy).sum((0, 1, 2))
            dxp[sl] += w9[3 * u + v] * dy
    return dxp[:, d:d + H, d:d + W], dw


def dw_fwd_grid(H, W, C, s, sms):
    """CTAs per image column of cvb_dw_fwd's grid (dwconv.cu:542-552): tiles x 64-channel blocks per image, gz = ceil(8 #SM / per_img)"""
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    TW = 16 if (s == 1 and Wo > 8) else 8
    TH = (16 if Ho > 8 else 8) if s == 1 else 8
    per_img = math.ceil(Ho / TH) * math.ceil(Wo / TW) * math.ceil(C / 64)
    return math.ceil(8 * sms / per_img)


def dw_bwd_grid(H, W, C, s, sms):
    """the same for cvb_dw_bwd (dwconv.cu:603-617): 8- or 16-wide tiles, gz = ceil(4 #SM / per_img)"""
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    TW = 16 if Wo > 8 else 8
    TH = (16 if Ho > 8 else 8) if s == 1 else 8
    per_img = math.ceil(Ho / TH) * math.ceil(Wo / TW) * math.ceil(C / 64)
    return math.ceil(4 * sms / per_img)


def dw_batch(gz):
    """B = 3 gz + 1: every CTA's batch loop runs three images, the first CTA of each tile a fourth"""
    B = 3 * gz + 1
    passes(B, gz)
    return B


# the MobileViTv2-1.0 depthwise layers at 256x256 input (H = W, C, stride), and one C that is not a multiple of 64
DW_LAYERS = [(128, 64, 1), (128, 128, 2), (64, 256, 1), (64, 256, 2), (32, 512, 2), (32, 256, 1), (16, 384, 1), (16, 768, 2), (8, 512, 1),
             (32, 144, 1)]


def _dw_params(C, seed):
    w = bf(rnd(C, 9, scale=0.3, seed=seed)).float()
    Wt = w.t().contiguous()
    xp = (1 + 0.2 * rnd(C, seed=seed + 1), 0.3 * rnd(C, seed=seed + 2))
    gp = (1 + 0.2 * rnd(C, seed=seed + 3), 0.3 * rnd(C, seed=seed + 4), 0.1 * rnd(C, seed=seed + 5))
    return Wt, xp, gp


def _check_dw_fwd(ops, B, H, C, s, d, x_mode, seed):
    W = H
    X = bf(rnd(B * H * W, C, seed=seed))
    Wt, xp, _ = _dw_params(C, seed + 10)

    def run():
        col = zeros64(2, C)
        Y = ops.dw_fwd(X, B, H, W, C, s, Wt, x_mode=x_mode, x_p=xp, col_stats=col, dilation=d)
        return Y, col

    Y, col = twice(run, ("Y", "col_stats"))
    xa = load_ref(x_mode, X, xp + (None,)).double().view(B, H, W, C)
    ref = dw_ref_fwd(xa, Wt.double(), s, d).view(-1, C)
    close(Y, ref, what="dw fwd")
    o = Y.double()
    close_stat(col[0], o.sum(0), "col_sum")
    close_stat(col[1], (o * o).sum(0), "col_sq")


def _check_dw_bwd(ops, B, H, C, s, d, g_mode, x_mode, seed):
    W = H
    Ho, Wo = (H - 1) // s + 1, (W - 1) // s + 1
    X = bf(rnd(B * H * W, C, seed=seed))
    DZ, Y2 = bf(rnd(B * Ho * Wo, C, seed=seed + 1)), bf(rnd(B * Ho * Wo, C, seed=seed + 2))
    Wt, xp, gp = _dw_params(C, seed + 10)

    def run():
        col = zeros64(2, C)
        DX, dWt = ops.dw_bwd(DZ, X, B, H, W, C, s, Wt, g_mode=g_mode, Y2=Y2 if g_mode == 5 else None, g_p=gp, x_mode=x_mode, x_p=xp,
                             col_stats=col if x_mode != 0 else None, dilation=d)
        return DX, dWt, col

    DX, dWt, col = twice(run, ("dX", "dW", "col_stats"))
    dy = load_ref(g_mode, DZ, gp, Y2).double().view(B, Ho, Wo, C)
    xa = load_ref(x_mode, X, xp + (None,)).double().view(B, H, W, C)
    da, dw = dw_ref_bwd(xa, dy, Wt.double(), s, d)
    da = da.reshape(-1, C)
    if x_mode == 2:
        da = da * dsilu(xp[0].double() * X.double() + xp[1].double())
    close(DX, da, what="dX")
    close(dWt, dw, rtol=3e-3, atol=3e-3 * float(dw.abs().max()) + 1e-5, what="dW")
    if x_mode != 0 and d == 1:
        # the walk kernels take interior tiles' statistics from fp32 values and edge tiles' from the stored ones (test_dw_bwd)
        close_stat(col[0], da.sum(0), "sum dz", rtol=6e-3)
        close_stat(col[1], (da * X.double()).sum(0), "sum dz*x", rtol=6e-3)
    elif x_mode != 0:
        # the dilated kernel sums the stored values
        close_stat(col[0], DX.double().sum(0), "sum dz")
        close_stat(col[1], (DX.double() * X.double()).sum(0), "sum dz*x")


@pytest.mark.parametrize("H,C,s", DW_LAYERS)
@pytest.mark.parametrize("x_mode", [0, 1, 2])
def test_dw_fwd_batch_loop(ops, sms, H, C, s, x_mode):
    B = dw_batch(dw_fwd_grid(H, H, C, s, sms))
    _check_dw_fwd(ops, B, H, C, s, 1, x_mode, seed=700 + H + C)


@pytest.mark.parametrize("H,C,s", DW_LAYERS)
@pytest.mark.parametrize("g_mode,x_mode", [(0, 0), (5, 1), (0, 2), (5, 2)])
def test_dw_bwd_batch_loop(ops, sms, H, C, s, g_mode, x_mode):
    B = dw_batch(dw_bwd_grid(H, H, C, s, sms))
    _check_dw_bwd(ops, B, H, C, s, 1, g_mode, x_mode, seed=800 + H + C)


def dwd_grid(C, sms):
    """cvb_dw_{fwd,bwd}_dilated (dwconv_dilated.cu:227-238): blocks of (cx channel chunks x py pixels), at most 4 #SM blocks -> (cap, py)"""
    cc, cx = C // 8, 1
    while cx < cc and cx < 32:
        cx *= 2
    return 4 * sms, 256 // cx


def dwd_batch(H, C, sms):
    """images of H x H such that every block's pixel loop runs >= 3 passes and the pixels do not split evenly over the blocks"""
    cap, py = dwd_grid(C, sms)
    B = math.ceil((3 * cap * py + 1) / (H * H))
    while (B * H * H) % (cap * py) == 0:
        B += 1
    passes(math.ceil(B * H * H / py), cap)
    return B


# C = 384 is 48 chunks of 8 channels over a 32-wide block: the kernel's channel-chunk loop runs twice
@pytest.mark.parametrize("C,dil", [(256, 2), (384, 2), (256, 4), (384, 4)])
@pytest.mark.parametrize("x_mode", [0, 1, 2])
def test_dw_fwd_dilated_grid_loop(ops, sms, C, dil, x_mode):
    H = 32
    _check_dw_fwd(ops, dwd_batch(H, C, sms), H, C, 1, dil, x_mode, seed=900 + C + dil)


@pytest.mark.parametrize("C,dil", [(256, 2), (384, 2), (256, 4), (384, 4)])
@pytest.mark.parametrize("g_mode,x_mode", [(0, 0), (5, 1), (0, 2), (5, 2)])
def test_dw_bwd_dilated_grid_loop(ops, sms, C, dil, g_mode, x_mode):
    """dW used to be added with fp32 atomics straight into the caller's buffer: it now goes through the fp64 scratch like the dense path"""
    H = 32
    _check_dw_bwd(ops, dwd_batch(H, C, sms), H, C, 1, dil, g_mode, x_mode, seed=950 + C + dil)


# ------------------------------------------------------------------------------------------- pointwise GEMMs at the benched shapes
BENCHED_GEMM = [(2097152, 128, 64, 0), (2097152, 128, 64, 1), (2097152, 64, 32, 2), (524288, 256, 128, 0), (131072, 264, 128, 4),
                (32768, 392, 192, 4), (8192, 520, 256, 4), (131072, 128, 264, 0), (32768, 192, 392, 0), (8192, 256, 520, 0)]


@pytest.mark.parametrize("M,N,K,a_mode", BENCHED_GEMM)
def test_pw_gemm_benched_bitwise(ops, M, N, K, a_mode):
    """the test_pw_gemm_benched_shapes shapes (batch 128) with column and per-sample statistics"""
    B = 128
    rps = M // B
    A = bf(rnd(M, K, seed=1001))
    W = bf(rnd(N, K, scale=K ** -0.5, seed=1002))
    bias = rnd(N, seed=1003)
    p = (1 + 0.2 * rnd(K, seed=1004), 0.3 * rnd(K, seed=1005), None)
    row = (0.2 * rnd(B, seed=1006), 1 + 0.3 * rnd(B, seed=1007).abs())

    def run():
        col, samp = zeros64(2, N), zeros64(2, B)
        out = ops.pw_gemm(A, W, N, a_mode=a_mode, a_p=p, row_stats=row if a_mode == 4 else None, rows_per_sample=rps, bias=bias,
                          col_stats=col, samp_stats=samp)
        return out, col, samp

    out, col, samp = twice(run, ("out", "col_stats", "samp_stats"))
    ref = load_ref(a_mode, A, p, None, row, rps).double() @ W.double().t() + bias.double()
    close(out, ref, what="out")
    o = out.double()
    close_stat(col[0], o.sum(0), "col_sum")
    close_stat(col[1], (o * o).sum(0), "col_sq")
    close_stat(samp[0], o.view(B, -1).sum(1), "samp_sum")
    close_stat(samp[1], (o * o).view(B, -1).sum(1), "samp_sq")


@pytest.mark.parametrize("tc", [True, False], ids=["wgmma", "mma_sync"])
@pytest.mark.parametrize("e_name", ["silu_bwd", "lin_bwd"])
def test_pw_gemm_bwd_epilogues_bitwise(ops, tc, e_name):
    """the input-gradient epilogues with the producer's BatchNorm-backward statistics, on both kernel families: SILU_BWD (BatchNorm + SiLU
    producer) and LIN_BWD (BatchNorm without an activation: the lazily-normalised module boundary, otherwise reached only through the models)"""
    M, N, K = 131072, 256, 128
    A = bf(rnd(M, K, seed=1011))
    W = bf(rnd(N, K, scale=K ** -0.5, seed=1012))
    Y = bf(rnd(M, N, seed=1013))
    sc, sh = 1 + 0.2 * rnd(N, seed=1014), 0.3 * rnd(N, seed=1015)
    e_mode = ops.E_SILU_BWD if e_name == "silu_bwd" else ops.E_LIN_BWD

    def run():
        prev = ops.set_tc_enabled(tc)
        try:
            col = zeros64(2, N)
            out = ops.pw_gemm(A, W, N, e_mode=e_mode, Y=Y, e_p=(sc, sh), col_stats=col)
            return out, col
        finally:
            ops.set_tc_enabled(prev)

    out, col = twice(run, ("out", "col_stats"))
    acc = A.double() @ W.double().t()
    ref = acc * dsilu(sc.double() * Y.double() + sh.double()) if e_name == "silu_bwd" else acc
    close(out, ref, what=e_name)
    o = out.double()
    close_stat(col[0], o.sum(0), "sum dz")
    close_stat(col[1], (o * Y.double()).sum(0), "sum dz*y")


@pytest.mark.parametrize("ws", [True, False])
def test_pw_gemm_gn_bwd_bitwise(ops, ws):
    """GroupNorm-backward epilogue at batch 128 on the 32x32 map: with the per-sample workspace (wgmma kernel, sum form) and without.  The
    workspace finalize used to add its fp64 per-sample sums into dgamma / dbeta with atomics: about half of the channels differed run to run."""
    B, rps, N, K = 128, 1024, 256, 256
    M = B * rps
    A, W = bf(rnd(M, K, seed=1021)), bf(rnd(N, K, scale=K ** -0.5, seed=1022))
    X = bf(rnd(M, N, seed=1023))
    gamma = 1 + 0.2 * rnd(N, seed=1024)
    row = (0.2 * rnd(B, seed=1025), 1 + 0.3 * rnd(B, seed=1026).abs())

    def run():
        col, samp = zeros64(2, N), zeros64(2, B)
        gn_ws = zeros64(2, B, N) if ws else None
        out = ops.pw_gemm(A, W, N, e_mode=ops.E_GN_BWD, Y=X, e_p=(gamma, None), row_stats=row, rows_per_sample=rps, col_stats=col,
                          samp_stats=samp, gn_ws=gn_ws)
        return out, col, samp

    out, col, samp = twice(run, ("g", "col_stats", "samp_stats"))
    v = A.double() @ W.double().t()
    xh = (X.double() - row[0].double().repeat_interleave(rps)[:, None]) * row[1].double().repeat_interleave(rps)[:, None]
    close(out, v * gamma.double(), what="g")
    close_stat(col[0], v.sum(0), "dbeta", rtol=5e-3)
    close_stat(col[1], (v * xh).sum(0), "dgamma", rtol=5e-3)
    o = out.double()
    close_stat(samp[0], o.view(B, -1).sum(1), "sum g", rtol=5e-3)
    close_stat(samp[1], (o * xh).view(B, -1).sum(1), "sum g*xh", rtol=5e-3)


@pytest.mark.parametrize("M,N,K,g_mode,a_mode", [(2097152, 128, 64, 5, 0), (2097152, 64, 64, 5, 2), (524288, 256, 128, 5, 0), (131072, 264, 128, 0, 4),
                                                  (32768, 392, 192, 0, 4), (8192, 520, 256, 0, 4)])
@pytest.mark.parametrize("tc", [True, False], ids=["wgmma", "mma_sync"])
def test_pw_wgrad_benched_bitwise(ops, M, N, K, g_mode, a_mode, tc):
    """the test_pw_wgrad_benched_shapes shapes on both weight-gradient kernels: split-M partials meet in the fp64 scratch"""
    B = 128
    rps = M // B
    G, G2, A = bf(rnd(M, N, seed=1031)), bf(rnd(M, N, seed=1032)), bf(rnd(M, K, seed=1033))
    gp = (1 + 0.2 * rnd(N, seed=1034), 0.3 * rnd(N, seed=1035), 0.1 * rnd(N, seed=1036))
    ap = (1 + 0.2 * rnd(K, seed=1037), 0.3 * rnd(K, seed=1038))
    row = (0.2 * rnd(B, seed=1039), 1 + 0.3 * rnd(B, seed=1040).abs())

    def run():
        prev = ops.set_tc_enabled(tc)
        try:
            db = torch.zeros(N, device="cuda")
            dW = ops.pw_wgrad(G, A, N, K, g_mode=g_mode, G2=G2 if g_mode == 5 else None, g_p=gp, a_mode=a_mode, a_p=ap,
                              row_stats=row if a_mode == 4 else None, rows_per_sample=rps, dbias=db)
            return dW, db
        finally:
            ops.set_tc_enabled(prev)

    dW, db = twice(run, ("dW", "dbias"))
    Gr = load_ref(g_mode, G, gp, G2).double()
    Ar = load_ref(a_mode, A, ap + (None,), None, row, rps).double()
    ref = Gr.t() @ Ar
    close(dW, ref, rtol=2e-3, atol=2e-3 * float(ref.abs().max()) + 1e-5, what="dW", rel_l2=1e-3)
    close(db, Gr.sum(0), rtol=2e-3, atol=2e-3 * float(Gr.sum(0).abs().max()) + 1e-4, what="dbias", rel_l2=1e-3)


# ------------------------------------------------------------------------------------------- BatchNorm / GroupNorm reductions, 128 x 128^2 rows
def test_bn_bwd_reduce_bitwise(ops):
    M, C = 128 * 128 * 128, 64
    D, Y = bf(rnd(M, C, seed=1101)), bf(rnd(M, C, seed=1102) * 1.5 + 0.3)
    bn = torch.stack([rnd(C, seed=1103), rnd(C, seed=1104).abs() + 0.5, 1 + 0.2 * rnd(C, seed=1105), 0.3 * rnd(C, seed=1106)])

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


def test_gn_stats_and_bwd_apply_bitwise(ops):
    B, rps, C = 128, 128 * 128, 64
    M = B * rps
    X, G, DR = bf(rnd(M, C, seed=1111) + 0.5), bf(rnd(M, C, seed=1112)), bf(rnd(M, C, seed=1113))
    xs = X.double().view(B, -1)
    mean, var = xs.mean(1), xs.var(1, unbiased=False)
    gn = torch.stack([mean, (var + 1e-5).rsqrt()]).float()
    xh = (xs - gn[0].double()[:, None]) * gn[1].double()[:, None]
    g = G.double().view(B, -1)
    ss = torch.stack([g.sum(1), (g * xh).sum(1)])

    def run():
        st, cs = zeros64(2, B), zeros64(C)
        ops.gn_stats(X, B, rps, st)
        DX = ops.gn_bwd_apply(G, X, gn, ss, rps * C, B, rps, DRES=DR, col_sum=cs)
        return st, DX, cs

    st, DX, cs = twice(run, ("gn stats", "dX", "col_sum"))
    close_stat(st[0], xs.sum(1), "gn sum")
    close_stat(st[1], (xs * xs).sum(1), "gn sq")
    n = rps * C
    ref = (gn[1].double()[:, None] * (g - ss[0][:, None] / n - xh * ss[1][:, None] / n)).view(M, C) + DR.double()
    close(DX, ref, what="gn dx")
    close_stat(cs, ref.sum(0), "col sum of dx", rtol=5e-3)


def test_gn_bwd_standalone_bitwise(ops):
    B, rps, C = 128, 128 * 128, 64
    M = B * rps
    X = bf(rnd(M, C, seed=1121) * 1.3 + 0.4)
    gamma = 1 + 0.2 * rnd(C, seed=1122)
    xs = X.double().view(B, -1)
    gn = torch.stack([xs.mean(1), (xs.var(1, unbiased=False) + 1e-5).rsqrt()]).float()
    xh = ((xs - gn[0].double()[:, None]) * gn[1].double()[:, None]).view(B, rps, C)
    V = bf(1 + 0.5 * xh.float().view(M, C) + 0.3 * rnd(M, C, seed=1123))
    DR = bf(rnd(M, C, seed=1124))

    def run():
        dg, db, ws = zeros64(C), zeros64(C), zeros64(2, B)
        DX = ops.gn_bwd(V, X, gn, gamma, rps * C, B, rps, dg, db, ws, DRES=DR)
        return DX, dg, db, ws

    DX, dg, db, ws = twice(run, ("dX", "dgamma", "dbeta", "per-sample sums"))
    v = V.double().view(B, rps, C)
    g = v * gamma.double()
    n = rps * C
    sg, sgx = g.view(B, -1).sum(1), (g * xh).view(B, -1).sum(1)
    close_stat(ws[0], sg, "sum g", rtol=1e-4)
    close_stat(ws[1], sgx, "sum g*xhat", rtol=1e-4)
    close_stat(db, v.sum((0, 1)), "dbeta", rtol=1e-4)
    close_stat(dg, (v * xh).sum((0, 1)), "dgamma", rtol=1e-4)
    ref = (gn[1].double()[:, None, None] * (g - sg[:, None, None] / n - xh * sgx[:, None, None] / n)).view(M, C) + DR.double()
    close(DX, ref, what="gn dx")


# ------------------------------------------------------------------------------------------- linear attention at batch 128
def _unfold(t):
    B, C = t.shape[:2]
    return F.unfold(t, kernel_size=2, stride=2).reshape(B, C, 4, -1)


# MobileViTv2-1.0: layer_3 (d = 128) at 32^2, layer_4 (192) at 16^2, layer_5 (256) at 8^2
@pytest.mark.parametrize("H,d", [(32, 128), (16, 192), (8, 256)])
def test_linattn_bitwise(ops, H, d):
    B, W = 128, H
    ldq = 2 * d + 8
    M = B * H * W
    QKV = bf(rnd(M, ldq, seed=1201))
    DO = bf(rnd(M, d, seed=1202))

    def run():
        O, S, CTX = ops.linattn_fwd(QKV, B, H, W, d)
        db = torch.zeros(ldq, device="cuda")
        DQKV = ops.linattn_bwd(QKV, DO, S, CTX, B, H, W, d, dbias=db)
        return O, S, CTX, DQKV, db

    O, S, CTX, DQKV, db = twice(run, ("O", "S", "CTX", "dQKV", "dbias"))
    q4 = QKV.double().view(B, H, W, ldq).permute(0, 3, 1, 2)

    def fold(p):
        Bc, C, P, N = p.shape
        return F.fold(p.reshape(Bc, C * P, N), output_size=(H, W), kernel_size=2, stride=2).permute(0, 2, 3, 1).reshape(-1, C)

    k = _unfold(q4[:, :d]).requires_grad_(True)
    v = _unfold(q4[:, d:2 * d]).requires_grad_(True)
    q = _unfold(q4[:, 2 * d:2 * d + 1]).requires_grad_(True)
    s = torch.softmax(q, dim=-1)
    ctx = (k * s).sum(-1, keepdim=True)
    out = torch.relu(v) * ctx
    close(O, fold(out.detach()), what="O")
    close(CTX, ctx.detach().squeeze(-1).permute(0, 2, 1), rtol=2e-3, atol=1e-4, what="ctx")
    close(S, s.detach().squeeze(1), rtol=2e-3, atol=1e-5, what="scores")
    out.backward(_unfold(DO.double().view(B, H, W, d).permute(0, 3, 1, 2)))
    dk, dv, dq = fold(k.grad), fold(v.grad), fold(q.grad)[:, 0]
    close(DQKV[:, :d], dk, what="dK")
    close(DQKV[:, d:2 * d], dv, what="dV")
    close(DQKV[:, 2 * d], dq, rtol=3e-2, atol=2e-2 * float(dq.abs().max()) + 1e-6, what="dq")
    assert float(DQKV[:, 2 * d + 1:].float().abs().max()) == 0.0
    sums = DQKV[:, :2 * d + 1].double().sum(0)
    close(db[:2 * d + 1], sums, rtol=2e-3, atol=2e-3 * float(sums.abs().max()) + 1e-5, what="dbias")


# d = 336 / 448 (MobileViTv2-1.75): the 8-channel groups of one row span three warps, so linattn_bwd sums three warp pieces of ds
@pytest.mark.parametrize("Mp,d", [(256, 128), (64, 192), (16, 256), (64, 336), (16, 448)])
def test_linattn_cross_bitwise(ops, Mp, d):
    B, P, N = 128, 4, Mp
    ld = 2 * d + 8
    QKP = bf(rnd(B * P * Mp, ld, seed=1211))
    QKVX = bf(rnd(B * P * N, ld, seed=1212))
    DO = bf(rnd(B * P * N, d, seed=1213))

    def run():
        O, S, CTX = ops.linattn_cross_fwd(QKP, QKVX, B, P, Mp, N, d)
        db = torch.zeros(ld, device="cuda")
        DQKP, DQKVX = ops.linattn_cross_bwd(QKP, QKVX, DO, S, CTX, B, P, Mp, N, d, dbias=db)
        return O, S, CTX, DQKP, DQKVX, db

    O, S, CTX, DQKP, DQKVX, db = twice(run, ("O", "S", "CTX", "dQK_prev", "dV_x", "dbias"))
    qk = QKP.double().view(B, P, Mp, ld)
    key = qk[..., :d].clone().requires_grad_(True)
    query = qk[..., 2 * d].clone().requires_grad_(True)
    value = QKVX.double().view(B, P, N, ld)[..., d:2 * d].clone().requires_grad_(True)
    s = torch.softmax(query, dim=-1)
    ctx = (key * s[..., None]).sum(2)
    out = torch.relu(value) * ctx[:, :, None, :]
    close(O, out.detach().reshape(-1, d), what="O")
    close(S, s.detach(), rtol=2e-3, atol=1e-5, what="scores")
    close(CTX, ctx.detach(), rtol=2e-3, atol=1e-4, what="ctx")
    out.backward(DO.double().view(B, P, N, d))
    close(DQKP[:, :d], key.grad.reshape(-1, d), what="dkey")
    dq = query.grad.reshape(-1)
    close(DQKP[:, 2 * d], dq, rtol=3e-2, atol=2e-2 * float(dq.abs().max()) + 1e-6, what="dquery")
    close(DQKVX[:, d:2 * d], value.grad.reshape(-1, d), what="dvalue")
    sums = torch.cat([DQKP[:, :d].double().sum(0), DQKVX[:, d:2 * d].double().sum(0), DQKP[:, 2 * d:2 * d + 1].double().sum(0)])
    close(db[:2 * d + 1], sums, rtol=2e-3, atol=2e-3 * float(sums.abs().max()) + 1e-5, what="dbias")


# ------------------------------------------------------------------------------------------- pooling and loss at batch 128 / 1024
@pytest.mark.parametrize("B", [128, 1024])
def test_pool_and_ce_bitwise(ops, B):
    HW, C, NC = 64, 512, 1000
    X = bf(rnd(B * HW, C, seed=1301))
    logits = bf(rnd(B, NC, scale=3.0, seed=1302))
    target = torch.randint(0, NC, (B,), device="cuda", generator=torch.Generator(device="cuda").manual_seed(1303))
    target[::7] = -1
    gout, gscale = torch.tensor([0.7], device="cuda"), torch.tensor([1024.0], device="cuda")

    def run():
        p = ops.global_pool_fwd(X, B, HW)
        loss, lse, nv = ops.ce_fwd(logits, NC, target, -1, 0.1)
        d = ops.ce_bwd(logits, NC, target, -1, 0.1, lse, nv, gout, gscale, NC)
        return p, loss, lse, nv, d

    p, loss, lse, nv, d = twice(run, ("pool", "loss", "lse", "n_valid", "dlogits"))
    close(p, X.double().view(B, HW, C).mean(1), what="pool fwd")
    lg = logits.double().requires_grad_(True)
    ref = F.cross_entropy(lg, target, ignore_index=-1, label_smoothing=0.1)
    ref.backward()
    assert float(nv) == float((target != -1).sum())
    assert float((lse.double() - torch.logsumexp(lg.detach(), 1)).abs().max()) <= 1e-5 * float(lse.abs().max()) + 1e-5
    assert abs(float(loss) - float(ref)) <= 3e-5 * abs(float(ref)) + 1e-6, (float(loss), float(ref))
    close(d, lg.grad * 0.7 * 1024.0, what="dlogits")


# ------------------------------------------------------------------------------------------- optimizer tail past its grid caps
class _Tail:
    """flat fp32 buffers for cvb_grad_norm + cvb_adamw_step, sized for this test (partials from cvb_grad_norm_blocks of this n)"""

    def __init__(self, lib, n, wd, *, lr=2e-3, max_norm=10.0, growth_interval=2000, ema=0.1, seed=0):
        self.lib, self.n = lib, n
        g = torch.Generator(device="cuda").manual_seed(seed)
        self.p = torch.randn(n, device="cuda", generator=g)
        self.m = torch.zeros(n, device="cuda")
        self.v = torch.zeros(n, device="cuda")
        self.wd = wd
        self.ema = self.p.clone() if ema is not None else None
        self.ema_m = 0.0 if ema is None else float(ema)
        self.stats = torch.zeros(4, device="cuda")
        self.partials = torch.zeros(2 * lib.cvb_grad_norm_blocks(n), device="cuda")
        self.scale = torch.tensor([65536.0, 0.0], device="cuda")
        self.step_count = torch.zeros(1, device="cuda")
        self.hp = torch.tensor([lr], device="cuda")
        self.max_norm, self.gi = float(max_norm), int(growth_interval)

    def step(self, grads, grad_div):
        st = torch.cuda.current_stream().cuda_stream
        self.lib.cvb_grad_norm(grads.data_ptr(), self.n, self.scale.data_ptr(), float(grad_div), self.stats.data_ptr(),
                               self.partials.data_ptr(), st)
        self.lib.cvb_adamw_step(self.p.data_ptr(), grads.data_ptr(), self.m.data_ptr(), self.v.data_ptr(), self.wd.data_ptr(), self.n,
                                self.hp.data_ptr(), 0.9, 0.999, 1e-8, self.max_norm, self.stats.data_ptr(), self.scale.data_ptr(),
                                self.step_count.data_ptr(), 2.0, 0.5, self.gi, self.ema.data_ptr() if self.ema is not None else None,
                                self.ema_m, self.partials.data_ptr(), st)

    def state(self):
        out = [self.p, self.m, self.v, self.stats, self.scale, self.step_count, self.partials]
        return [t.clone() for t in out] + ([self.ema.clone()] if self.ema is not None else [])


class _RefTail:
    """GradScaler.unscale_ -> clip_grad_norm_ -> torch.optim.AdamW(foreach=False) -> GradScaler.update, and the EMA, on fp64 copies"""

    def __init__(self, p0, wd, *, lr=2e-3, max_norm=10.0, growth_interval=2000, ema=0.1):
        # the kernel receives its hyper-parameters as fp32: 1 - float32(0.999) is 1.3e-5 away from 0.001, which exp_avg_sq shows
        f32 = lambda x: float(torch.tensor(x, dtype=torch.float32))  # noqa: E731
        self.groups = [(wd == w).nonzero().squeeze(1) for w in torch.unique(wd).tolist()]
        self.wds = torch.unique(wd).tolist()
        self.params = [torch.nn.Parameter(p0.double()[idx].clone()) for idx in self.groups]
        self.opt = torch.optim.AdamW([{"params": [p], "weight_decay": w} for p, w in zip(self.params, self.wds)], lr=f32(lr),
                                     betas=(f32(0.9), f32(0.999)), eps=f32(1e-8), foreach=False)
        self.n = p0.numel()
        self.scale, self.tracker, self.gi = 65536.0, 0, growth_interval
        self.max_norm = max_norm
        self.ema = p0.double().clone() if ema is not None else None
        self.ema_m = f32(ema) if ema is not None else None

    def flat(self):
        out = torch.empty(self.n, device="cuda", dtype=F64)
        for idx, p in zip(self.groups, self.params):
            out[idx] = p.detach()
        return out

    def moments(self):
        m, v = torch.empty(self.n, device="cuda", dtype=F64), torch.empty(self.n, device="cuda", dtype=F64)
        for idx, p in zip(self.groups, self.params):
            st = self.opt.state.get(p, {})
            m[idx] = st["exp_avg"] if st else 0.0
            v[idx] = st["exp_avg_sq"] if st else 0.0
        return m, v

    def step(self, grads, grad_div):
        g = grads.double() / (self.scale * grad_div)
        finite = bool(torch.isfinite(g).all())
        self.sumsq = float(g.square().sum())
        if finite:
            if self.max_norm > 0:
                norm = float(g.norm())
                g = g * min(1.0, self.max_norm / (norm + 1e-6))
            for idx, p in zip(self.groups, self.params):
                p.grad = g[idx].clone()
            self.opt.step()
            self.tracker += 1
            if self.tracker >= self.gi:
                self.scale, self.tracker = self.scale * 2.0, 0
        else:
            self.scale, self.tracker = self.scale * 0.5, 0
        if self.ema is not None:
            self.ema = self.ema * (1 - self.ema_m) + self.ema_m * self.flat()
        return g


def _tail_n(sms):
    """cvb_grad_norm: float4 items over min(ceil(n/4 / 256), 4 #SM) blocks of 256 (optim.cu:127-133); three full passes, a fourth for the first
    seven blocks, and n % 4 = 3 scalars for block 0 thread 0.  cvb_adamw_step's 8 #SM blocks (optim.cu:147-149) then loop ~6 times."""
    cap = 4 * sms
    n = 3 * (cap * 256 * 4) + 7 * 256 * 4 + 3
    passes(n // 4, cap * 256)
    passes(n, 8 * sms * 256)
    return n


def _check_tail(tail, ref, what):
    p, m, v, stats, scale, step = tail.state()[:6]
    rp = ref.flat()
    rm, rv = ref.moments()
    err = float((p.double() - rp).abs().max())
    assert err <= 2e-6 + 1e-5 * float(rp.abs().max()), f"{what}: params max abs diff {err}"
    for got, want, name in ((m, rm, "exp_avg"), (v, rv, "exp_avg_sq")):
        e = float((got.double() - want).abs().max())
        assert e <= 1e-5 * float(want.abs().max()) + 1e-12, f"{what}: {name} max abs diff {e}"
    assert float(scale[0]) == ref.scale and int(scale[1]) == ref.tracker, (what, scale.tolist(), ref.scale, ref.tracker)
    if ref.ema is not None:
        e = float((tail.ema.double() - ref.ema).abs().max())
        assert e <= 2e-6 + 1e-5 * float(ref.ema.abs().max()), f"{what}: EMA max abs diff {e}"


def test_grad_norm_adamw_step_past_grid_caps(ops, sms):
    """per-element weight decay, grad_div 4 (DDP's world size), EMA on, clipping active; then a step with inf in the last block's range and one
    with NaN in the n % 4 tail, each skipped with the scale backed off and the EMA still updated; then a normal step.  Twice, bitwise."""
    from ml_cvnets_b200 import _lib as L
    lib = L.load()
    n = _tail_n(sms)
    idx = torch.arange(n, device="cuda")
    wd = torch.where(idx % 3 == 0, torch.tensor(0.05, device="cuda"), torch.where(idx % 3 == 1, torch.tensor(0.1, device="cuda"),
                                                                                     torch.tensor(0.0, device="cuda")))
    blocks = lib.cvb_grad_norm_blocks(n)
    assert blocks == 4 * sms
    gen = torch.Generator(device="cuda").manual_seed(1401)
    grads = []
    for it in range(4):
        # loss scale 65536 x grad_div 4; unscaled norms ~1270 (step 0) and ~250 (step 3 at scale 16384): the clip is active in both
        g = torch.randn(n, device="cuda", generator=gen) * 65536.0 * 4 * (0.05 if it != 0 else 1.0)
        if it == 1:
            g[4 * ((3 * blocks - 1) * 256 + 100) + 1] = float("inf")  # float4 item of the last block's third pass
        if it == 2:
            g[n - 1] = float("nan")  # the n % 4 scalars after the last float4
        grads.append(g)

    def run():
        tail = _Tail(lib, n, wd, seed=1402)
        for g in grads:
            tail.step(g, 4.0)
        return tail.state()

    names = ("params", "exp_avg", "exp_avg_sq", "stats", "scale", "step", "partials", "ema")
    twice(run, names)
    tail = _Tail(lib, n, wd, seed=1402)
    ref = _RefTail(tail.p, wd)
    for it, g in enumerate(grads):
        tail.step(g, 4.0)
        ref.step(g, 4.0)
        torch.cuda.synchronize()
        _check_tail(tail, ref, f"step {it}")
        if it in (1, 2):
            assert float(tail.stats[1]) == 1.0, f"step {it}: non-finite count {float(tail.stats[1])}, want 1"
        else:
            assert float(tail.stats[1]) == 0.0
            assert abs(float(tail.stats[0]) - ref.sumsq) <= 1e-5 * ref.sumsq, (it, float(tail.stats[0]), ref.sumsq)
    assert float(tail.step_count) == 2.0 and float(tail.scale[0]) == 65536.0 * 0.25


def test_adamw_step_scale_growth_without_clipping(ops, sms):
    """growth_interval 2: the loss scale doubles after every second finite step; max_norm 0 turns clipping off (large gradients untouched)"""
    from ml_cvnets_b200 import _lib as L
    lib = L.load()
    n = _tail_n(sms)
    wd = torch.full((n,), 0.05, device="cuda")
    gen = torch.Generator(device="cuda").manual_seed(1411)
    tail = _Tail(lib, n, wd, max_norm=0.0, growth_interval=2, ema=None, seed=1412)
    ref = _RefTail(tail.p, wd, max_norm=0.0, growth_interval=2, ema=None)
    scales = []
    for it in range(5):
        g = torch.randn(n, device="cuda", generator=gen) * float(tail.scale[0]) * 3.0  # unscaled norm ~ 3800: clipping would change the step
        tail.step(g, 1.0)
        ref.step(g, 1.0)
        torch.cuda.synchronize()
        _check_tail(tail, ref, f"step {it}")
        assert abs(float(tail.stats[0]) - ref.sumsq) <= 1e-5 * ref.sumsq, (float(tail.stats[0]), ref.sumsq)
        scales.append(float(tail.scale[0]))
    assert scales == [65536.0, 131072.0, 131072.0, 262144.0, 262144.0]


# ------------------------------------------------------------------------------------------- declared exceptions: fp64 comparison only
def ln_bwd_ctas(M, sms):
    """cvb_ln_bwd (norm.cu:931-933): CTAs of 8 rows, at most 4 #SM"""
    return min(math.ceil(M / 8), 4 * sms)


@pytest.mark.parametrize("C", [768, 1024])
def test_ln_bwd_past_grid_cap(ops, sms, C):
    """ViT-B/16 at batch 256 (M = 256 x 197 tokens): each capped CTA loops over many 8-row groups.  dgamma / dbeta are fp32 atomics
    (NONDETERMINISTIC), so this is the fp64 comparison only."""
    M = 50432
    passes(math.ceil(M / 8), ln_bwd_ctas(M, sms))
    X = bf(rnd(M, C, seed=1501) * 1.5 + 0.3)
    V = bf(rnd(M, C, seed=1502))
    R = bf(rnd(M, C, seed=1503))
    gamma = 1 + 0.2 * rnd(C, seed=1504)
    ln = ops.ln_stats(X, 1e-5)
    col, cs = zeros64(2, C), zeros64(C)
    DX = ops.ln_bwd(V, X, ln, gamma, col, DRES=R, col_sum=cs)
    xh = (X.double() - ln[0].double()[:, None]) * ln[1].double()[:, None]
    v = V.double()
    g = v * gamma.double()
    ref = ln[1].double()[:, None] * (g - g.mean(1, keepdim=True) - xh * (g * xh).mean(1, keepdim=True)) + R.double()
    close(DX, ref, what="ln_bwd dx")
    close_stat(col[0], v.sum(0), "dbeta", rtol=5e-3)
    close_stat(col[1], (v * xh).sum(0), "dgamma", rtol=5e-3)
    close_stat(cs, DX.double().sum(0), "col_sum", rtol=5e-3)


# ------------------------------------------------------------------------------------------- weight preparation past its grid caps
def test_prep_weights_past_grid_cap(ops):
    """cvb_prep_weights caps its grid at 64 x 1024 items per descriptor (norm.cu:1046-1048): the ViT-B qkv projection (2304 x 768, row-major and
    transposed) and a 768 x 3 x 16 x 16 patch stem (kinds 4 / 5: (ci, tap) -> (tap, ci) order and its transpose), bitwise"""
    qkv = torch.nn.Parameter(rnd(2304, 768, seed=1601))
    stem = torch.nn.Parameter(rnd(768, 3, 16, 16, seed=1602))
    P = ops.PreparedWeights()
    i0 = P.add(qkv, P.KIND_ROWMAJOR)
    i1 = P.add(qkv, P.KIND_TRANSPOSED)
    i4 = P.add(stem, P.KIND_PATCH, rot=256)
    i5 = P.add(stem, P.KIND_PATCH_T, rot=256)
    P.prepare()
    assert P._max_elems > 3 * 64 * 1024
    patch = stem.detach().permute(0, 2, 3, 1).reshape(768, 768)  # columns (u, v, ci) = the im2col patch order
    same(P.get(i0), qkv.detach().to(BF), "kind 0")
    same(P.get(i1), qkv.detach().t().to(BF), "kind 1")
    same(P.get(i4), patch.to(BF), "kind 4")
    same(P.get(i5), patch.t().to(BF), "kind 5")


def test_unprep_grad_past_grid_cap(ops, sms):
    """cvb_unprep_grad's grid is capped at 16 #SM blocks of 256 (grid_for, norm.cu:822-828): kinds 0 (row rotation, strided source), 2 (tap-major
    depthwise dW) and 4 ((tap, ci) -> (ci, tap)) at >= 3 passes, bitwise"""
    cap = 16 * sms * 256
    cols = 768
    rows = 3 * cap // cols + 5
    passes(rows * cols, cap)
    src = rnd(rows, cols + 8, seed=1611)
    same(ops.unprep_grad(src, rows, cols, cols + 8, 0, rot=1), src[:, :cols].roll(1, 0), "kind 0")
    C = 3 * cap // 9 + 17
    passes(C * 9, cap)
    tap = rnd(9, C, seed=1612)
    same(ops.unprep_grad(tap, C, 9, C, 2), tap.t(), "kind 2")
    taps, cin = 256, 3
    src4 = rnd(rows, taps * cin + 8, seed=1613)
    want = src4[:, :taps * cin].reshape(rows, taps, cin).permute(0, 2, 1).reshape(rows, taps * cin)
    same(ops.unprep_grad(src4, rows, taps * cin, taps * cin + 8, 4, rot=taps), want, "kind 4")

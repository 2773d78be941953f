"""EfficientNet on the GPU (-m gpu): the depthwise 5x5 walk kernels against fp32 torch on identical bf16-rounded operands, ConvLayer2d 5x5 /
EfficientNetBlock / EfficientNet-b0 against the fixtures of the real reference (tests/golden/efficientnet_fp32.pt), stochastic depth under
identical masks, a captured SGD training step run twice, and cvb_sgd_step against torch.optim.SGD.

Tolerances as in test_modules_gpu.py: activations are bf16 at every layer boundary, so outputs <= 2e-2, input gradients <= 4e-2 and parameter
gradients <= 5e-2 rel-L2 (cosine >= 1 - tol) against fp32, or within 3x the error of the fp32 restatement itself run under bf16 autocast."""
import copy
import os

import pytest
import torch
import torch.nn.functional as F

import efficientnet_ref as E
from golden_sample import at_sample, ref_norm
from oracle import cvnets_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as m
    return m


@pytest.fixture(scope="module")
def fx(golden_dir):
    return torch.load(os.path.join(golden_dir, "efficientnet_fp32.pt"), weights_only=False)


def rel_l2(a, b):
    a, b = a.detach().float().cpu(), b.detach().float().cpu()
    return float((a - b).norm() / (b.norm() + 1e-12))


def cosine(a, b):
    a, b = a.detach().float().cpu().flatten(), b.detach().float().cpu().flatten()
    return float(torch.dot(a, b) / (a.norm() * b.norm() + 1e-20))


def bf(t):
    return t.bfloat16().float()


# ------------------------------------------------------------------------------------------------------------------ kernels
def _act(z, x_mode, ops):
    return F.silu(z) if x_mode == ops.A_AFF_SILU else z


# (B, C, H, W): EfficientNet-b0's 5x5 widths 144 / 240 / 672 / 1152 (C % 64 != 0 included) at 28^2 / 14^2 / 7^2 and non-square maps
SHAPES = [(2, 144, 28, 28), (1, 240, 28, 28), (2, 240, 14, 14), (1, 672, 14, 14), (2, 672, 7, 7), (1, 1152, 7, 7), (2, 144, 14, 10), (1, 240, 10, 18)]


@pytest.mark.parametrize("stride", [1, 2])
@pytest.mark.parametrize("B,C,H,W", SHAPES)
def test_dw5_kernels_vs_torch(pkg, B, C, H, W, stride):
    """Forward with every load mode and the fp64 BN statistics of the output; backward with RAW / BNB gradients and every load mode: input
    gradient (through the producer's activation), producer-BN statistics and dW; dW bitwise identical across two runs."""
    from ml_cvnets_b200 import ops
    K = 5
    g = torch.Generator(device="cuda").manual_seed(B * 10007 + C * 31 + H * 7 + W + stride)
    x = torch.randn(B * H * W, C, device="cuda", generator=g).bfloat16()
    w = bf(torch.randn(C, 1, K, K, device="cuda", generator=g) / K)
    Wt = w.reshape(C, K * K).t().contiguous()
    p0 = 1.0 + 0.2 * torch.randn(C, device="cuda", generator=g)
    p1 = 0.1 * torch.randn(C, device="cuda", generator=g)
    x4 = x.float().view(B, H, W, C).permute(0, 3, 1, 2)
    Ho, Wo = (H - 1) // stride + 1, (W - 1) // stride + 1
    to_2d = lambda t: t.permute(0, 2, 3, 1).reshape(-1, t.shape[1])  # noqa: E731
    for x_mode in (ops.A_RAW, ops.A_AFF, ops.A_AFF_SILU):
        xp = (p0, p1) if x_mode != ops.A_RAW else (None, None)
        z = x4 * p0.view(1, -1, 1, 1) + p1.view(1, -1, 1, 1) if x_mode != ops.A_RAW else x4
        a = _act(z, x_mode, ops)
        st = torch.zeros(2, C, device="cuda", dtype=torch.float64)
        y = ops.dw_fwd(x, B, H, W, C, stride, Wt, x_mode=x_mode, x_p=xp, col_stats=st, ksize=K)
        y_ref = F.conv2d(bf(a), w, stride=stride, padding=2, groups=C)  # the kernel rounds the transformed operand to bf16 in shared memory
        assert rel_l2(y, to_2d(y_ref)) <= 1e-2, (x_mode, rel_l2(y, to_2d(y_ref)))
        yf = y.float()
        assert rel_l2(st[0], yf.sum(0).double()) <= 1e-2 and rel_l2(st[1], (yf * yf).sum(0).double()) <= 1e-2, x_mode
        if stride == 2 and (H % 2 or W % 2):
            continue
        for g_mode in ((ops.A_RAW, ops.A_BNB) if x_mode == ops.A_RAW else (ops.A_BNB,)):
            dz = torch.randn(B * Ho * Wo, C, device="cuda", generator=g).bfloat16()
            if g_mode == ops.A_BNB:
                c = [0.5 + torch.rand(C, device="cuda", generator=g), 0.1 * torch.randn(C, device="cuda", generator=g),
                     0.1 * torch.randn(C, device="cuda", generator=g)]
                dy = bf(c[0] * dz.float() + c[1] * y.float() + c[2])
                kw = dict(g_mode=ops.A_BNB, Y2=y, g_p=c)
            else:
                dy, kw = dz.float(), {}
            dy4 = dy.view(B, Ho, Wo, C).permute(0, 3, 1, 2)
            sd = torch.zeros(2, C, device="cuda", dtype=torch.float64)
            dx, dWt = ops.dw_bwd(dz, x, B, H, W, C, stride, Wt, x_mode=x_mode, x_p=xp, col_stats=sd if x_mode != ops.A_RAW else None, ksize=K, **kw)
            da = torch.nn.grad.conv2d_input(x4.shape, w, dy4, stride=stride, padding=2, groups=C)
            if x_mode == ops.A_AFF_SILU:
                s = torch.sigmoid(z)
                da = da * (s + z * s * (1 - s))
            dw_ref = torch.nn.grad.conv2d_weight(a, w.shape, dy4, stride=stride, padding=2, groups=C)
            assert rel_l2(dx, to_2d(da)) <= 1e-2, (x_mode, g_mode, rel_l2(dx, to_2d(da)))
            assert rel_l2(dWt.t().reshape(C, 1, K, K), dw_ref) <= 5e-3, (x_mode, g_mode, rel_l2(dWt.t().reshape(C, 1, K, K), dw_ref))
            if x_mode != ops.A_RAW:
                dxf = dx.float()
                assert rel_l2(sd[0], dxf.sum(0).double()) <= 2e-2 and rel_l2(sd[1], (dxf * x.float()).sum(0).double()) <= 2e-2
            _, dWt2 = ops.dw_bwd(dz, x, B, H, W, C, stride, Wt, x_mode=x_mode, x_p=xp, ksize=K, **kw)
            assert torch.equal(dWt, dWt2), "5x5 dW is not bitwise reproducible"


def test_dw5_rejects_dilation_and_odd_stride2_backward(pkg):
    from ml_cvnets_b200 import _lib as L, ops
    x = torch.zeros(2 * 7 * 7 * 64, device="cuda", dtype=torch.bfloat16).view(-1, 64)
    Wt = torch.zeros(25, 64, device="cuda")
    with pytest.raises(L.CvbError):
        ops.dw_fwd(x, 2, 7, 7, 64, 1, Wt, dilation=2, ksize=5)
    with pytest.raises(L.CvbError):
        ops.dw_bwd(torch.zeros(2 * 4 * 4, 64, device="cuda", dtype=torch.bfloat16), x, 2, 7, 7, 64, 2, Wt, ksize=5)


# ------------------------------------------------------------------------------------------------------------------ modules
def _load(module, shapes, seed, prefix="m."):
    P = O.seeded_fill_(shapes, seed)
    module.load_state_dict({k[len(prefix):]: v for k, v in P.items()}, strict=True)
    return module.cuda().train()


def _autocast_errors(fn, shapes, f, prefix="m."):
    P = O.clone_params(O.seeded_fill_(dict(shapes), f["seed"]), device="cuda")
    x = O.seeded_input(f["x_shape"], f["x_seed"]).cuda().requires_grad_(True)
    with torch.autocast("cuda", dtype=torch.bfloat16):
        y = fn(P, x)
    y.backward(O.seeded_input(tuple(y.shape), f["gy_seed"]).cuda().to(y.dtype))
    out = {"y": rel_l2(*at_sample(y.float(), f["y"])), **{k: rel_l2(*at_sample(P[prefix + k].grad, g)) for k, g in f["grads"].items()}}
    out.update({"buffer " + k: rel_l2(*at_sample(P[prefix + k], b)) for k, b in f["buffers"].items() if not k.endswith("num_batches_tracked")})
    return out


def _check(module, f, auto, out_tol=2e-2, gx_tol=4e-2, gp_tol=5e-2, check_gx=True):
    x = O.seeded_input(f["x_shape"], f["x_seed"]).cuda().requires_grad_(check_gx)
    y = module(x)
    gy = O.seeded_input(tuple(y.shape), f["gy_seed"]).cuda()
    y.backward(gy.to(y.dtype))
    torch.cuda.synchronize()
    e = rel_l2(*at_sample(y.float(), f["y"]))
    assert e <= max(out_tol, 3.0 * auto["y"]), f"output rel-L2 {e:.4g} (autocast {auto['y']:.3g})"
    if check_gx:
        e = rel_l2(*at_sample(x.grad, f["gx"]))
        assert e <= gx_tol, f"input-grad rel-L2 {e:.4g}"
    named = dict(module.named_parameters())
    for k, g in f["grads"].items():
        ours, ref = at_sample(named[k].grad, g)
        e, c = rel_l2(ours, ref), cosine(ours, ref)
        tol = max(gp_tol, 3.0 * auto[k])
        small = ref_norm(g) < 1e-3 * float(gy.norm())
        assert (e <= tol and c >= 1 - tol) or small, f"{k}: rel-L2 {e:.4g} (tol {tol:.3g}) cos {c:.5f}"
    bufs = dict(module.named_buffers())
    for k, b in f["buffers"].items():
        if k.endswith("num_batches_tracked"):
            assert int(bufs[k]) == int(b if torch.is_tensor(b) else b["val"][0]), k
        else:
            e = rel_l2(*at_sample(bufs[k], b))
            assert e <= max(1e-2, 3.0 * auto["buffer " + k]), f"{k}: {e:.4g} (autocast {auto['buffer ' + k]:.3g})"


@pytest.mark.parametrize("name", ["dw5_s1", "dw5_s2"])
def test_conv_layer_dw5(pkg, fx, name):
    f = fx[name]
    c = f["cfg"]
    shapes = {}
    O._conv_bn(shapes, "m", c["c"], c["c"], 5, groups=c["c"])
    fn = lambda P, x: O.conv_layer_2d(P, "m", x, stride=c["stride"], groups=c["c"], use_act=False)  # noqa: E731
    auto = _autocast_errors(fn, shapes, f)
    m = _load(pkg.ConvLayer2d(pkg.default_effnet_opts(), c["c"], c["c"], 5, stride=c["stride"], groups=c["c"], use_norm=True, use_act=False), shapes, f["seed"])
    _check(m, f, auto)


def _block(pkg, c, p=0.0):
    return pkg.EfficientNetBlock(p, opts=pkg.default_effnet_opts(), in_channels=c["cin"], out_channels=c["cout"], kernel_size=c["kernel_size"],
                                 stride=c["stride"], expand_ratio=c["expand_ratio"], dilation=1, use_se=True, squeeze_factor=c["expand_ratio"] * 4,
                                 act_fn_name="swish", se_scale_fn_name="sigmoid")


@pytest.mark.parametrize("name", ["eb_e1_k3", "eb_e6_k5_s2", "eb_e6_k5_res"])
def test_efficientnet_block(pkg, fx, name):
    f = fx[name]
    c = f["cfg"]
    shapes = {}
    E.efficientnet_block_shapes(shapes, "m", c["cin"], c["cout"], c["expand_ratio"], c["kernel_size"])
    auto = _autocast_errors(lambda P, x: E.efficientnet_block(P, "m", x, stride=c["stride"]), shapes, f)
    m = _load(_block(pkg, c), shapes, f["seed"])
    assert repr(m) == f["repr"]
    _check(m, f, auto)


def test_efficientnet_block_stochastic_depth_training(pkg, fx):
    """Stochastic depth p = 0.5 in training against the fp32 restatement under the SAME per-sample factors (regenerated from the module's
    key); the factors are constant per sample and keep about 1 - p of the samples.  Eval mode is the plain residual block."""
    from ml_cvnets_b200 import ops
    c = fx["eb_e6_k5_res"]["cfg"]
    p, B, H, W = 0.5, 16, 12, 10
    shapes = {}
    E.efficientnet_block_shapes(shapes, "m", c["cin"], c["cout"], c["expand_ratio"], c["kernel_size"])
    m = _load(_block(pkg, c, p), shapes, 91)
    P = O.clone_params(O.seeded_fill_(dict(shapes), 91), device="cuda")
    g = torch.Generator(device="cuda").manual_seed(5)
    x = bf(torch.randn(B, c["cin"], H, W, device="cuda", generator=g))
    gy = bf(torch.randn(B, c["cout"], H, W, device="cuda", generator=g))
    ops.rng_seed(1234)
    xg = x.clone().requires_grad_(True)
    y = m(xg)
    y.backward(gy.to(y.dtype))
    ops.rng_seed(1234)
    key = ops.rng_next("cuda")  # the block's only draw: StochasticDepthAddFn's key
    ones = torch.ones(B * H * W, c["cout"], device="cuda", dtype=torch.bfloat16)
    fac = ops.dropout_fwd(ones, None, 0.0, key, p_row=p, rows_per_sample=H * W).float().view(B, H * W * c["cout"])
    assert torch.equal(fac, fac[:, :1].expand_as(fac)), "stochastic-depth factor varies inside a sample"
    keep = (fac[:, 0] != 0).float()
    assert 0 < float(keep.sum()) < B
    xo = x.clone().requires_grad_(True)
    yo = E.efficientnet_block(P, "m", xo, stride=1, drop_mask=keep / (1 - p))
    yo.backward(gy)
    assert rel_l2(y, yo) <= 2e-2, rel_l2(y, yo)
    assert rel_l2(xg.grad, xo.grad) <= 5e-2, rel_l2(xg.grad, xo.grad)
    for k, prm in m.named_parameters():
        e = rel_l2(prm.grad, P["m." + k].grad)
        assert e <= 6e-2, f"{k}: {e:.4g}"
    # keep rate of the kernel's per-sample draw over many samples
    big = ops.dropout_fwd(torch.ones(4096 * 4, 8, device="cuda", dtype=torch.bfloat16), None, 0.0, ops.rng_next("cuda"), p_row=0.3, rows_per_sample=4)
    per = big.float().view(4096, 32)
    assert torch.equal(per, per[:, :1].expand_as(per))
    assert abs(float((per[:, 0] != 0).float().mean()) - 0.7) < 0.04
    m.eval()
    P2 = O.clone_params(O.seeded_fill_(dict(shapes), 91), device="cuda")
    assert rel_l2(m(x), E.efficientnet_block(P2, "m", x, stride=1, training=False)) <= 2e-2


# ------------------------------------------------------------------------------------------------------------------ model
def test_efficientnet_b0(pkg, fx):
    f = fx["b0_64"]
    shapes = E.efficientnet_shapes("b0")
    auto = _autocast_errors(lambda P, x: E.efficientnet_forward(P, x, mode="b0"), shapes, f, prefix="")
    m = _load(pkg.EfficientNet(pkg.default_effnet_opts("b0")), shapes, f["seed"], prefix="")
    # at 64^2 and batch 2 the last stage's BatchNorms see 8 values per channel: their running statistics are held to 3x the autocast error
    _check(m, f, auto, check_gx=False)
    ends = m.extract_end_points_all(O.seeded_input(f["x_shape"], f["x_seed"]).cuda(), use_l5_exp=True)
    assert [tuple(v.shape[1:]) for v in ends.values()] == [(16, 32, 32), (24, 16, 16), (40, 8, 8), (112, 4, 4), (320, 2, 2), (1280, 2, 2)]


def _sgd_run(pkg, steps=3):
    from ml_cvnets_b200 import ops
    torch.manual_seed(0)
    model = pkg.EfficientNet(pkg.default_effnet_opts("b0", n_classes=16, **{"model.classification.efficientnet.stochastic_depth_prob": 0.2})).cuda()
    ts = pkg.TrainStep(model, optimizer="sgd", lr=0.1, momentum=0.9, nesterov=True, weight_decay=4e-5, max_norm=None, label_smoothing=0.1,
                       ema_momentum=0.0005)
    g = torch.Generator(device="cuda").manual_seed(1)
    x = torch.randn(8, 3, 64, 64, device="cuda", generator=g)
    y = torch.randint(0, 16, (8,), device="cuda", generator=g)
    ops.rng_seed(7)
    ts.capture(x, y)
    losses = [ts(x, y).clone() for _ in range(steps)]
    torch.cuda.synchronize()
    return torch.stack(losses), ts.opt.flat_p.clone(), ts.opt.ema.clone(), ts.opt.momentum_buffer.clone()


def test_train_step_sgd_captured_reproducible(pkg):
    """EfficientNet-b0 (stochastic depth 0.2) captured with SGD-Nesterov, EMA and label smoothing, three replays, run twice: the stochastic-depth
    masks, the squeeze-excitation scale gradients (fp64 scratch, cvb_se_scale_bwd) and the optimizer are deterministic, so the runs agree bit
    for bit."""
    a, b = _sgd_run(pkg), _sgd_run(pkg)
    assert torch.isfinite(a[0]).all()
    for name, u, v in zip(("losses", "params", "ema", "momentum"), a, b):
        assert torch.equal(u, v), (name, rel_l2(u, v))


# ------------------------------------------------------------------------------------------------------------------ SGD step
class _Tiny(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.conv = torch.nn.Conv2d(16, 32, 3, bias=False)
        self.bn = torch.nn.BatchNorm2d(32)
        self.fc = torch.nn.Linear(32, 10)


def test_sgd_step_vs_torch(pkg):
    """cvb_sgd_step (through FlatSGD) against torch.optim.SGD(momentum 0.9, nesterov, weight_decay 4e-5) with the two parameter groups of
    no_decay_bn_filter_bias, on the same unscaled gradients over several steps; the skip-on-inf path (no update, momentum kept, loss scale
    backed off, EMA still moving), the EMA itself and a state_dict round trip."""
    from ml_cvnets_b200 import FlatSGD
    torch.manual_seed(3)
    ours = _Tiny().cuda()
    ref = copy.deepcopy(ours)
    decay = [p for p in ref.parameters() if p.dim() > 1]
    no_decay = [p for p in ref.parameters() if p.dim() == 1]
    opt_ref = torch.optim.SGD([{"params": decay, "weight_decay": 4e-5}, {"params": no_decay, "weight_decay": 0.0}], lr=0.05, momentum=0.9,
                              nesterov=True)
    opt = FlatSGD(ours, lr=0.05, momentum=0.9, nesterov=True, weight_decay=4e-5, init_scale=1024.0, ema_momentum=0.1)
    ema = [p.detach().clone() for p in ours.parameters()]
    g = torch.Generator(device="cuda").manual_seed(4)
    for it in range(5):
        grads = [torch.randn(p.shape, device="cuda", generator=g) for p in ref.parameters()]
        for p, gr in zip(ref.parameters(), grads):
            p.grad = gr.clone()
        for p, gr in zip(ours.parameters(), grads):
            p.grad.copy_(gr * 1024.0)  # p.grad is a view of the flat buffer; the kernel unscales by the (power-of-two) loss scale
        opt_ref.step()
        opt.step()
        for e, p in zip(ema, ref.parameters()):
            e.mul_(0.9).add_(0.1 * p.detach())
        for (n, p), q in zip(ours.named_parameters(), ref.parameters()):
            assert rel_l2(p, q) <= 1e-6, (it, n, rel_l2(p, q))
        for e, p in zip(ema, opt.ema_parameters(ours).values()):
            assert rel_l2(p, e) <= 1e-6
    bufs = torch.cat([opt_ref.state[p]["momentum_buffer"].flatten() for p in ref.parameters()])
    ours_buf = torch.cat([opt.momentum_buffer[o:o + k] for o, k in (opt.ws.offsets[id(p)] for p in ours.parameters())])
    assert rel_l2(ours_buf, bufs) <= 1e-6
    # skip on inf: parameters and momentum unchanged, scale halved, step count unchanged, EMA still updated
    p_before, m_before, e_before = opt.flat_p.clone(), opt.momentum_buffer.clone(), opt.ema.clone()
    steps_before, scale_before = float(opt.step_count[0]), float(opt.scale[0])
    next(ours.parameters()).grad.view(-1)[0] = float("inf")
    opt.step()
    torch.cuda.synchronize()
    assert torch.equal(opt.flat_p, p_before) and torch.equal(opt.momentum_buffer, m_before)
    assert float(opt.scale[0]) == scale_before * 0.5 and float(opt.step_count[0]) == steps_before
    assert torch.allclose(opt.ema, e_before * 0.9 + 0.1 * p_before, rtol=1e-6, atol=1e-7)
    # state_dict round trip: a fresh optimizer loaded from the checkpoint takes the same next step
    sd = opt.state_dict()
    assert set(sd) == {"momentum_buffer", "step", "scale", "lr", "ema"}
    twin_model = copy.deepcopy(ours)
    twin = FlatSGD(twin_model, lr=0.05, momentum=0.9, nesterov=True, weight_decay=4e-5, ema_momentum=0.1)
    twin.flat_p.copy_(opt.flat_p)
    twin.load_state_dict(sd)
    gr = torch.randn(opt.n, device="cuda", generator=g)
    opt.flat_g.copy_(gr * float(opt.scale[0]))
    twin.flat_g.copy_(gr * float(twin.scale[0]))
    opt.step()
    twin.step()
    assert torch.equal(opt.flat_p, twin.flat_p) and torch.equal(opt.momentum_buffer, twin.momentum_buffer) and torch.equal(opt.ema, twin.ema)


def test_sgd_step_kernel_raises_on_nesterov_without_momentum(pkg):
    from ml_cvnets_b200 import _lib as L
    lib = L.load()
    # Nesterov without momentum is rejected (torch.optim.SGD raises for it too)
    with pytest.raises(L.CvbError, match="cvb_sgd_step failed"):
        lib.cvb_sgd_step(None, None, None, None, 0, None, 0.0, 1, 0.0, None, None, None, 2.0, 0.5, 2000, None, 0.0, None, None)

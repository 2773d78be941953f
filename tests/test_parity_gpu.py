"""Parity at the BENCHMARK configuration (-m gpu): MobileViTv2-1.0, 256x256, train mode, per-GPU batch 128 (and 32), seeded.

Truth = the fp32 oracle (pinned to the real reference by tests/golden) run on the same GPU with TF32 disabled.  Reported for every
quantity: our error AND the error of the same oracle under torch bf16 autocast (= what the reference's own AMP path gives on this GPU),
and the distance from north_star's "forward logits within 1e-3 rel".

Measured on an H100 80GB HBM3 at a 700 W power limit (seeded random weights, DESIGN.md section 6): END-TO-END, train mode, batch 128:
logits rel-L2 6.1e-2 (torch autocast: 7.1e-2), whole-gradient cosine 0.9864 (autocast 0.9833); eval mode: 3.1e-2 (autocast 2.7e-2).  The 1e-3 of north_star is an
fp32-class tolerance that no bf16-activation implementation of this 60-layer network reaches -- the reference's own AMP path included:
the END-TO-END numbers are dominated by the amplification of bf16 rounding (2^-9 per stored activation) through BatchNorm / GroupNorm
re-normalisations of a randomly initialised net.  So the tests assert three things with FIXED bounds:

  (1) STAGE-WISE parity at the benchmark shapes: every module (stem, each InvertedResidual, each MobileViTBlockv2, the classifier head),
      fed the fp32 oracle's input of that stage, reproduces the oracle's output of that stage within rel-L2 <= 1.5e-2 (train mode, batch 128)
      -- the bound that pins the kernels themselves, free of cross-layer amplification;
  (2) END-TO-END: eval logits <= 4e-2, train logits <= 8e-2, loss within 2e-3 relative, whole-gradient cosine >= 0.98;
  (3) END-TO-END vs the same-precision comparator: never worse than 1.15x the torch-autocast error on the same quantity (+ 2e-3).
"""
import json
import os

import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def pkg():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    import ml_cvnets_b200 as m
    return m


def rel_l2(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    return float((a - b).norm() / (b.norm() + 1e-30))


def cosine(a, b):
    a, b = a.detach().double().flatten(), b.detach().double().flatten()
    return float(torch.dot(a, b) / (a.norm() * b.norm() + 1e-30))


def _setup(pkg, seed, width=1.0):
    model = pkg.MobileViTv2(pkg.default_opts(width_multiplier=width))
    P = O.seeded_fill_(O.mobilevit_v2_shapes(width), seed)
    model.load_state_dict(P, strict=True)
    return model.cuda(), P


def _record(name, d):
    out = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "gpurun_out")
    try:
        os.makedirs(out, exist_ok=True)
        with open(os.path.join(out, f"parity_{name}.json"), "w") as f:
            json.dump(d, f, indent=1)
    except OSError:
        pass


def train_parity_record(pkg, B, width=1.0):
    """One train-mode forward / backward of ours, the fp32 oracle and the oracle under torch bf16 autocast on the same seeded batch:
    the record of their distances, and the per-parameter tuples of the parameters carrying a non-negligible share of the gradient."""
    model, P = _setup(pkg, 2024, width)
    model.train()
    x = O.seeded_input((B, 3, 256, 256), 31).cuda()
    y = (torch.arange(B, device="cuda") * 37) % 1000
    logits = model(x)
    loss = pkg.cross_entropy(logits, y, label_smoothing=0.1)
    loss.backward()
    ours = {k: p.grad.detach().float().clone() for k, p in model.named_parameters()}
    ours_logits, ours_loss = logits.detach().float().clone(), float(loss)
    del logits, loss
    model.zero_grad(set_to_none=True)
    torch.cuda.empty_cache()
    # truth: fp32 oracle on this GPU
    P32 = O.clone_params(P, device="cuda")
    l32 = O.mobilevit_v2_forward(P32, x, width_multiplier=width, training=True)
    loss32 = F.cross_entropy(l32, y, label_smoothing=0.1)
    loss32.backward()
    g32 = {k: v.grad.detach().clone() for k, v in P32.items() if v.requires_grad and v.grad is not None}
    l32 = l32.detach().clone()
    loss32 = float(loss32)
    del P32
    torch.cuda.empty_cache()
    # same-precision comparator: the oracle under torch bf16 autocast
    Pa = O.clone_params(P, device="cuda")
    with torch.autocast("cuda", dtype=torch.bfloat16):
        la = O.mobilevit_v2_forward(Pa, x, width_multiplier=width, training=True)
        lossa = F.cross_entropy(la, y, label_smoothing=0.1)
    lossa.backward()
    ga = {k: v.grad.detach().float().clone() for k, v in Pa.items() if v.requires_grad and v.grad is not None}
    la = la.detach().float().clone()
    del Pa
    torch.cuda.empty_cache()

    e_log, a_log = rel_l2(ours_logits, l32), rel_l2(la, l32)
    keys = [k for k in ours if k in g32]
    flat = lambda d: torch.cat([d[k].flatten().double() for k in keys])  # noqa: E731
    cos_all, cos_all_a = cosine(flat(ours), flat(g32)), cosine(flat(ga), flat(g32))
    rel_all, rel_all_a = rel_l2(flat(ours), flat(g32)), rel_l2(flat(ga), flat(g32))
    gnorm = float(flat(g32).norm())
    per = []
    for k in keys:
        n = float(g32[k].norm())
        per.append((k, n / gnorm, cosine(ours[k], g32[k]), cosine(ga[k], g32[k]), rel_l2(ours[k], g32[k]), rel_l2(ga[k], g32[k])))
    sig = [t for t in per if t[1] >= 1e-3]  # parameters carrying a non-negligible share of the gradient
    worst = min(sig, key=lambda t: t[2])
    med_rel = sorted(t[4] for t in sig)[len(sig) // 2]
    med_rel_a = sorted(t[5] for t in sig)[len(sig) // 2]
    rec = {"width": width, "B": B, "logits_rel_l2": e_log, "autocast_logits_rel_l2": a_log, "north_star_1e-3_x": e_log / 1e-3, "loss": ours_loss,
           "loss_fp32": loss32, "loss_autocast": float(lossa),
           "grad_cosine_all": cos_all, "autocast_grad_cosine_all": cos_all_a, "grad_rel_l2_all": rel_all, "autocast_grad_rel_l2_all": rel_all_a,
           "median_param_grad_rel_l2": med_rel, "autocast_median_param_grad_rel_l2": med_rel_a,
           "worst_param": {"name": worst[0], "cosine": worst[2], "autocast_cosine": worst[3]}, "n_params": len(keys), "n_significant": len(sig)}
    return rec, sig


@pytest.mark.parametrize("B", [128, 32])
def test_benchmark_config_train_parity(pkg, B):
    rec, sig = train_parity_record(pkg, B)
    e_log, a_log, ours_loss, loss32 = rec["logits_rel_l2"], rec["autocast_logits_rel_l2"], rec["loss"], rec["loss_fp32"]
    cos_all, rel_all, rel_all_a = rec["grad_cosine_all"], rec["grad_rel_l2_all"], rec["autocast_grad_rel_l2_all"]
    worst = min(sig, key=lambda t: t[2])
    print("\n[parity B=%d train] " % B + json.dumps(rec))
    _record(f"train_B{B}", rec)
    assert e_log <= 8e-2, rec
    assert e_log <= 1.15 * a_log + 2e-3, rec
    assert abs(ours_loss - loss32) <= 2e-3 * abs(loss32), rec
    assert cos_all >= 0.98, rec
    assert rel_all <= 1.15 * rel_all_a + 2e-3, rec
    assert worst[2] >= min(0.95, worst[3] - 1e-2), rec
    for t in sig:
        assert t[4] <= 1.5 * t[5] + 2e-2, t


def test_benchmark_config_eval_parity(pkg):
    B = 128
    model, P = _setup(pkg, 2024)
    model.eval()
    x = O.seeded_input((B, 3, 256, 256), 32).cuda()
    with torch.no_grad():
        a = model(x).float()
        Pg = O.clone_params(P, requires_grad=False, device="cuda")
        ref = O.mobilevit_v2_forward(Pg, x, training=False)
        with torch.autocast("cuda", dtype=torch.bfloat16):
            ac = O.mobilevit_v2_forward(Pg, x, training=False).float()
    e, ea = rel_l2(a, ref), rel_l2(ac, ref)
    top1 = float((a.argmax(1) == ref.argmax(1)).float().mean())
    rec = {"B": B, "eval_logits_rel_l2": e, "autocast_eval_logits_rel_l2": ea, "north_star_1e-3_x": e / 1e-3, "top1_agreement": top1}
    print("\n[parity eval] " + json.dumps(rec))
    _record("eval_B128", rec)
    assert e <= 4e-2, rec
    assert e <= 1.25 * ea + 2e-3, rec
    assert top1 >= 0.95, rec


def stagewise_record(pkg, width=1.0, B=128):
    """Each module fed the fp32 oracle's input of its stage, train mode at 256x256: rel-L2 of its output against the oracle's, per stage."""
    model, P = _setup(pkg, 2024, width)
    model.train()
    model.fuse_boundaries = False
    x = O.seeded_input((B, 3, 256, 256), 31).cuda()
    Pg = O.clone_params(P, requires_grad=False, device="cuda")
    with torch.no_grad():
        ref_logits, stages = O.mobilevit_v2_forward(Pg, x, width_multiplier=width, training=True, return_stages=True)
        names = [pre for _, pre, _ in O.mobilevit_v2_layout(width)]
        rec, prev = {}, x
        for pre in names:
            mod = model
            for part in pre.split("."):
                mod = mod[int(part)] if part.isdigit() else getattr(mod, part)
            out = mod(prev)
            rec[pre] = rel_l2(out, stages[pre])
            prev = stages[pre]
        from ml_cvnets_b200 import functional as Fn
        feats = stages[names[-1]]
        # the classifier head through the public path, on the oracle's last feature map
        saved = model.extract_features
        model.extract_features = lambda t, *a, **k: Fn.to_bf16_cl(feats)
        try:
            head_out = model(x)
        finally:
            model.extract_features = saved
        rec["classifier"] = rel_l2(head_out, ref_logits)
    return rec


def test_benchmark_config_stagewise_parity(pkg):
    """(1) of the module docstring: each module on the oracle's own stage input, batch 128 @ 256x256, train mode."""
    rec = stagewise_record(pkg)
    print("\n[stage-wise parity B=128 train] " + json.dumps(rec))
    _record("stagewise_B128", rec)
    for k, e in rec.items():
        assert e <= 1.5e-2, (k, e, rec)

"""wgmma attention core (csrc/mha_tc.cu) against the fp32 formula AND the mma.sync kernels (csrc/mha.cu), plus same-box A/B timing.

    python tools/check_mha_tc.py [--stage fwd|bwd|time] [--out gpurun_out/mha_tc_check.txt]

Without --stage every stage runs in its own subprocess under a timeout (a dead-locked mbarrier pipeline must not take the box down).
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(1, 16, 1), (2, 64, 2), (2, 77, 8), (2, 128, 2), (1, 129, 1), (2, 197, 12), (2, 256, 2), (3, 200, 3)]


def ref_attn(qkv, B, S, H, scale, amask, kpm):
    import torch
    x = qkv.float().view(B, S, 3, H, 64).permute(2, 0, 3, 1, 4)
    q, k, v = x[0] * scale, x[1], x[2]
    att = q @ k.transpose(-1, -2)
    if amask is not None:
        att = att + amask[:, None]
    if kpm is not None:
        att = att.masked_fill(kpm[:, None, None, :].bool(), float("-inf"))
    att = torch.softmax(att, dim=-1)
    return (att @ v).transpose(1, 2).reshape(B * S, H * 64)


def masks(kind, B, S):
    import torch
    amask = kpm = None
    if kind == "causal":
        amask = torch.full((S, S), float("-inf"), device="cuda").triu(1)[None].repeat(B, 1, 1).contiguous()
    if kind == "padding":
        kpm = torch.zeros(B, S, dtype=torch.uint8, device="cuda")
        kpm[:, S - max(1, S // 5):] = 1
    return amask, kpm


def rel(a, b):
    a, b = a.double(), b.double()
    return float((a - b).norm() / (b.norm() + 1e-30))


def stage_check(which, out):
    import torch
    from ml_cvnets_b200 import _lib as L
    from ml_cvnets_b200 import ops
    lib = L.load()
    torch.backends.cuda.matmul.allow_tf32 = False
    worst = 0.0
    for (B, S, H) in SHAPES:
        for mk in ("none", "causal", "padding"):
            g = torch.Generator(device="cuda").manual_seed(7)
            qkv = torch.randn(B * S, 3 * H * 64, device="cuda", generator=g).to(torch.bfloat16)
            dO = torch.randn(B * S, H * 64, device="cuda", generator=g).to(torch.bfloat16)
            amask, kpm = masks(mk, B, S)
            scale = 64 ** -0.5
            lib.cvb_set_mha_impl(0)
            O0, LSE0 = ops.mha_fwd(qkv, B, S, H, 64, scale, attn_mask=amask, key_padding_mask=kpm)
            x = qkv.float().requires_grad_(True)
            ref = ref_attn(x, B, S, H, scale, amask, kpm)
            rec = {"stage": which, "B": B, "S": S, "H": H, "mask": mk}
            if which == "fwd":
                lib.cvb_set_mha_impl(5)
                O1, LSE1 = ops.mha_fwd(qkv, B, S, H, 64, scale, attn_mask=amask, key_padding_mask=kpm)
                torch.cuda.synchronize()
                rec.update(tc_vs_ref=rel(O1, ref.detach()), old_vs_ref=rel(O0, ref.detach()), lse_maxdiff=float((LSE1 - LSE0).abs().max()),
                           nan=int(torch.isnan(O1.float()).sum()))
                bad = rec["tc_vs_ref"] > 6e-3 or rec["lse_maxdiff"] > 1e-2 or rec["nan"]
            else:
                ref.backward(dO.float())
                D0 = ops.mha_bwd(qkv, O0, dO, LSE0, B, S, H, 64, scale, attn_mask=amask, key_padding_mask=kpm)
                lib.cvb_set_mha_impl(6)
                D1 = ops.mha_bwd(qkv, O0, dO, LSE0, B, S, H, 64, scale, attn_mask=amask, key_padding_mask=kpm)
                torch.cuda.synchronize()
                C = H * 64
                rec.update(tc_vs_ref=rel(D1, x.grad), old_vs_ref=rel(D0, x.grad), dq=rel(D1[:, :C], x.grad[:, :C]), dk=rel(D1[:, C:2 * C], x.grad[:, C:2 * C]),
                           dv=rel(D1[:, 2 * C:], x.grad[:, 2 * C:]), nan=int(torch.isnan(D1.float()).sum()))
                bad = rec["tc_vs_ref"] > 1.2e-2 or rec["nan"]
            rec["ok"] = not bad
            worst = max(worst, rec["tc_vs_ref"])
            out.write(json.dumps(rec) + "\n")
            out.flush()
    lib.cvb_set_mha_impl(3)
    out.write(json.dumps({"stage": which, "worst_rel_l2": worst}) + "\n")


def stage_time(out):
    import torch
    from ml_cvnets_b200 import _lib as L
    from ml_cvnets_b200 import ops
    lib = L.load()
    for (B, S, H, mk) in [(256, 197, 12, "none"), (256, 77, 8, "causal")]:
        g = torch.Generator(device="cuda").manual_seed(7)
        qkv = torch.randn(B * S, 3 * H * 64, device="cuda", generator=g).to(torch.bfloat16)
        dO = torch.randn(B * S, H * 64, device="cuda", generator=g).to(torch.bfloat16)
        amask, kpm = masks(mk, B, S)
        scale = 64 ** -0.5
        rec = {"stage": "time", "B": B, "S": S, "H": H, "mask": mk}
        flops_f = 4.0 * B * H * S * S * 64
        for name, mask in (("old", 0), ("tc", 7)):
            lib.cvb_set_mha_impl(mask)
            O, LSE = ops.mha_fwd(qkv, B, S, H, 64, scale, attn_mask=amask, key_padding_mask=kpm)
            for fn, key, fl in ((lambda: ops.mha_fwd(qkv, B, S, H, 64, scale, attn_mask=amask, key_padding_mask=kpm), "fwd", flops_f),
                                (lambda: ops.mha_bwd(qkv, O, dO, LSE, B, S, H, 64, scale, attn_mask=amask, key_padding_mask=kpm), "bwd", 2.5 * flops_f)):
                for _ in range(3):
                    fn()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                e0.record()
                for _ in range(20):
                    fn()
                e1.record()
                torch.cuda.synchronize()
                us = e0.elapsed_time(e1) * 1000 / 20
                rec[f"{name}_{key}_us"] = round(us, 1)
                rec[f"{name}_{key}_tflops"] = round(fl / us / 1e6, 1)
        out.write(json.dumps(rec) + "\n")
        out.flush()
    lib.cvb_set_mha_impl(3)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--stage", default=None)
    ap.add_argument("--out", default=os.path.join(ROOT, "gpurun_out", "mha_tc_check.txt"))
    a = ap.parse_args()
    os.makedirs(os.path.dirname(a.out), exist_ok=True)
    if a.stage is None:
        rc = 0
        for st in ("fwd", "bwd", "time"):
            try:
                r = subprocess.run([sys.executable, os.path.abspath(__file__), "--stage", st, "--out", a.out], timeout=150)
                code = r.returncode
            except subprocess.TimeoutExpired:
                code = 124
            with open(a.out, "a") as f:
                f.write(json.dumps({"stage": st, "exit": code}) + "\n")
            rc = rc or code
        print(open(a.out).read())
        return rc
    with open(a.out, "a") as out:
        if a.stage == "time":
            stage_time(out)
        else:
            stage_check(a.stage, out)
    return 0


if __name__ == "__main__":
    sys.exit(main())

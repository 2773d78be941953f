"""MobileViT-v1 XS and S, the two modes the recipes train (config/classification/imagenet/mobilevit.yaml, the RangeAugment mobilevit_v1
recipe: ``mit.mode: small``), CPU only.

The fp32 oracle against the real reference's fixtures (tests/golden/make_golden_mit_modes.py), the drop-in model's state_dict against the
reference's key / shape / dtype contract, and the configuration table of all three modes.

The geometry table: every kernel call of the model at the recipe's base crop and per-GPU batch (256x256, 128 images), derived from the oracle's
parameter tree and layout, minus the shapes MobileViT-XXS gives the same kernels.  ``tests/test_mobilevit_v1_modes_gpu.py`` runs each entry.
Restatements of the host-side dispatch rules (csrc/gemm.cu ``cvb_pw_gemm`` / ``dispatch_tile``, csrc/gemm_tc.cu ``cvb_pw_gemm_tc``,
csrc/wgrad_tc.cu ``cvb_pw_wgrad_tc``, csrc/mha.cu, ops.py's wide-layer policy) pin which paths the table reaches: both pointwise GEMM kernels
(including the mma.sync kernel's resident weight panel at K up to 1440 and its narrow ragged tiles), both weight-gradient kernels at
M = 131 072, the mma.sync attention family at head dims 24 - 60, and never the wide-layer pre-pass.

The recipe sampler's crops where a block's token count equals its transformer dim are listed per mode: there the reference's LayerNorm takes
its channel-first branch and the library refuses (modules.py TransformerEncoder.prepare)."""
import json
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import cvnets_oracle as O
from test_oracle_golden import _noise_floor

MODES = ["x_small", "small"]
B, RES = 128, 256        # the recipes' per-GPU batch and base crop (train_batch_size0, crop_size_width)
PATCH, HEADS = 2, 4      # every MobileViT-v1 config: 2x2 patches, 4 heads
FIXTURE = {"x_small": "mobilevit_v1_xs_fp32.pt", "small": "mobilevit_v1_s_fp32.pt"}


def load_mit_fixture(golden_dir, mode):
    """the real reference's record of one mode (tests/golden/make_golden_mit_modes.py writes one file per mode)"""
    return torch.load(os.path.join(golden_dir, FIXTURE[mode]), weights_only=False)


# ------------------------------------------------------------------------------------------- the geometry table
def attn_blocks(mode, batch=B, res=RES):
    """one dict per MobileViTBlock: layer, map size H, channels c, transformer dim d, ffn, encoder count, heads, head dim, tokens S, sequences"""
    shapes = O.mobilevit_v1_shapes(mode)
    out = []
    for kind, pre, kw in O.mobilevit_v1_layout(mode):
        if kind != "mvit":
            continue
        li = int(pre.split("_")[1].split(".")[0])
        c = shapes[pre + ".fusion.block.conv.weight"].shape[0]
        d = shapes[pre + ".local_rep.conv_1x1.block.conv.weight"].shape[0]
        ffn = shapes[pre + ".global_rep.0.pre_norm_ffn.1.weight"].shape[0]
        H = res >> li
        out.append(dict(layer=li, pre=pre, H=H, c=c, d=d, ffn=ffn, n=kw["n_blocks"], heads=HEADS, hd=d // HEADS, S=(H // PATCH) ** 2,
                        seqs=batch * PATCH * PATCH, B=batch))
    return out


def inverted_residuals(mode, res=RES):
    """(prefix, H_in, Cin, hid, Cout, stride) of every InvertedResidual"""
    shapes = O.mobilevit_v1_shapes(mode)
    out, H = [], res // 2
    for kind, pre, kw in O.mobilevit_v1_layout(mode):
        if kind != "ir":
            continue
        hid, cin = shapes[pre + ".block.exp_1x1.block.conv.weight"].shape[:2]
        cout = shapes[pre + ".block.red_1x1.block.conv.weight"].shape[0]
        out.append((pre, H, cin, hid, cout, kw["stride"]))
        H = (H - 1) // kw["stride"] + 1
    return out


def head(mode):
    """(Cin, Cout) of conv_1x1_exp and (Cin, classes) of the classifier; conv_1x1_exp runs on the 8x8 map of a 256x256 input"""
    shapes = O.mobilevit_v1_shapes(mode)
    e = shapes["conv_1x1_exp.block.conv.weight"]
    return (e.shape[1], e.shape[0]), tuple(shapes["classifier.fc.weight"].shape[::-1])


def units(mode, batch=B):
    """every kernel-level unit of the model at batch x 256x256: (kind, shape key, description); the shape key holds every dimension the
    kernels see (M included) and nothing else, so equal keys are the same kernel calls"""
    out = []
    for g in attn_blocks(mode, batch):
        M = batch * g["H"] ** 2
        out += [("attention", (g["seqs"], g["S"], g["heads"], g["hd"]), g),
                ("conv3x3", (batch, g["H"], g["c"], g["c"]), dict(g, conv="local_rep.conv_3x3")),
                ("conv3x3", (batch, g["H"], 2 * g["c"], g["c"]), dict(g, conv="fusion")),
                ("block_1x1", (M, g["c"], g["d"]), g),
                ("encoder", (M, g["d"], g["ffn"], g["S"]), g),
                ("layernorm", (M, g["d"]), g),
                ("tokens", (batch, g["H"], g["c"], g["d"]), g)]
    for pre, H, cin, hid, cout, s in inverted_residuals(mode):
        out.append(("ir", (batch, H, cin, hid, cout, s), dict(pre=pre, H=H, cin=cin, hid=hid, cout=cout, stride=s, B=batch)))
    (ce, ex), (cf, ncls) = head(mode)
    out.append(("head", (batch, ce, ex, ncls), dict(B=batch, cin=ce, exp=ex, ncls=ncls, HW=(RES >> 5) ** 2)))
    return out


def table():
    """the units of XS and S, each shape once, minus those XXS gives the same kernels: {id: (kind, description)}"""
    seen = {(k, key) for k, key, _ in units("xx_small")}
    out = {}
    for mode in MODES:
        for kind, key, desc in units(mode):
            if (kind, key) in seen:
                continue
            seen.add((kind, key))
            where = desc.get("pre") or "head"
            uid = f"{mode}-{where}" + (f"-{desc['conv'].split('.')[-1]}" if "conv" in desc else "") + f"-{kind}"
            out[uid] = (kind, dict(desc, mode=mode))
    return out


# ------------------------------------------------------------------------------------------- the GEMMs of each unit
def unit_gemms(kind, g):
    """(name, M, N, K, a_mode, e_mode) of the pointwise GEMMs and (name, M, N, K, g_mode, a_mode) of the weight gradients one unit issues
    (functional.py PointwiseConvFn / InvertedResidualFn / _encoder_forward / _encoder_backward / PoolLinearFn / LinearFn)"""
    from ml_cvnets_b200 import ops as o
    fwd, wg = [], []
    if kind == "conv3x3":
        M, cin, cout = g["B"] * g["H"] ** 2, (2 * g["c"] if g["conv"] == "fusion" else g["c"]), g["c"]
        fwd += [("fwd", M, cout, 9 * cin, o.A_RAW, o.E_STORE), ("dgrad", M, 9 * cin, cout, o.A_BNB, o.E_STORE)]
        wg += [("wgrad", M, cout, 9 * cin, o.A_BNB, o.A_RAW)]
    elif kind == "block_1x1":
        M, c, d = g["B"] * g["H"] ** 2, g["c"], g["d"]
        fwd += [("conv_1x1", M, d, c, o.A_RAW, o.E_STORE), ("conv_1x1 dgrad", M, c, d, o.A_RAW, o.E_STORE),
                ("conv_proj", M, c, d, o.A_RAW, o.E_STORE), ("conv_proj dgrad", M, d, c, o.A_BNB, o.E_STORE)]
        wg += [("conv_1x1 wgrad", M, d, c, o.A_RAW, o.A_RAW), ("conv_proj wgrad", M, c, d, o.A_BNB, o.A_RAW)]
    elif kind == "encoder":
        M, C, ffn = g["B"] * g["H"] ** 2, g["d"], g["ffn"]
        fwd += [("qkv", M, 3 * C, C, o.A_GN, o.E_STORE), ("out_proj", M, C, C, o.A_RAW, o.E_STORE), ("ffn1", M, ffn, C, o.A_GN, o.E_STORE),
                ("ffn2", M, C, ffn, o.A_SILU, o.E_STORE), ("ffn2 (dropout)", M, C, ffn, o.A_RAW, o.E_STORE),
                ("ffn2 dgrad", M, ffn, C, o.A_RAW, o.E_SILU_BWD), ("ffn2 dgrad (dropout)", M, ffn, C, o.A_RAW, o.E_STORE),
                ("ffn1 dgrad", M, C, ffn, o.A_RAW, o.E_STORE), ("out_proj dgrad", M, C, C, o.A_RAW, o.E_STORE),
                ("qkv dgrad", M, C, 3 * C, o.A_RAW, o.E_STORE)]
        wg += [("ffn2 wgrad", M, C, ffn, o.A_RAW, o.A_SILU), ("ffn2 wgrad (dropout)", M, C, ffn, o.A_RAW, o.A_RAW),
               ("ffn1 wgrad", M, ffn, C, o.A_RAW, o.A_GN), ("out_proj wgrad", M, C, C, o.A_RAW, o.A_RAW), ("qkv wgrad", M, 3 * C, C, o.A_RAW, o.A_GN)]
    elif kind == "ir":
        M, M2 = g["B"] * g["H"] ** 2, g["B"] * ((g["H"] - 1) // g["stride"] + 1) ** 2
        cin, hid, cout = g["cin"], g["hid"], g["cout"]
        fwd += [("exp_1x1", M, hid, cin, o.A_RAW, o.E_STORE), ("red_1x1", M2, cout, hid, o.A_AFF_SILU, o.E_STORE),
                ("red_1x1 dgrad", M2, hid, cout, o.A_BNB, o.E_SILU_BWD), ("exp_1x1 dgrad", M, cin, hid, o.A_BNB, o.E_STORE)]
        wg += [("red_1x1 wgrad", M2, cout, hid, o.A_BNB, o.A_AFF_SILU), ("exp_1x1 wgrad", M, hid, cin, o.A_BNB, o.A_RAW)]
    elif kind == "head":
        M, npad = g["B"] * g["HW"], (g["ncls"] + 7) // 8 * 8
        fwd += [("conv_1x1_exp", M, g["exp"], g["cin"], o.A_RAW, o.E_STORE), ("conv_1x1_exp dgrad", M, g["cin"], g["exp"], o.A_BNB, o.E_STORE),
                ("classifier", g["B"], npad, g["exp"], o.A_RAW, o.E_STORE), ("classifier dgrad", g["B"], g["exp"], npad, o.A_RAW, o.E_STORE)]
        wg += [("conv_1x1_exp wgrad", M, g["exp"], g["cin"], o.A_BNB, o.A_RAW), ("classifier wgrad", g["B"], npad, g["exp"], o.A_RAW, o.A_RAW)]
    return fwd, wg


# ------------------------------------------------------------------------------------------- restatements of the host dispatch rules
def gemm_kernel(N, K, a_mode):
    """cvb_pw_gemm: the wgmma kernel for N >= 96 unless a ragged last 128-channel tile would stay mostly idle (cvb_pw_gemm_tc); else the
    mma.sync kernel with its weight panel resident in shared memory (dispatch_tile / launch_gemm): the widest N tile that leaves two CTAs
    per SM a >= 4-stage ring, else one CTA per SM with >= 3 stages -> ("wgmma", None) or ("mma.sync", (BN, CTAs per SM))"""
    from ml_cvnets_b200 import ops as o
    if N >= 96 and not (N % 128 != 0 and N % 128 < 64 and N < 256):
        return "wgmma", None
    KT = (K + 31) // 32
    nvec = {o.A_AFF: 2, o.A_AFF_SILU: 2, o.A_GN: 2, o.A_BNB: 3}.get(a_mode, 0)
    a_stage = 128 * 32 * 2 * (2 if a_mode == o.A_BNB else 1)

    def fits(BN, two):
        fixed = KT * BN * 64 + 128 * (BN + 8) * 2 + nvec * KT * 128 + 1024
        budget = (108 if two else 216) * 1024
        nst = min(8, (budget - fixed) // a_stage) if fixed < budget else 0
        return nst >= (4 if two else 3)

    want128 = N > 64 and (N + 63) // 64 * 64 >= (N + 127) // 128 * 128
    order = ([(128, True)] if want128 else []) + ([(64, True)] if N > 32 else [(32, True)])
    order += ([(128, False)] if want128 else []) + ([(64, False)] if N > 32 else []) + [(32, False)]
    for BN, two in order:
        if fits(BN, two):
            return "mma.sync", (BN, 2 if two else 1)
    return "wgmma", None  # K too large for any resident panel: the wgmma kernel streams the weights


def wgrad_kernel(N, K, g_mode):
    """cvb_pw_wgrad: the wgmma kernel (wgrad_tc.cu) for K % 64 == 0, N >= 32 and not both N, K <= 64; else the mma.sync split-K kernel,
    whose partials meet in fp64 atomics"""
    from ml_cvnets_b200 import ops as o
    if K % 64 == 0 and K >= 64 and N >= 32 and not (N <= 64 and K <= 64) and g_mode in (o.A_RAW, o.A_BNB):
        return "wgmma"
    return "mma.sync"


def prepass(kind, N, K, mode):
    """ops.pw_gemm / pw_wgrad materialise a load-mode prologue first for wide late-stage layers (WIDE_K / WIDE_N / WIDE_N_WGRAD)"""
    from ml_cvnets_b200 import ops as o
    return mode != o.A_RAW and K >= o.WIDE_K and N >= (o.WIDE_N if kind == "fwd" else o.WIDE_N_WGRAD)


def attention_family(hd, S):
    """csrc/mha.cu: head_dim != 64 runs the mma.sync kernels with a whole head in shared memory (S <= 256); head_dim 64 the wgmma ones"""
    assert S <= 256 or hd == 64
    return "mma.sync" if hd != 64 else "wgmma"


def head_load_chunk(hd):
    """mha.cu load_rows: 16-byte chunks at the padded head dim, 8-byte chunks for hd % 4 == 0, else 4-byte chunks"""
    return 16 if hd in (16, 32, 64) else (8 if hd % 4 == 0 else 4)


def gemm_routes():
    """(unit id, gemm name, M, N, K, kernel, mma.sync tile) of every pointwise GEMM, and (unit id, name, M, N, K, kernel) of every weight gradient"""
    fw, wg = [], []
    for uid, (kind, g) in table().items():
        f, w = unit_gemms(kind, g)
        fw += [(uid, name, M, N, K, *gemm_kernel(N, K, a)) for name, M, N, K, a, _ in f]
        wg += [(uid, name, M, N, K, wgrad_kernel(N, K, gm)) for name, M, N, K, gm, _ in w]
    return fw, wg


# ------------------------------------------------------------------------------------------- the recipe sampler's crops
def recipe_crops(base=RES, lo=160, hi=320, n_scales=5, div=32):
    """data/sampler/utils.py image_batch_pairs for the recipes' settings (crop 256, 160 - 320, 5 scales, multiples of 32): (crop, batch)"""
    from ml_cvnets_b200.modules import make_divisible
    crops = sorted({make_divisible(v, div) for v in set(np.linspace(lo, hi, n_scales)) | {base}})
    return [(c, max(1, int(round(base * base * B / (c * c), 2)))) for c in crops]


def colliding_crops(mode):
    """crops at which some MobileViTBlock has as many tokens per patch position as transformer channels (N == d)"""
    out = []
    for crop, _ in recipe_crops():
        for g in attn_blocks(mode, res=crop):
            if g["H"] % PATCH == 0 and g["S"] == g["d"]:
                out.append((crop, g["layer"], g["d"]))
    return out


# ------------------------------------------------------------------------------------------- tests: fixtures, contract, configuration
@pytest.fixture(scope="module")
def contract(golden_dir):
    with open(os.path.join(golden_dir, "state_dict_contract_mit.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("mode", MODES)
def test_oracle_matches_reference(golden_dir, mode):
    """eval forward at 1x3x256x256 and a train-mode forward / backward at 2x3x256x256: the tolerances of test_oracle_golden.py's XXS test"""
    from golden_sample import at_sample
    fx = load_mit_fixture(golden_dir, mode)
    assert fx["mode"] == mode and fx["res"] == RES
    shapes = O.mobilevit_v1_shapes(mode)
    assert {k: list(v.shape) for k, v in shapes.items()} == {k: s for k, s in fx["keys"]}
    P = O.clone_params(O.seeded_fill_(shapes, fx["seed"]))
    with torch.no_grad():
        ev = O.mobilevit_v1_forward(P, O.seeded_input((1, 3, RES, RES), fx["eval_x_seed"]), mode=mode, training=False)
    assert float((ev - fx["eval_logits"]).norm() / fx["eval_logits"].norm()) <= 2e-5
    logits = O.mobilevit_v1_forward(P, O.seeded_input((fx["batch"], 3, RES, RES), fx["x_seed"]), mode=mode, training=True)
    loss = F.cross_entropy(logits, fx["labels"], label_smoothing=0.1)
    loss.backward()
    assert float((logits.detach() - fx["logits"]).norm() / fx["logits"].norm()) <= 5e-5
    assert abs(float(loss) - float(fx["loss"])) <= 1e-5
    assert fx["grad_norms"].keys() == {k for k, p in P.items() if p.requires_grad}
    for k, n in fx["grad_norms"].items():
        assert abs(float(P[k].grad.norm()) - n) <= 2e-3 * n + 1e-6, (k, float(P[k].grad.norm()), n)
    floor = _noise_floor(fx["grad_norms"].values())
    for k, g in fx["grads"].items():
        if fx["grad_norms"][k] < floor:
            assert float(P[k].grad.norm()) < 2 * floor, k
            continue
        ours, ref = at_sample(P[k].grad, g)
        assert float((ours - ref).norm() / (ref.norm() + 1e-12)) <= 2e-3, k


@pytest.mark.parametrize("mode", MODES)
def test_state_dict_contract(contract, mode):
    import ml_cvnets_b200 as m
    entries = contract[mode]
    sd = m.MobileViT(m.default_mit_opts(mode)).state_dict()
    assert list(sd.keys()) == [e[0] for e in entries]
    for k, shape, dtype in entries:
        assert list(sd[k].shape) == shape and str(sd[k].dtype) == "torch." + dtype, k
    assert {k: list(v.shape) for k, v in O.mobilevit_v1_shapes(mode).items()} == {k: shape for k, shape, _ in entries}


@pytest.mark.parametrize("mode", ["xx_small", "x_small", "small"])
def test_configuration_matches_oracle(mode):
    import ml_cvnets_b200 as m
    cfg = m.get_mit_configuration(m.default_mit_opts(mode))
    e, c1, c2, mits = O.MIT_MODES[mode]
    assert (cfg["layer1"]["expand_ratio"], cfg["layer1"]["out_channels"], cfg["layer2"]["out_channels"]) == (e, c1, c2)
    assert cfg["layer2"]["expand_ratio"] == e and cfg["last_layer_exp_factor"] == 4
    for i, (co, d, f, n) in enumerate(mits):
        c = cfg[f"layer{3 + i}"]
        assert (c["out_channels"], c["transformer_channels"], c["ffn_dim"], c["transformer_blocks"], c["mv_expand_ratio"]) == (co, d, f, n, e)
        assert (c["patch_h"], c["patch_w"], c["num_heads"], c["stride"]) == (PATCH, PATCH, HEADS, 2)


# ------------------------------------------------------------------------------------------- tests: the table and the paths it reaches
def test_geometry_table():
    blocks = {m: [(g["H"], g["c"], g["d"], g["ffn"], g["n"], g["hd"], g["S"]) for g in attn_blocks(m)] for m in MODES}
    assert blocks == {"x_small": [(32, 64, 96, 192, 2, 24, 256), (16, 80, 120, 240, 4, 30, 64), (8, 96, 144, 288, 3, 36, 16)],
                      "small": [(32, 96, 144, 288, 2, 36, 256), (16, 128, 192, 384, 4, 48, 64), (8, 160, 240, 480, 3, 60, 16)]}
    assert head("x_small") == ((96, 384), (384, 1000)) and head("small") == ((160, 640), (640, 1000))
    assert [ir[3] for ir in inverted_residuals("small")] == [64, 128, 256, 256, 256, 384, 512]  # expand ratio 4
    t = table()
    kinds = {}
    for kind, _ in t.values():
        kinds[kind] = kinds.get(kind, 0) + 1
    # layer_2.2 repeats layer_2.1, and layer_1.0 (16 -> 32, expand 4, 128^2) is the same in both modes; every other unit is new
    assert kinds == {"attention": 6, "conv3x3": 12, "block_1x1": 6, "encoder": 6, "layernorm": 6, "tokens": 6, "ir": 11, "head": 2}, kinds
    assert {g["hd"] for k, g in t.values() if k == "attention"} == {24, 30, 36, 48, 60}
    assert all(g["seqs"] == 512 for k, g in t.values() if k == "attention")


def test_pointwise_gemm_routes():
    """the table reaches the wgmma kernel and the mma.sync kernel, the latter with its resident weight panel at K up to 1440 (two CTAs per SM
    and one), and with 32-channel tiles whose last tile is ragged (N = 80 at K = 1440)"""
    fw, _ = gemm_routes()
    routes = {r[5] for r in fw}
    assert routes == {"wgmma", "mma.sync"}
    narrow = [r for r in fw if r[5] == "mma.sync"]
    assert all(r[3] < 96 or r[3] % 128 < 64 for r in narrow)
    assert max(r[4] for r in narrow if r[3] < 96) == 1440
    assert {r[6][1] for r in narrow} == {1, 2}
    assert any(r[3] == 80 and r[4] == 1440 and r[6] == (32, 1) for r in narrow), sorted({(r[3], r[4], r[6]) for r in narrow})
    assert any(r[3] in (144, 160) for r in narrow)  # ragged N >= 96 left to mma.sync
    # the dense convs' input-gradient GEMMs write N = 9 Cin up to 2880 on the wgmma kernel, most with a ragged last 128-channel tile
    dg = [r for r in fw if r[1] == "dgrad"]
    assert max(r[3] for r in dg) == 2880 and all(r[5] == "wgmma" for r in dg)
    assert {r[3] % 128 for r in dg} - {0}


def test_weight_gradient_routes():
    """K % 64 splits the dense convs' weight gradients between the two kernels, both at M = 131 072"""
    _, wg = gemm_routes()
    dense = {(r[4], r[5]) for r in wg if r[1] == "wgrad"}
    assert {K for K, _ in dense} == {576, 720, 864, 1152, 1440, 1728, 2304, 2880}
    assert {K for K, k in dense if k == "mma.sync"} == {720, 864, 1440}
    assert max(r[2] for r in wg if r[1] == "wgrad" and r[5] == "mma.sync") == 131072
    assert max(r[2] for r in wg if r[1] == "wgrad" and r[5] == "wgmma") == 131072


def test_attention_family_and_head_loads():
    t = table()
    att = [g for k, g in t.values() if k == "attention"]
    assert {attention_family(g["hd"], g["S"]) for g in att} == {"mma.sync"}
    assert {head_load_chunk(g["hd"]) for g in att} == {8, 4}  # head_dim 30 takes the 4-byte path
    assert {g["hd"] for g in att if head_load_chunk(g["hd"]) == 4} == {30}


def test_wide_layer_prepass_never_fires():
    from ml_cvnets_b200 import ops as o
    fires = []
    for uid, (kind, g) in table().items():
        f, w = unit_gemms(kind, g)
        fires += [(uid, n) for n, M, N, K, a, _ in f if prepass("fwd", N, K, a)]
        fires += [(uid, n) for n, M, N, K, _, a in w if prepass("wgrad", N, K, a)]
        if kind == "encoder":
            C, ffn = g["d"], g["ffn"]
            assert not (C >= o.WIDE_K and 3 * C >= o.WIDE_N_WGRAD and ffn >= o.WIDE_N_WGRAD)  # functional._encoder_forward keep_n
    assert not fires, fires


def test_recipe_crops_where_the_library_refuses():
    assert recipe_crops() == [(160, 327), (192, 227), (256, 128), (288, 101), (320, 81)]
    assert {m: colliding_crops(m) for m in ["xx_small", "x_small", "small"]} == {"xx_small": [], "x_small": [], "small": [(192, 3, 144)]}

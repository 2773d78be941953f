"""CPU-only checks (-m "not gpu"): the C-ABI library loads and exports every symbol include/cvnets_b200.h declares, the
host-side mirror keeps the reference's state_dict / signature contract, the product refuses to run without CUDA, the
drop-in modules match the reference classes' recorded contract (tests/golden/reference_contract.json), and the N>1 host logic
works under gloo."""
import hashlib
import inspect
import json
import os
import re
import subprocess
import sys

import pytest
import torch

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    import __graft_entry__ as ge
    ge.build()
    from ml_cvnets_b200 import _lib
    hdr = open(os.path.join(REPO, "include", "cvnets_b200.h")).read()
    declared = set(re.findall(r"CVB_API\s+(?:const\s+char\*|int)\s+(cvb_[a-z0-9_]+)\s*\(", hdr))
    assert len(declared) >= 20
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), name
    assert lib.cvb_abi_version() == _lib.ABI_VERSION
    out = subprocess.run(["nm", "-D", _lib.LIB_PATH], capture_output=True, text=True).stdout
    exported = set(re.findall(r" T (cvb_[a-z0-9_]+)", out))
    assert declared <= exported


def test_struct_layouts_match_c_compiler(tmp_path):
    """The C compiler's sizeof / offsetof of every argument struct, and sizeof of every scalar parameter type, equal the derived ctypes
    types': same field types and layout, not just the same names."""
    import ctypes
    from ml_cvnets_b200 import _lib
    structs = {n: t for n, t in vars(_lib).items() if isinstance(t, type) and issubclass(t, ctypes.Structure) and t is not ctypes.Structure}
    assert set(structs) == {"cvb_gemm_args", "cvb_wgrad_args", "cvb_dw_fwd_args", "cvb_dw_bwd_args", "cvb_prep_desc", "cvb_cast_desc"}
    want = {}
    for name, cls in structs.items():
        want[f"sizeof({name})"] = ctypes.sizeof(cls)
        want.update({f"offsetof({name}, {f})": getattr(cls, f).offset for f, _ in cls._fields_})
    scalars = dict(_lib._SCALARS, **{"void*": ctypes.c_void_p, "const char*": ctypes.c_char_p})
    want.update({f"sizeof({t})": ctypes.sizeof(c) for t, c in scalars.items()})
    probe = tmp_path / "probe.c"
    probe.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "cvnets_b200.h"\nint main(void) {\n'
                     + "".join(f'  printf("%s %zu\\n", "{k}", {k});\n' for k in want) + "  return 0;\n}\n")
    subprocess.run(["cc", "-std=c99", "-Wall", "-Werror", "-I", os.path.dirname(_lib.HEADER), str(probe), "-o", str(tmp_path / "probe")],
                   check=True)
    out = subprocess.run([str(tmp_path / "probe")], capture_output=True, text=True, check=True).stdout
    got = {k: int(v) for k, v in (line.rsplit(" ", 1) for line in out.splitlines())}
    assert got == want


def test_derived_signatures_at_abi_12():
    """Spot checks of the header -> ctypes mapping: int64_t, double, struct pointers, device descriptor tables, pointer arrays, const char*,
    and the ABI 12 constants."""
    import ctypes
    from ml_cvnets_b200 import _lib
    sigs = _lib._PROTOTYPES
    assert sigs["cvb_stem_im2col"][1][1:5] == [ctypes.c_int64] * 4 and sigs["cvb_stem_im2col"][1][5] is ctypes.c_int
    assert sigs["cvb_stem_im2col"][1][8:] == [ctypes.c_void_p] * 3  # A, mix (device float[6] or NULL), stream
    assert sigs["cvb_bn_finalize"][1][2] is ctypes.c_double and sigs["cvb_bn_finalize"][1][5] is ctypes.c_float
    assert sigs["cvb_na_compose"][1][3] is ctypes.POINTER(ctypes.c_void_p)
    assert sigs["cvb_na_param_grad"][1][4] is sigs["cvb_na_param_grad"][1][6] is ctypes.POINTER(ctypes.c_void_p)
    assert sigs["cvb_pw_gemm"] == (ctypes.c_int, [ctypes.POINTER(_lib.cvb_gemm_args), ctypes.c_void_p])
    assert sigs["cvb_prep_weights"][1][0] is ctypes.c_void_p  # descs_device: an address in device memory
    assert sigs["cvb_last_error"] == (ctypes.c_char_p, [])
    assert (_lib.ABI_VERSION, _lib.A_BNB, _lib.E_LIN_BWD, _lib.ACT_SIGMOID, _lib.PREP_PATCH_T) == (12, 5, 4, 5, 5)


def test_header_parser_rejects_unknown_input(tmp_path):
    from ml_cvnets_b200 import _lib
    hdr = open(_lib.HEADER).read()
    proto = "CVB_API int cvb_act_fwd(const void* X, void* Y, int64_t n, int kind, cvb_stream_t stream);"
    assert proto in hdr
    for bad in (hdr.replace(proto, proto.replace("int64_t n", "long n")), hdr.replace(proto, proto + "\nstatic int cvb_counter;")):
        (tmp_path / "h.h").write_text(bad)
        with pytest.raises(_lib.CvbError, match="unrecognised"):
            _lib._parse(str(tmp_path / "h.h"))


def test_failed_status_raises_with_the_library_message():
    import __graft_entry__ as ge
    ge.build()
    from ml_cvnets_b200 import _lib
    with pytest.raises(_lib.CvbError, match=r"^cvb_act_fwd failed \(rc=1\): cvb_act_fwd: bad arguments$"):
        _lib.load().cvb_act_fwd(None, None, 8, _lib.ACT_GELU, None)  # argument validation fails before any CUDA call


def test_apply_load_mode_rejects_shapes_past_its_row_kernel():
    """cvb_apply_load_mode runs a row-block kernel (a thread per 8 channels of a row, int row index): more than 8192 channels or 2^31 rows
    are rejected before any CUDA call."""
    import __graft_entry__ as ge
    ge.build()
    from ml_cvnets_b200 import _lib
    lib, p = _lib.load(), 256  # p: a non-NULL address that is never dereferenced
    with pytest.raises(_lib.CvbError, match=r"cvb_apply_load_mode: K = 8200, M = 100 "):
        lib.cvb_apply_load_mode(p, 8200, None, 0, _lib.A_AFF, p, p, None, None, None, 0, p, 8200, 100, 8200, None)
    with pytest.raises(_lib.CvbError, match=r"cvb_apply_load_mode: K = 64, M = 2147483648 "):
        lib.cvb_apply_load_mode(p, 64, None, 0, _lib.A_AFF, p, p, None, None, None, 0, p, 64, 1 << 31, 64, None)


def test_state_dict_contract_and_signatures(golden_dir):
    import ml_cvnets_b200 as m
    with open(os.path.join(golden_dir, "state_dict_contract.json")) as f:
        contract = json.load(f)
    for width, entries in contract.items():
        sd = m.MobileViTv2(m.default_opts(width_multiplier=float(width))).state_dict()
        assert list(sd.keys()) == [e[0] for e in entries]
        for k, shape, dtype in entries:
            assert list(sd[k].shape) == shape and str(sd[k].dtype) == "torch." + dtype, k
    # constructor signatures of the drop-ins (SURVEY.md 8b)
    assert list(inspect.signature(m.InvertedResidual.__init__).parameters)[1:8] == [
        "opts", "in_channels", "out_channels", "stride", "expand_ratio", "dilation", "skip_connection"]
    assert list(inspect.signature(m.MobileViTBlockv2.__init__).parameters)[1:14] == [
        "opts", "in_channels", "attn_unit_dim", "ffn_multiplier", "n_attn_blocks", "attn_dropout", "dropout", "ffn_dropout",
        "patch_h", "patch_w", "conv_ksize", "dilation", "attn_norm_layer"]
    assert list(inspect.signature(m.LinearSelfAttention.__init__).parameters)[1:5] == ["opts", "embed_dim", "attn_dropout", "bias"]
    model = m.MobileViTv2(m.default_opts())
    groups, mult = model.get_trainable_parameters(weight_decay=0.05, no_decay_bn_filter_bias=True)
    assert [len(g["params"]) for g in groups] == [65, 129] and mult == [1.0, 1.0]  # SURVEY.md App. B


def test_no_cpu_fallback():
    import ml_cvnets_b200 as m
    model = m.MobileViTv2(m.default_opts(width_multiplier=0.5))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        model(torch.randn(1, 3, 64, 64))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        m.InvertedResidual(m.default_opts(), 16, 16, 1, 2)(torch.randn(1, 16, 8, 8))
    # the stand-alone layers have kernel paths of their own (round 2) -- and likewise no CPU path
    for layer, x in ((m.LinearSelfAttention(m.default_opts(), 16), torch.randn(1, 16, 4, 4)), (m.LayerNorm2D_NCHW(16), torch.randn(1, 16, 4, 4)),
                     (m.LayerNorm(16), torch.randn(1, 4, 16)), (m.LinearLayer(16, 16), torch.randn(1, 4, 16)), (m.GlobalPool(), torch.randn(1, 16, 4, 4)),
                     (m.ConvLayer2d(m.default_opts(), 16, 16, 1), torch.randn(1, 16, 4, 4))):
        with pytest.raises(RuntimeError, match="no CPU fallback"):
            layer(x)
    with pytest.raises(RuntimeError, match="no CPU"):
        m.cross_entropy(torch.randn(2, 8), torch.tensor([1, 2]))


def test_product_does_not_import_the_oracle():
    for root, _, files in os.walk(os.path.join(REPO, "ml-cvnets_b200")):
        for fn in files:
            if fn.endswith((".py", ".cu", ".cuh")):
                src = open(os.path.join(root, fn)).read()
                assert "oracle" not in src.replace("no oracle", ""), f"{fn} mentions the oracle"


@pytest.fixture(scope="module")
def ref_contract(golden_dir):
    """Signatures, state_dict entries, child trees and reprs of the reference classes (tests/golden/make_golden_contract.py)."""
    with open(os.path.join(golden_dir, "reference_contract.json")) as f:
        return json.load(f)


def _sd_entries(mod):
    return [[k, list(v.shape), str(v.dtype)] for k, v in mod.state_dict().items()]


def _sd_digest(mod):
    e = _sd_entries(mod)
    return {"n_entries": len(e), "sha256": hashlib.sha256(json.dumps(e, separators=(",", ":")).encode()).hexdigest()}


def _params(f):
    return [p for p in inspect.signature(f).parameters if p not in ("args", "kwargs")]


def test_registration_with_reference_checkout(ref_contract):
    """The assemblers register.py registers with the reference (mobilevit_v2 / mobilevit / vit replacements) build the reference models'
    exact state_dicts: keys, shapes, dtypes and parameter count."""
    import ml_cvnets_b200 as m
    ours = m.MobileViTv2(m.default_opts(width_multiplier=1.0, **{"model.activation.name": "swish"}))
    ref = ref_contract["mobilevit_v2"]
    assert _sd_digest(ours) == ref["state_dict"]
    assert sum(p.numel() for p in ours.parameters()) == ref["n_params"] == 4901841
    assert len(ours._chain) == 10 and ours.fuse_boundaries and ours._chain[0] is ours.conv_1
    seg = m.MobileViTv2(m.default_opts(width_multiplier=1.0), output_stride=8)
    assert seg.layer_5[1].local_rep[0].block.conv.dilation == (4, 4)                                   # segmentation heads: output_stride is honoured
    assert _sd_digest(m.MobileViT(m.default_mit_opts("xx_small"))) == ref_contract["mobilevit_xx_small"]["state_dict"]
    assert _sd_digest(m.VisionTransformer(m.default_vit_opts("tiny"))) == ref_contract["vit_tiny"]["state_dict"]


def test_transformer_dropins_match_reference_contract(ref_contract):
    """MultiHeadAttention / TransformerEncoder: same constructor parameters, forward parameters, state_dict keys and shapes as the
    reference classes (SURVEY.md 8b)."""
    import ml_cvnets_b200 as ours
    ref = ref_contract["transformer"]
    assert _params(ours.MultiHeadAttention.__init__) == ref["params"]["mha_init"]
    assert _params(ours.MultiHeadAttention.forward)[:5] == ["self", "x_q", "x_kv", "key_padding_mask", "attn_mask"]
    assert _params(ours.TransformerEncoder.__init__) == ref["params"]["enc_init"]
    assert _params(ours.TransformerEncoder.forward) == ref["params"]["enc_forward"]
    for act in ("swish", "gelu"):
        a = ours.TransformerEncoder(ours.default_opts(**{"model.activation.name": act}), 64, 128, num_heads=4)
        assert _sd_entries(a) == ref[act]["state_dict"], act
        assert float(a.pre_norm_mha[0].eps) == ref[act]["eps"]
        assert repr(a).split("(")[0] == ref[act]["repr_head"]
    assert list(ours.MultiHeadAttention(64, 4).state_dict().keys()) == ref["mha_state_dict"]
    with pytest.raises(RuntimeError):
        a(torch.zeros(2, 5, 64))  # CPU input must raise


def test_se_block_and_dropout_children_match_reference_contract(ref_contract):
    """InvertedResidualSE / SqueezeExcitation (SURVEY.md 8f row 4) and the dropout / stochastic-depth children of TransformerEncoder: constructor
    parameters, child tree, state_dict keys / shapes and repr against the reference classes."""
    import ml_cvnets_b200 as ours
    ref = ref_contract["inverted_residual_se"]
    assert _params(ours.InvertedResidualSE.__init__) == ref["params"]["se_init"]
    assert _params(ours.SqueezeExcitation.__init__) == ref["params"]["sq_init"]
    opts = ours.default_opts(**{"model.activation.name": ref["activation"]})
    assert len(ref["configs"]) == 4
    for cfg in ref["configs"]:
        a = ours.InvertedResidualSE(opts, 24, 24, **cfg["kwargs"])
        assert _sd_entries(a) == cfg["state_dict"], cfg["kwargs"]
        assert [n for n, _ in a.block.named_children()] == cfg["children"]
        assert list(a.block._modules) == cfg["modules"]                       # incl. the shared activation registered twice
        assert repr(a) == cfg["repr"], (repr(a), cfg["repr"])
        assert a.use_res_connect == cfg["use_res_connect"]
    enc = ref
    e1 = ours.TransformerEncoder(opts, 64, 128, num_heads=4, dropout=0.1, ffn_dropout=0.2)
    assert [type(m).__name__ for m in e1.pre_norm_ffn] == enc["dropout_children"]["pre_norm_ffn"]
    assert [e1.pre_norm_mha[2].p, e1.pre_norm_ffn[3].p, e1.pre_norm_ffn[5].p] == enc["dropout_children"]["p"]
    s1 = ours.TransformerEncoder(opts, 64, 128, num_heads=4, stochastic_dropout=0.2)
    assert type(s1.drop_path).__name__ == enc["stochastic"]["drop_path"] == "StochasticDepth" and s1.drop_path.p == enc["stochastic"]["p"]
    assert list(s1.state_dict().keys()) == enc["stochastic"]["state_dict_keys"]


def _gloo_worker(rank, world, port, q):
    os.environ.update(RANK=str(rank), WORLD_SIZE=str(world), LOCAL_RANK=str(rank), MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    sys.path.insert(0, REPO)
    import torch.distributed as dist
    from ml_cvnets_b200 import dist as D
    import ml_cvnets_b200 as m
    r, w, lr = D.init("gloo")
    assert (r, w) == (rank, world)
    # max-over-ranks timing and the weak-scaling aggregate
    mx = D.max_over_ranks(10.0 + rank)
    thr = D.weak_scaling_throughput(128, w, mx)
    # gradient all-reduce semantics on the real parameter set (fp32 grads, SUM / world)
    torch.manual_seed(D.shard_seed(0, rank))
    model = m.MobileViTv2(m.default_opts(width_multiplier=0.5))
    ddp = D.wrap_ddp(model, lr, device_type="cpu")  # constructor broadcasts rank 0's parameters
    p0 = next(model.parameters()).detach().clone()
    grads = [torch.full_like(p, float(rank + 1)) for p in list(model.parameters())[:10]]
    D.allreduce_mean_(grads, w)
    ok_grad = all(torch.allclose(g, torch.full_like(g, (1 + world) / 2.0)) for g in grads)
    gathered = [torch.zeros_like(p0) for _ in range(w)]
    dist.all_gather(gathered, p0)
    ok_bcast = all(torch.equal(gathered[0], t) for t in gathered)
    q.put((rank, mx, thr, ok_grad, ok_bcast, D.shard_seed(0, rank)))
    dist.destroy_process_group()


def test_gloo_world_size_2():
    import torch.multiprocessing as mp
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 29533 + os.getpid() % 200
    procs = [ctx.Process(target=_gloo_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = sorted(q.get(timeout=240) for _ in procs)
    for p in procs:
        p.join(timeout=60)
        assert p.exitcode == 0
    for rank, mx, thr, ok_grad, ok_bcast, seed in res:
        assert mx == 11.0 and abs(thr - 2 * 128 / 11e-3) < 1e-6 and ok_grad and ok_bcast
    assert res[0][5] != res[1][5]

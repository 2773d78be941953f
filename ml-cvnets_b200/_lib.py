"""ctypes binding of libcvnets_b200.so (the C ABI in include/cvnets_b200.h).

The product path has NO fallback: if the library is missing or was not built for this GPU, importing
``ml_cvnets_b200.ops`` on a CUDA box raises.  ``load()`` never builds silently on the GPU box -- the ``.so``
is built in-tree by ``__graft_entry__.build()`` / ``csrc/build.py`` and travels with the snapshot.
"""
from __future__ import annotations

import ctypes
import os
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
# CVB_LIB: diagnostics only (A/B of two kernel builds on the same GPU box, tools/build_variant.sh); the product loads the in-tree library
LIB_PATH = os.environ.get("CVB_LIB") or os.path.join(_HERE, "csrc", "libcvnets_b200.so")
ABI_VERSION = 11

# load modes / epilogue modes (mirror include/cvnets_b200.h)
A_RAW, A_AFF, A_AFF_SILU, A_SILU, A_GN, A_BNB = 0, 1, 2, 3, 4, 5
E_STORE, E_SILU, E_SILU_BWD, E_GN_BWD, E_LIN_BWD = 0, 1, 2, 3, 4


class GemmArgs(Structure):
    _fields_ = [
        ("M", c_int), ("N", c_int), ("K", c_int),
        ("A", c_void_p), ("lda", c_int),
        ("A2", c_void_p), ("lda2", c_int),
        ("a_mode", c_int),
        ("a_p0", c_void_p), ("a_p1", c_void_p), ("a_p2", c_void_p),
        ("row_mean", c_void_p), ("row_rstd", c_void_p),
        ("rows_per_sample", c_int),
        ("W", c_void_p), ("ldw", c_int),
        ("bias", c_void_p),
        ("e_mode", c_int),
        ("Y", c_void_p), ("ldy", c_int),
        ("e_p0", c_void_p), ("e_p1", c_void_p),
        ("R", c_void_p), ("ldr", c_int),
        ("C", c_void_p), ("ldc", c_int), ("c_fp32", c_int),
        ("col_sum", c_void_p), ("col_sq", c_void_p),
        ("samp_sum", c_void_p), ("samp_sq", c_void_p),
        ("gn_ws", c_void_p),
    ]


class WgradArgs(Structure):
    _fields_ = [
        ("M", c_int), ("N", c_int), ("K", c_int),
        ("G", c_void_p), ("ldg", c_int), ("G2", c_void_p), ("ldg2", c_int), ("g_mode", c_int),
        ("g_p0", c_void_p), ("g_p1", c_void_p), ("g_p2", c_void_p),
        ("A", c_void_p), ("lda", c_int), ("a_mode", c_int),
        ("a_p0", c_void_p), ("a_p1", c_void_p),
        ("row_mean", c_void_p), ("row_rstd", c_void_p), ("rows_per_sample", c_int),
        ("dW", c_void_p), ("lddw", c_int),
        ("dbias", c_void_p),
    ]


class DwFwdArgs(Structure):
    _fields_ = [
        ("B", c_int), ("H", c_int), ("W", c_int), ("C", c_int), ("stride", c_int),
        ("X", c_void_p), ("x_mode", c_int), ("x_p0", c_void_p), ("x_p1", c_void_p),
        ("Wt", c_void_p), ("Y", c_void_p), ("col_sum", c_void_p), ("col_sq", c_void_p), ("dilation", c_int), ("ksize", c_int),
    ]


class DwBwdArgs(Structure):
    _fields_ = [
        ("B", c_int), ("H", c_int), ("W", c_int), ("C", c_int), ("stride", c_int),
        ("DZ", c_void_p), ("Y2", c_void_p), ("g_mode", c_int), ("g_p0", c_void_p), ("g_p1", c_void_p), ("g_p2", c_void_p),
        ("X", c_void_p), ("x_mode", c_int), ("x_p0", c_void_p), ("x_p1", c_void_p),
        ("Wt", c_void_p), ("DX", c_void_p), ("col_sum", c_void_p), ("col_sq", c_void_p), ("dWt", c_void_p), ("dilation", c_int),
        ("ksize", c_int),
    ]


class PrepDesc(Structure):
    _fields_ = [("src", c_void_p), ("dst", c_void_p), ("rows", c_int), ("cols", c_int), ("ldd", c_int),
                ("dst_rows", c_int), ("kind", c_int), ("rot", c_int)]


class CastDesc(Structure):
    _fields_ = [("src", c_void_p), ("dst", c_void_p), ("n", c_int), ("pad", c_int)]


_SIGS = {
    "cvb_last_error": (c_char_p, []),
    "cvb_abi_version": (c_int, []),
    "cvb_device_info": (c_int, [POINTER(c_int), POINTER(c_int), POINTER(c_int)]),
    "cvb_pw_gemm": (c_int, [POINTER(GemmArgs), c_void_p]),
    "cvb_set_tc_enabled": (c_int, [c_int]),
    "cvb_set_pdl_enabled": (c_int, [c_int]),
    "cvb_set_mha_impl": (c_int, [c_int]),
    "cvb_rng_next": (c_int, [c_void_p, c_void_p, c_void_p]),
    "cvb_dropout_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "cvb_dropout_bwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_int, c_float, c_float, c_void_p, c_void_p]),
    "cvb_se_scale_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "cvb_se_scale_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "cvb_pw_wgrad": (c_int, [POINTER(WgradArgs), c_void_p]),
    "cvb_apply_load_mode": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p,
                                    c_int, c_int64, c_int, c_void_p]),
    "cvb_dw_fwd": (c_int, [POINTER(DwFwdArgs), c_void_p]),
    "cvb_dw_bwd": (c_int, [POINTER(DwBwdArgs), c_void_p]),
    "cvb_stem_im2col": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_int, c_int, c_void_p, c_void_p]),
    "cvb_bn_finalize": (c_int, [c_void_p, c_void_p, c_double, c_void_p, c_void_p, c_float, c_float, c_void_p, c_void_p, c_void_p,
                                c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "cvb_bn_eval_scale_shift": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p]),
    "cvb_bn_bwd_finalize": (c_int, [c_void_p, c_void_p, c_double, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p,
                                    c_void_p, c_void_p, c_int, c_void_p]),
    "cvb_bn_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "cvb_bn_bwd_reduce": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "cvb_gn_finalize": (c_int, [c_void_p, c_void_p, c_double, c_float, c_void_p, c_void_p, c_int, c_void_p]),
    "cvb_gn_stats": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "cvb_gn_bwd_apply": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_double, c_void_p, c_void_p, c_int, c_int,
                                 c_int, c_void_p, c_void_p]),
    "cvb_gn_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_double, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p,
                           c_void_p, c_void_p]),
    "cvb_linattn_cross_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p,
                                      c_void_p]),
    "cvb_linattn_cross_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                      c_void_p, c_void_p, c_void_p, c_void_p]),
    "cvb_linattn_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "cvb_linattn_bwd": (c_int, [c_void_p, c_int, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p,
                                c_void_p, c_void_p]),
    "cvb_mha_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "cvb_mha_bwd": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_int, c_float, c_void_p, c_void_p,
                            c_void_p, c_int, c_void_p]),
    "cvb_ln_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p, c_void_p, c_void_p,
                           c_void_p]),
    "cvb_act_fwd": (c_int, [c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "cvb_act_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_int, c_void_p]),
    "cvb_ln_stats": (c_int, [c_void_p, c_int, c_int64, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "cvb_grad_norm_blocks": (c_int, [c_int64]),
    "cvb_grad_norm": (c_int, [c_void_p, c_int64, c_void_p, c_float, c_void_p, c_void_p, c_void_p]),
    "cvb_adamw_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_float, c_float, c_float, c_float, c_void_p,
                               c_void_p, c_void_p, c_float, c_float, c_int, c_void_p, c_float, c_void_p, c_void_p]),
    "cvb_sgd_step": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int64, c_void_p, c_float, c_int, c_float, c_void_p, c_void_p, c_void_p,
                             c_float, c_float, c_int, c_void_p, c_float, c_void_p, c_void_p]),
    "cvb_ce_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "cvb_ce_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int,
                           c_void_p, c_void_p, c_void_p, c_void_p]),
    "cvb_embedding_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "cvb_embedding_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "cvb_eot_gather_fwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "cvb_eot_gather_bwd": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "cvb_l2norm_fwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_float, c_void_p]),
    "cvb_l2norm_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "cvb_transpose_bf16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p]),
    "cvb_add_bf16_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_int64, c_void_p]),
    "cvb_zs_class_embed": (c_int, [c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "cvb_zs_logits_topk": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p, c_void_p]),
    "cvb_stem_im2col_mix": (c_int, [c_void_p, c_int64, c_int64, c_int64, c_int64, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "cvb_im2col": (c_int, [c_void_p, c_int, c_int64, c_int64, c_int64, c_int64, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int,
                           c_void_p]),
    "cvb_col2im": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "cvb_patch_permute": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
    "cvb_concat2": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int64, c_void_p, c_void_p]),
    "cvb_split2": (c_int, [c_void_p, c_int, c_int, c_int64, c_void_p, c_void_p, c_void_p]),
    "cvb_vit_tokens_interp_fwd": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "cvb_vit_tokens_interp_bwd": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_int, c_int, c_int, c_void_p]),
    "cvb_cast_f64_f32": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "cvb_memset_zero": (c_int, [c_void_p, c_int64, c_void_p]),
    "cvb_global_pool_fwd": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "cvb_global_pool_bwd": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "cvb_col_sum": (c_int, [c_void_p, c_int, c_int, c_int64, c_int, c_void_p, c_void_p]),
    "cvb_prep_weights": (c_int, [c_void_p, c_int, c_int, c_void_p]),
    "cvb_unprep_grad": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p]),
}

EXPORTS = tuple(_SIGS.keys())
_lib = None


class CvbError(RuntimeError):
    pass


def load(path: str = LIB_PATH):
    """dlopen the kernel library and attach argument types.  Raises if it is missing or has the wrong ABI."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise CvbError(
            f"{path} not found: build it with `python ml-cvnets_b200/csrc/build.py` (or __graft_entry__.build()). "
            "ml-cvnets_b200 has no CPU / PyTorch fallback by design.")
    lib = ctypes.CDLL(path)
    for name, (res, args) in _SIGS.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
    if lib.cvb_abi_version() != ABI_VERSION:
        raise CvbError(f"ABI mismatch: library {lib.cvb_abi_version()} vs python {ABI_VERSION}; rebuild the library")
    _lib = lib
    return lib


def check(rc: int, what: str):
    if rc != 0:
        msg = _lib.cvb_last_error().decode("utf-8", "replace") if _lib is not None else "?"
        raise CvbError(f"{what} failed (rc={rc}): {msg}")

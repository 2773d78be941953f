"""ctypes binding of libcvnets_b200.so, derived from the C ABI in include/cvnets_b200.h.

The header is parsed at import: every ``typedef struct`` becomes a ``ctypes.Structure`` of the same name, every ``CVB_*`` enum value and
``CVB_ABI_VERSION`` a module constant without the prefix (``A_BNB``, ``ACT_GELU``, ``PREP_PATCH``, ``ABI_VERSION``), and ``load()`` attaches
each ``CVB_API`` prototype's restype / argtypes.  Entry points that return a status raise ``CvbError`` with ``cvb_last_error()`` on failure.

The product path has NO fallback: if the library is missing or was not built for this GPU, importing
``ml_cvnets_b200.ops`` on a CUDA box raises.  ``load()`` never builds silently on the GPU box -- the ``.so``
is built in-tree by ``__graft_entry__.build()`` / ``csrc/build.py`` and travels with the snapshot.
"""
from __future__ import annotations

import ctypes
import os
import re
from ctypes import POINTER, Structure, c_char_p, c_double, c_float, c_int, c_int64, c_void_p

_HERE = os.path.dirname(os.path.abspath(__file__))
HEADER = os.path.join(os.path.dirname(_HERE), "include", "cvnets_b200.h")
# CVB_LIB: diagnostics only (A/B of two kernel builds on the same GPU box, tools/build_variant.sh); the product loads the in-tree library
LIB_PATH = os.environ.get("CVB_LIB") or os.path.join(_HERE, "csrc", "libcvnets_b200.so")

# the entry points whose return value is not a status (no CvbError on non-zero)
_NOT_STATUS = ("cvb_last_error", "cvb_abi_version", "cvb_grad_norm_blocks", "cvb_set_tc_enabled", "cvb_set_pdl_enabled", "cvb_set_mha_impl")
_SCALARS = {"int": c_int, "int64_t": c_int64, "float": c_float, "double": c_double, "cvb_stream_t": c_void_p}

# one top-level item of the comment-free header per match; anything else is an error
_ITEM = re.compile(r"""\s*(?:
    \#define[^\S\n]+CVB_(?P<define>\w+)[^\S\n]+(?P<value>\d+)[^\S\n]*\n
  | \#(?!define[^\S\n]+CVB_(?!API\b))[^\n]*\n | extern\s+"C"\s*\{ | \}
  | typedef\s+void\s*\*\s*cvb_stream_t\s*;
  | enum\s*\{(?P<enum>[^}]*)\}\s*;
  | typedef\s+struct\s*\{(?P<struct>[^}]*)\}\s*(?P<struct_name>\w+)\s*;
  | CVB_API\s+(?P<proto>[^;(]*)\((?P<params>[^)]*)\)\s*;
)""", re.X)


class CvbError(RuntimeError):
    pass


def _parse_error(what: str, text: str):
    return CvbError(f"{HEADER}: unrecognised {what}: {' '.join(text.split())[:120]!r}")


def _ctype(base: str, stars: int, name: str, structs: dict, decl: str):
    if base not in _SCALARS and base not in structs and base not in ("void", "char", "unsigned char"):
        raise _parse_error("type", decl)
    if stars == 0 and base in _SCALARS:
        return _SCALARS[base]
    if stars == 1:
        # a struct pointer is a host argument block passed by reference, except `*_device`: a descriptor table in device memory (an address)
        if base in structs and not name.endswith("_device"):
            return POINTER(structs[base])
        return c_char_p if base == "char" else c_void_p
    if stars == 2:  # T* const*: a host array of device pointers
        return POINTER(c_void_p)
    raise _parse_error("type", decl)


def _declare(decl: str, structs: dict):
    """``const float* a, b`` -> [("a", c_void_p), ("b", c_float)]: one base type, comma-separated declarators."""
    m = re.fullmatch(r"\s*(?:const\s+)?(unsigned\s+char|\w+)(.*)", decl, re.S)
    out = []
    for d in (m.group(2).split(",") if m else [""]):
        dm = re.fullmatch(r"\s*((?:\*\s*(?:const\b\s*)?)*)(\w+)\s*", d)
        if not dm:
            raise _parse_error("declaration", decl)
        out.append((dm.group(2), _ctype(" ".join(m.group(1).split()), dm.group(1).count("*"), dm.group(2), structs, decl)))
    return out


def _parse(path: str):
    with open(path) as f:
        text = re.sub(r"/\*.*?\*/|//[^\n]*", " ", f.read(), flags=re.S).strip() + "\n"
    consts, structs, protos = {}, {}, {}
    pos = 0
    while text[pos:].strip():
        m = _ITEM.match(text, pos)
        if not m:
            raise _parse_error("declaration", text[pos:])
        pos = m.end()
        if m["define"]:
            consts[m["define"]] = int(m["value"])
        elif m["enum"] is not None:
            value = -1
            for item in filter(str.strip, m["enum"].split(",")):
                em = re.fullmatch(r"\s*CVB_(\w+)\s*(?:=\s*(\d+)\s*)?", item)
                if not em:
                    raise _parse_error("enumerator", item)
                value = int(em[2]) if em[2] else value + 1
                consts[em[1]] = value
        elif m["struct"] is not None:
            fields = [f for decl in m["struct"].split(";") if decl.strip() for f in _declare(decl, structs)]
            structs[m["struct_name"]] = type(m["struct_name"], (Structure,), {"_fields_": fields})
        elif m["proto"] is not None:
            [(name, restype)] = _declare(m["proto"], structs)
            params = [] if m["params"].strip() == "void" else m["params"].split(",")
            protos[name] = (restype, [t for p in params for _, t in _declare(p, structs)])
    return consts, structs, protos


_consts, _structs, _PROTOTYPES = _parse(HEADER)
globals().update(_consts)
globals().update(_structs)
EXPORTS = tuple(_PROTOTYPES)
_lib = None


def load(path: str = LIB_PATH):
    """dlopen the kernel library and attach argument types.  Raises if it is missing or has the wrong ABI."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(path):
        raise CvbError(
            f"{path} not found: build it with `python ml-cvnets_b200/csrc/build.py` (or __graft_entry__.build()). "
            "ml-cvnets_b200 has no CPU / PyTorch fallback by design.")
    undeclared = sorted(set(_NOT_STATUS) - set(_PROTOTYPES))
    if undeclared:
        raise CvbError(f"{HEADER} does not declare {undeclared}")
    lib = ctypes.CDLL(path)

    def errcheck(rc, fn, args):
        if rc != 0:
            raise CvbError(f"{fn.__name__} failed (rc={rc}): {lib.cvb_last_error().decode('utf-8', 'replace')}")
        return rc

    for name, (res, args) in _PROTOTYPES.items():
        fn = getattr(lib, name)  # AttributeError if a declared symbol is not exported
        fn.restype = res
        fn.argtypes = args
        if name not in _NOT_STATUS:
            fn.errcheck = errcheck
    if lib.cvb_abi_version() != _consts["ABI_VERSION"]:
        raise CvbError(f"ABI mismatch: library {lib.cvb_abi_version()} vs header {_consts['ABI_VERSION']}; rebuild the library")
    _lib = lib
    return lib

"""CPU-only guard: every kernel entry point the C ABI exports is exercised by at least one GPU test.

An export counts as tested when a ``tests/test_*_gpu.py`` file names it (``cvb_xxx``, e.g. through ``lib.cvb_xxx``) or calls one of the
``ops.py`` wrappers that launch it (``ops.<wrapper>``).  Host-only entry points that launch no kernel are exempt, each for a stated reason."""
import ast
import glob
import os
import re

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# entry points that launch no kernel of their own: nothing for a kernel-level test to compare against a reference
EXEMPT = {
    "cvb_abi_version": "returns a compile-time constant; test_host_cpu.py checks it against the Python binding",
    "cvb_last_error": "host-side error string, read by ops.check on every failing call",
    "cvb_device_info": "host-side device attribute query",
    "cvb_set_pdl_enabled": "host-side launch-attribute switch; every GPU test runs with its default",
    "cvb_grad_norm_blocks": "host-side scratch-size query for cvb_grad_norm",
    "cvb_memset_zero": "a cudaMemsetAsync, no kernel",
}


def _exports():
    hdr = open(os.path.join(REPO, "include", "cvnets_b200.h")).read()
    return sorted(set(re.findall(r"CVB_API\s+(?:const\s+char\*|int)\s+(cvb_[a-z0-9_]+)\s*\(", hdr)))


def _ops_wrappers():
    """export -> names under which tests reach it through ops.py: module-level functions, and classes for methods."""
    src = open(os.path.join(REPO, "ml-cvnets_b200", "ops.py")).read()
    found = {}

    def visit(node, name):
        for sub in ast.walk(node):
            if isinstance(sub, ast.Attribute) and sub.attr.startswith("cvb_"):
                found.setdefault(sub.attr, set()).add(name)

    for node in ast.parse(src).body:
        if isinstance(node, (ast.FunctionDef, ast.ClassDef)):
            visit(node, node.name)
    return found


def _gpu_test_sources():
    files = sorted(glob.glob(os.path.join(REPO, "tests", "test_*_gpu.py")))
    assert files
    return "\n".join(open(f).read() for f in files)


def test_exemptions_are_real_exports():
    exports = set(_exports())
    assert set(EXEMPT) <= exports, set(EXEMPT) - exports
    assert all(reason.strip() for reason in EXEMPT.values())


def test_nondeterministic_list_names_only_real_exports():
    """test_reproducible_gpu.py leaves the entry points in its NONDETERMINISTIC dict out of the bitwise checks: each must be an export, with a reason"""
    tree = ast.parse(open(os.path.join(REPO, "tests", "test_reproducible_gpu.py")).read())
    found = [ast.literal_eval(n.value) for n in tree.body
             if isinstance(n, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "NONDETERMINISTIC" for t in n.targets)]
    assert len(found) == 1 and found[0]
    exempt = found[0]
    assert set(exempt) <= set(_exports()), set(exempt) - set(_exports())
    assert all(reason.strip() for reason in exempt.values())


def test_ops_wrappers_call_real_exports():
    exports = set(_exports())
    unknown = set(_ops_wrappers()) - exports
    assert not unknown, f"ops.py calls symbols the header does not declare: {sorted(unknown)}"


def test_every_kernel_export_is_called_by_a_gpu_test():
    exports = _exports()
    assert len(exports) >= 60
    wrappers = _ops_wrappers()
    text = _gpu_test_sources()
    missing = []
    for name in exports:
        if name in EXEMPT:
            continue
        if re.search(r"\b%s\b" % name, text):
            continue
        via = sorted(wrappers.get(name, ()))
        if any(re.search(r"\bops\.%s\b" % w, text) for w in via):
            continue
        missing.append(f"{name} (ops wrappers: {', '.join(via) or 'none'})")
    assert not missing, "exports no GPU test calls:\n  " + "\n  ".join(missing)

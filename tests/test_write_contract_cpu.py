"""CPU-only guard of the write-set contract table, and the negative controls of the guard-banded buffer helper.

Every export of include/cvnets_b200.h that launches a kernel has a row in CONTRACT (tests/test_write_contract_gpu.py, read with ast, not
imported) naming its written, accumulated and partially written outputs and the GPU test that checks them.  The host-only exports are
test_kernel_coverage_cpu.py's EXEMPT set and the cvb_set_* testing hooks.  The helper's checks must fail on a corrupted guard element, a
corrupted gap element and a region element left at the sentinel, or a passing GPU test would mean nothing."""
import ast
import os

import pytest
import torch

from test_kernel_coverage_cpu import EXEMPT, _exports
from write_guard import Guarded, bits, sentinel_bits

REPO = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GPU_FILE = os.path.join(REPO, "tests", "test_write_contract_gpu.py")


def _gpu_module():
    return ast.parse(open(GPU_FILE).read())


def _contract():
    found = [ast.literal_eval(n.value) for n in _gpu_module().body
             if isinstance(n, ast.Assign) and any(isinstance(t, ast.Name) and t.id == "CONTRACT" for t in n.targets)]
    assert len(found) == 1
    return found[0]


def _host_only(name):
    return name in EXEMPT or name.startswith("cvb_set_")


def test_contract_covers_every_kernel_export():
    table = _contract()
    missing = [e for e in _exports() if not _host_only(e) and e not in table]
    assert not missing, f"exports without a write-set row: {missing}"
    extra = set(table) - set(_exports())
    assert not extra, f"rows for names the header does not export: {sorted(extra)}"
    host = [e for e in table if _host_only(e)]
    assert not host, f"rows for host-only exports: {host}"


def test_contract_rows_are_well_formed():
    tests = {n.name for n in _gpu_module().body if isinstance(n, ast.FunctionDef) and n.name.startswith("test_")}
    for name, row in _contract().items():
        assert set(row) == {"written", "accumulated", "partial", "test"}, name
        outs = row["written"] + row["accumulated"] + row["partial"]
        assert outs, f"{name}: names no output"
        assert len(outs) == len(set(outs)), f"{name}: an output is listed twice"
        assert row["test"] in tests, f"{name}: {row['test']} is not a test of {os.path.basename(GPU_FILE)}"


# ------------------------------------------------------------------------------------------- negative controls of the helper
DTYPES = [torch.float32, torch.bfloat16, torch.float64, torch.int64, torch.int32]


def _written(dtype, shape=(5, 12), ld=16):
    g = Guarded(shape, dtype, device="cpu", ld=ld if len(shape) == 2 else None, guard_rows=2, min_guard=64)
    g.fill(torch.arange(g.view.numel()).reshape(g.view.shape) % 7 + 1)
    return g


@pytest.mark.parametrize("dtype", DTYPES)
def test_sentinel_is_a_fixed_pattern(dtype):
    g = Guarded((3, 8), dtype, device="cpu", ld=16, guard_rows=1, min_guard=16)
    assert bool((bits(g.buf) == sentinel_bits(dtype)).all())
    if dtype.is_floating_point:
        assert bool(g.buf.float().isnan().all()), "the fp32 / bf16 / fp64 sentinels are NaNs"
    assert g.front * g.buf.element_size() % 128 == 0, "the region keeps 128-byte alignment"
    assert g.front >= 16 and g.back >= 16 and g.ld == 16


@pytest.mark.parametrize("dtype", DTYPES)
def test_clean_buffer_passes(dtype):
    g = _written(dtype)
    g.check("clean")
    v = _written(dtype, shape=(37,))
    v.check("clean vector")


@pytest.mark.parametrize("dtype", DTYPES)
@pytest.mark.parametrize("where", ["front", "back", "gap"])
def test_one_corrupted_band_element_fails(dtype, where):
    g = _written(dtype)
    if where == "front":
        g.buf[g.front - 1] = 0
    elif where == "back":
        g.buf[g.front + g.rows * g.ld] = 0
    else:
        g.padded[2, g.width] = 0  # the first gap element after row 2: a write one column past N
    with pytest.raises(AssertionError, match="overwritten"):
        g.check_bands(where)


@pytest.mark.parametrize("dtype", DTYPES)
def test_far_guard_element_fails(dtype):
    g = _written(dtype, shape=(40,))
    g.buf[-1] = 3
    with pytest.raises(AssertionError, match="back guard"):
        g.check_bands("last element")


@pytest.mark.parametrize("dtype", DTYPES)
def test_unwritten_region_element_fails(dtype):
    g = _written(dtype)
    bits(g.view)[3, 11] = sentinel_bits(dtype)
    with pytest.raises(AssertionError, match="never written"):
        g.check_written("skipped store")
    g.check_bands("bands are fine")


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16, torch.float64])
def test_accumulated_into_written_output_fails(dtype):
    """sentinel + value on the device gives the canonical NaN, not the sentinel's bits: a written output must also be finite"""
    g = _written(dtype)
    g.view[1, 4] = float("nan")
    assert int(bits(g.view[1:2, 4:5].contiguous())) != sentinel_bits(dtype)
    with pytest.raises(AssertionError, match="not finite"):
        g.check_written("+= instead of =")
    g.view[1, 4] = float("inf")
    with pytest.raises(AssertionError, match="not finite"):
        g.check_written("inf")


def test_untouched_columns_check():
    g = Guarded((4, 24), torch.bfloat16, device="cpu", guard_rows=1, min_guard=16)
    g.view[:, :8] = 1.0
    g.check_written("written columns", slice(0, 8))
    g.check_untouched("untouched columns", slice(8, 24))
    g.view[1, 9] = 0.0
    with pytest.raises(AssertionError, match="must leave alone"):
        g.check_untouched("one stray store", slice(8, 24))


def test_prior_fill_keeps_bands():
    g = Guarded((6,), torch.float64, device="cpu", min_guard=8)
    g.fill(torch.tensor([1.0, -2.0, 3.0, 0.5, 7.0, -1.0]))
    g.check("prior")
    assert g.region().tolist() == [1.0, -2.0, 3.0, 0.5, 7.0, -1.0]

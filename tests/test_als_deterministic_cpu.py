"""Deterministic ALS without a GPU: the option key is accepted by ALSOption and by the backend's option parsing (which
comes before the device check), the C ABI gained no symbol for it, and the benchmark's split-row model."""
import os
import re
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_option_class_accepts_the_key_and_defaults_do_not_list_it():
    import buffalo
    opt = buffalo.ALSOption().get_default_option()
    assert "deterministic" not in opt
    opt.update(deterministic=True, _b200_det_scratch_mb=64)
    assert buffalo.ALSOption().is_valid_option(opt)


@pytest.mark.parametrize("optimizer", ["llt", "ldlt", "manual_cg", "ialspp"])
@pytest.mark.parametrize("d", [20, 64, 128, 256])
def test_backend_accepts_the_key_up_to_the_device_check(optimizer, d):
    import torch
    from buffalo_b200 import _cabi, backend
    g = backend.CuALS()
    opt = dict(d=d, optimizer=optimizer, deterministic=True)
    if torch.cuda.is_available():
        assert g.init(opt) is True
        return
    with pytest.raises(_cabi.BackendError) as e:
        g.init(opt)
    assert "no CPU fallback" in str(e.value)


def test_negative_scratch_budget_is_an_option_error():
    from buffalo_b200 import backend
    g = backend.CuALS()
    assert g.init(dict(d=128, deterministic=True, _b200_det_scratch_mb=-1)) is False
    assert "_b200_det_scratch_mb" in g.last_error


def test_no_new_abi_symbol():
    """The option travels in the JSON: header and ctypes table list the same bfl_als_* entry points as before."""
    from buffalo_b200 import _cabi
    header = open(os.path.join(ROOT, "include", "buffalo_b200.h")).read()
    in_header = set(re.findall(r"\b(bfl_als_\w+)\s*\(", header))
    lib = _cabi.lib()
    for name in in_header:
        assert hasattr(lib, name), name
    assert not [n for n in in_header if "determin" in n]
    src = open(os.path.join(ROOT, "buffalo_b200", "_cabi.py")).read()
    assert set(re.findall(r"\b(bfl_als_\w+)\b", src)) <= in_header | {"bfl_als_t"}


def test_memory_estimate_of_the_trainer():
    from buffalo_b200.algo.als import ALS
    assert ALS.deterministic_bytes(1000, 10, 64) == 16 * 1000 + (64 << 20)
    assert ALS.deterministic_bytes(10, 1000) == 16 * 1000 + (2 << 30)
    assert ALS.deterministic_bytes(10, 10, 0.5) == 160 + (1 << 19)


def test_benchmark_split_row_model():
    sys.path.insert(0, os.path.join(ROOT, "benchmarks"))
    import als_deterministic_bench as b
    sb = b.slot_bytes(128)
    assert sb == 4 * (128 * 128 + 2 * 128 + 4)
    # rows: 1536 (not split), 1537 (1 chunk), 2049 (2), 9000 (5), 40000 (20)
    m = b.split_model([0, 1, 1536, 1537, 2049, 9000, 40000], 128, budget_bytes=1 << 40)
    assert (m["split_rows"], m["chunks"], m["batches"]) == (4, 28, 1)
    assert m["peak_scratch_bytes"] == (28 + 4) * sb and m["default_scratch_bytes"] == 4 * sb
    assert m["default_bytes"] == (4 + 2 * 28 + 3 * 4) * sb and m["deterministic_bytes"] == (28 + 28 + 4 + 3 * 4) * sb
    # a budget of 9 slots: {1537, 2049} (2 + 3 slots), {9000} (6), {40000} alone although it needs 21
    m = b.split_model([1537, 2049, 9000, 40000], 128, budget_bytes=9 * sb)
    assert m["batches"] == 3 and m["peak_scratch_bytes"] == 21 * sb
    assert b.split_model([5, 100], 256, 1 << 30)["batches"] == 0
    assert b.kernel_class("void bfl::tc::als_tc_kernel<128, true, false, true>(bfl::tc::TcArgs)") == "partial"
    assert b.kernel_class("void bfl::tc::als_tc_kernel<(int)128, (bool)0, (bool)1, (bool)0>(bfl::tc::TcArgs)") is None
    assert b.kernel_class("bfl::tc::tc_chunk_reduce_kernel(float const*, ...)") == "chunk_reduce"

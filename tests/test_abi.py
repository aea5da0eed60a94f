"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/buffalo_b200.h declares, and refuses to run without a Hopper (sm_90) GPU (no CPU fallback)."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared():
    text = open(os.path.join(ROOT, "include", "buffalo_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(bfl_[a-z0-9_]+)\s*\(", text)))


def test_header_symbols_exported():
    from buffalo_b200 import _cabi
    handle = ctypes.CDLL(_cabi.LIB_PATH)
    names = _declared()
    assert len(names) >= 40
    for n in names:
        assert hasattr(handle, n), "missing export %s" % n
    assert set(names) == set(_cabi.PROTOTYPES), set(names) ^ set(_cabi.PROTOTYPES)


def test_library_is_sm90_only():
    from buffalo_b200 import _cabi
    lib = _cabi.lib()
    assert lib.bfl_compiled_sm() == 90
    assert lib.bfl_abi_version() == 1


def _holders():
    from buffalo_b200 import backend
    return {"als": backend.CuALS, "bpr": lambda: backend.CuSGD("bpr"), "warp": lambda: backend.CuSGD("warp"),
            "plsi": backend.CuPLSI}


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from buffalo_b200 import _cabi
    for kind, make in _holders().items():
        with pytest.raises(_cabi.BackendError) as e:
            make().init({"d": 16})
        assert "no CPU fallback" in str(e.value), kind


def test_bad_option_file_returns_false_or_raises():
    # reference: init() returns False on a missing option file (lib/algo.cc:22-34) and the Python
    # layer asserts (buffalo/algo/als.py:43)
    for kind, make in _holders().items():
        obj = make()
        assert obj.init(b"/nonexistent/option.json") is False, kind
        assert "File not exists" in obj.last_error, kind


@pytest.mark.parametrize("kind,opt,msg", [
    ("als", {"d": 0}, "d must be in [1, 512], got 0"),
    ("als", {"d": 513}, "d must be in [1, 512], got 513"),
    ("als", {"d": 16, "optimizer": "eigen_cg"}, "optimizer 'eigen_cg' is not available on the H100 backend"),
    ("bpr", {"d": 0}, "d must be in [1, 512]"),
    ("warp", {"d": 600}, "d must be in [1, 512]"),
    ("warp", {"d": 16, "optimizer": "sgd"}, "optimizer must be adagrad or adam"),
    ("plsi", {"d": 0}, "d must be in [1, 512]"),
])
def test_option_errors_return_false_before_device_check(kind, opt, msg):
    # option errors come before the device check: they return False with or without a GPU
    obj = _holders()[kind]()
    assert obj.init(opt) is False
    assert msg in obj.last_error


def test_product_never_imports_oracle():
    bad = []
    for pkg in ("buffalo_b200", "buffalo"):
        base = os.path.join(ROOT, pkg)
        for dp, _, fs in os.walk(base):
            for f in fs:
                if f.endswith((".py", ".cu", ".cuh", ".h", ".sh")):
                    src = open(os.path.join(dp, f)).read()
                    if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M) or "libbuffalo_oracle" in src:
                        bad.append(os.path.join(dp, f))
    assert not bad, bad

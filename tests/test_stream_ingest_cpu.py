"""Stream device-ingest routing and constants that need no GPU (data/stream.py)."""
import numpy as np
import pytest

from buffalo import Stream, StreamOptions
from buffalo_b200.data import stream as smod


def test_whitespace_constant_is_pythons():
    assert list(smod.WHITESPACE) == [c for c in range(0x110000) if chr(c).isspace()]


def _opt(tmp_path, text):
    (tmp_path / "main").write_text(text)
    opt = StreamOptions().get_default_option()
    opt.input.main = str(tmp_path / "main")
    opt.data.path = str(tmp_path / "s.h5py")
    opt.data.tmp_dir = str(tmp_path)
    return opt


def _forbid_device(monkeypatch):
    def boom(*a, **k):
        raise AssertionError("the device path must not run")
    monkeypatch.setattr(smod, "_device_ingest", boom)


def test_small_file_stays_on_host(tmp_path, monkeypatch):
    _forbid_device(monkeypatch)
    st = Stream(_opt(tmp_path, "a b c\nb c\n"))
    st.create()
    assert not hasattr(st, "ingest_stats")
    assert st.get_header()["num_items"] == 3


def test_no_device_stays_on_host(tmp_path, monkeypatch):
    from buffalo_b200 import backend
    _forbid_device(monkeypatch)
    monkeypatch.setattr(smod, "DEVICE_INGEST_MIN_BYTES", 0)
    monkeypatch.setattr(backend, "device_available", lambda: False)
    st = Stream(_opt(tmp_path, "a b c\nb c\n"))
    st.create()
    assert not hasattr(st, "ingest_stats")


def test_non_utf8_locale_stays_on_host(tmp_path, monkeypatch):
    from buffalo_b200 import backend
    _forbid_device(monkeypatch)
    monkeypatch.setattr(smod, "DEVICE_INGEST_MIN_BYTES", 0)
    monkeypatch.setattr(backend, "device_available", lambda: True)
    monkeypatch.setattr(smod.locale, "getpreferredencoding", lambda do_setlocale=True: "latin-1")
    Stream(_opt(tmp_path, "a b\n")).create()


def test_sppmi_still_raises_before_device_work(tmp_path, monkeypatch):
    from buffalo_b200 import backend
    _forbid_device(monkeypatch)
    monkeypatch.setattr(smod, "DEVICE_INGEST_MIN_BYTES", 0)
    monkeypatch.setattr(backend, "device_available", lambda: True)
    opt = _opt(tmp_path, "a b\n")
    opt.data.sppmi = {"windows": 5, "k": 10}
    with pytest.raises(NotImplementedError):
        Stream(opt).create()


def test_find_cut():
    buf = np.frombuffer(b"ab c\nde f\ngh", np.uint8)
    assert smod._find_cut(buf, len(buf), 16) == 10
    with pytest.raises(smod._Fallback):
        smod._find_cut(np.frombuffer(b"abcdef", np.uint8), 6, 6)

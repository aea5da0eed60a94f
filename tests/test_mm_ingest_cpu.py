"""Host side of the device MatrixMarket parser (data/mm.py): routing, header parsing and the host re-parse of the value
tokens the device leaves to it.  No GPU needed (the block/carry protocol is in test_text_ingest_cpu.py)."""
import numpy as np
import pytest

from buffalo_b200.data import mm as mmmod


def _mm(tmp_path, text, name="in.mtx"):
    from buffalo import MatrixMarket, MatrixMarketOptions
    src = tmp_path / name
    src.write_bytes(text.encode() if isinstance(text, str) else text)
    opt = MatrixMarketOptions().get_default_option()
    opt.input.main = str(src)
    opt.data.tmp_dir = str(tmp_path)
    opt.data.path = str(tmp_path / "db.h5py")
    opt.data.validation = {}
    return MatrixMarket(opt)


TEXT = "%%MatrixMarket matrix coordinate integer general\n%\n% c\n4 3 5\n1 1 1\n2 1 3\n3 3 1\n4 2 1\n4 2 2\n"


def _spy(monkeypatch):
    calls = []

    def fake(*args, **kw):
        calls.append(args)
        raise mmmod._Fallback("test")
    monkeypatch.setattr(mmmod, "_device_ingest", fake)
    return calls


@pytest.mark.parametrize("device,min_bytes,routed", [(False, 0, False), (True, 1 << 30, False), (True, 0, True)])
def test_routing(tmp_path, monkeypatch, device, min_bytes, routed):
    from buffalo_b200 import backend
    calls = _spy(monkeypatch)
    monkeypatch.setattr(backend, "device_available", lambda: device)
    monkeypatch.setattr(mmmod, "DEVICE_INGEST_MIN_BYTES", min_bytes)
    db = _mm(tmp_path, TEXT)
    db.create()                                   # a declined device parse falls back to the host path
    assert len(calls) == int(routed)
    assert list(db.get_group("rowwise")["indptr"][:]) == [1, 2, 3, 5]
    assert not hasattr(db, "ingest_stats")


def test_scipy_and_array_inputs_stay_on_host(tmp_path, monkeypatch):
    from buffalo_b200 import backend
    calls = _spy(monkeypatch)
    monkeypatch.setattr(backend, "device_available", lambda: True)
    monkeypatch.setattr(mmmod, "DEVICE_INGEST_MIN_BYTES", 0)
    db = _mm(tmp_path, TEXT)
    db.opt.input.main = np.eye(3, dtype=np.float32)
    db.create()
    assert calls == []


def test_header(tmp_path):
    p = tmp_path / "h.mtx"
    p.write_text(TEXT)
    assert mmmod._read_mm_header(str(p)) == (4, 3, 5, 4)
    assert mmmod._data_offset(str(p), 4) == TEXT.index("1 1 1")
    p.write_bytes(TEXT.replace("\n", "\r\n").encode())
    assert mmmod._read_mm_header(str(p)) == (4, 3, 5, 4)
    assert mmmod._data_offset(str(p), 4) == TEXT.replace("\n", "\r\n").index("1 1 1")
    p.write_bytes(b"%%MatrixMarket matrix coordinate integer general\r% c\n4 3 5\n1 1 1\n")
    assert mmmod._read_mm_header(str(p))[3] == 3
    assert mmmod._data_offset(str(p), 3) is None  # a bare '\r' ends a header line: left to the host path


def test_value_tokens_match_host_reader(tmp_path):
    toks = ["0.12345678901234567", "12345678901234567", "1e-30", "3.4e38", "3.5e38", "1e-40", "1.4e-45", "-0", "nan",
            "NaN", "inf", "-inf", ".5", "5.", "1E+400", "-2e-39", "+7", "0.1", "NA"]
    p = tmp_path / "t.mtx"
    p.write_text("%%%%MatrixMarket matrix coordinate real general\n3 2 %d\n" % len(toks) +
                 "".join("%d %d %s\n" % (i % 3 + 1, i % 2 + 1, t) for i, t in enumerate(toks)))
    want = mmmod._read_mm_text(str(p))[4]
    got = mmmod._parse_value_tokens([t.encode() for t in toks])
    assert got.dtype == np.float32 and got.tobytes() == want.tobytes()
    with pytest.raises(ValueError):
        mmmod._parse_value_tokens([b"1.5x"])

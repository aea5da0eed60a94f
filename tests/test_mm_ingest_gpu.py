"""Device MatrixMarket parser (csrc/mm_ingest.cu, data/mm.py::_device_ingest): every case builds the same text file
through the host path (pandas) and the device path and compares every array and attr of the two databases bitwise.
Files the device grammar rejects must fall back to the host path and still match; out-of-range indices raise."""
import os

import numpy as np
import pytest

from tests.mm_files import write_mm

pytestmark = pytest.mark.gpu

BANNER = "%%MatrixMarket matrix coordinate real general\n"


def _build(tmp_path, name, text, device, monkeypatch, block=None, validation=True, prepro=None, seed=7):
    from buffalo_b200.data import mm as mmmod
    from buffalo import MatrixMarket, MatrixMarketOptions
    src = tmp_path / (name + ".mtx")
    if not src.exists():
        src.write_bytes(text if isinstance(text, bytes) else text.encode())
    monkeypatch.setattr(mmmod, "DEVICE_INGEST_MIN_BYTES", 0 if device else 1 << 62)
    if block:
        monkeypatch.setattr(mmmod, "DEVICE_INGEST_BLOCK_BYTES", block)
    opt = MatrixMarketOptions().get_default_option()
    opt.input.main = str(src)
    opt.data.tmp_dir = str(tmp_path)
    opt.data.path = str(tmp_path / ("%s_%s.h5py" % (name, "dev" if device else "host")))
    if not validation:
        opt.data.validation = {}
    if prepro:
        opt.data.value_prepro = prepro
    np.random.seed(seed)
    db = MatrixMarket(opt)
    db.create()
    return db


def _contents(db):
    h = db.handle
    out = {"attrs": {k: h.attrs[k] for k in ("num_users", "num_items", "num_nnz", "completed")}}
    for g in ("rowwise", "colwise", "vali", "idmap"):
        if g not in h:
            continue
        grp = h[g]
        out[g] = {k: np.asarray(grp[k][:]) for k in grp.keys()}
        if g == "vali":
            out[g]["attrs"] = {k: grp.attrs[k] for k in ("method", "n", "num_samples")}
    return out


def assert_same_db(a, b):
    ca, cb = _contents(a), _contents(b)
    assert ca.keys() == cb.keys()
    assert ca["attrs"] == cb["attrs"]
    for g in ca:
        if g == "attrs":
            continue
        assert ca[g].keys() == cb[g].keys(), g
        for k in ca[g]:
            if k == "attrs":
                assert ca[g][k] == cb[g][k]
                continue
            x, y = ca[g][k], cb[g][k]
            assert x.dtype == y.dtype and x.shape == y.shape, (g, k, x.dtype, y.dtype, x.shape, y.shape)
            assert x.tobytes() == y.tobytes(), (g, k)


def both(tmp_path, name, text, monkeypatch, expect_device=True, **kw):
    host = _build(tmp_path, name, text, False, monkeypatch, **kw)
    dev = _build(tmp_path, name, text, True, monkeypatch, **kw)
    assert hasattr(dev, "ingest_stats") == expect_device, "device path %s" % ("expected" if expect_device else "not expected")
    assert_same_db(host, dev)
    return host, dev


def mm_text(U, I, lines, banner=BANNER, nnz=None, eol="\n", final_eol=True):
    body = eol.join(lines)
    head = banner + "%d %d %d" % (U, I, len(lines) if nnz is None else nnz) + eol
    return head + body + (eol if final_eol and lines else "")


def random_lines(rng, U, I, n, fmt):
    r = rng.integers(1, U + 1, n)
    c = rng.integers(1, I + 1, n)
    return [fmt(a, b, rng) for a, b in zip(r, c)]


# ---- values -------------------------------------------------------------------------------------
FAST_VALUES = ["1", "5", "0", "-0", "+3", "-7", "0.5", "3.25", "-0.125", "+2.5", "1e3", "2.5E-3", "1.5e+10", "-4e-22",
               "123456789012345", "0.000001", "99999.99999", "7e22", "12345.6789e-5", "0000012", "-0.0"]
SLOW_VALUES = ["0.12345678901234567", "12345678901234567", "1e-30", "3.4e38", "3.5e38", "1e-40", "1.4e-45", "1e-46",
               "-2e-39", "nan", "NaN", "inf", "-inf", ".5", "5.", "1e23", "1e-23", "123456789012345678901234567890",
               "0.1234567890123456789e5", "1E+400"]


@pytest.mark.parametrize("values", [FAST_VALUES, SLOW_VALUES, FAST_VALUES + SLOW_VALUES], ids=["fast", "slow", "mixed"])
def test_values_match_host(cuda_lib, tmp_path, monkeypatch, values):
    rng = np.random.default_rng(len(values))
    lines = random_lines(rng, 40, 30, 3000, lambda a, b, r: "%d %d %s" % (a, b, values[r.integers(len(values))]))
    _, dev = both(tmp_path, "v", mm_text(40, 30, lines), monkeypatch)
    if values is FAST_VALUES:
        assert dev.ingest_stats["device_ms"]["patch"] == 0.0           # nothing left to the host parser


def test_random_decimals_match_host(cuda_lib, tmp_path, monkeypatch):
    rng = np.random.default_rng(5)
    toks = []
    for _ in range(40000):
        nd = int(rng.integers(1, 19))
        digs = "".join(rng.choice(list("0123456789"), nd))
        k = int(rng.integers(0, nd + 1))
        t = digs[:k] + ("." + digs[k:] if k < nd else "")
        t = ("0" + t) if t.startswith(".") else t
        if rng.random() < 0.4:
            t += "eE"[int(rng.integers(2))] + str(int(rng.integers(-45, 45)))
        toks.append(("-" if rng.random() < 0.3 else "") + t)
    lines = ["%d %d %s" % (i % 97 + 1, i % 89 + 1, t) for i, t in enumerate(toks)]
    both(tmp_path, "dec", mm_text(97, 89, lines), monkeypatch)


# ---- layout -------------------------------------------------------------------------------------
def test_pattern_file(cuda_lib, tmp_path, monkeypatch):
    rng = np.random.default_rng(1)
    lines = random_lines(rng, 50, 60, 4000, lambda a, b, r: "%d %d" % (a, b))
    both(tmp_path, "pat", mm_text(50, 60, lines, banner="%%MatrixMarket matrix coordinate pattern general\n"), monkeypatch)


@pytest.mark.parametrize("eol,final_eol", [("\n", True), ("\r\n", True), ("\n", False), ("\r\n", False)])
def test_whitespace_comments_and_line_ends(cuda_lib, tmp_path, monkeypatch, eol, final_eol):
    rng = np.random.default_rng(2)
    forms = ["%d %d %s", "%d\t%d\t%s", "  %d   %d \t %s", "\t%d %d %s  ", "%d %d %s %% inline comment", "%d %d %s%%c",
             "%d  %d  %s\t%% tab then comment"]

    def fmt(a, b, r):
        return forms[r.integers(len(forms))] % (a, b, ["1", "2.5", "-3e-2", "4"][r.integers(4)])
    lines = []
    for ln in random_lines(rng, 70, 40, 3000, fmt):
        lines.append(ln)
        x = rng.random()
        if x < 0.05:
            lines.append("% a comment line \"quoted\" and \t tab")
        elif x < 0.08:
            lines.append("")
        elif x < 0.10:
            lines.append(" \t  ")
        elif x < 0.11:
            lines.append("%")
    both(tmp_path, "ws", mm_text(70, 40, lines, eol=eol, final_eol=final_eol, nnz=3000), monkeypatch)


def test_comments_and_blanks_before_data(cuda_lib, tmp_path, monkeypatch):
    text = BANNER + "% one\n%\n% two\n3 4 5\n\n% inside\n\n1 1 1\n2 4 2\n\n3 2 7.5\n1 1 9\n"
    both(tmp_path, "pre", text, monkeypatch)


def test_duplicates_keep_file_order(cuda_lib, tmp_path, monkeypatch):
    rng = np.random.default_rng(3)
    lines = ["%d %d %d" % (rng.integers(1, 4), rng.integers(1, 3), i) for i in range(5000)]
    host, dev = both(tmp_path, "dup", mm_text(3, 2, lines), monkeypatch, validation=False)
    # within one (row, col) run the values are the running line numbers: file order
    ind, key, val = (np.asarray(dev.handle["rowwise"][k][:]) for k in ("indptr", "key", "val"))
    beg = 0
    for end in ind:
        k, v = key[beg:end], val[beg:end]
        for c in np.unique(k):
            assert np.all(np.diff(v[k == c]) > 0)
        beg = end


def test_empty_rows_and_columns(cuda_lib, tmp_path, monkeypatch):
    rng = np.random.default_rng(4)
    lines = ["%d %d %d" % (3 * rng.integers(1, 300), 7 * rng.integers(1, 100), rng.integers(1, 6)) for _ in range(8000)]
    both(tmp_path, "holes", mm_text(1000, 800, lines), monkeypatch)


def test_single_entry(cuda_lib, tmp_path, monkeypatch):
    both(tmp_path, "one", mm_text(5, 3, ["2 3 4.5"]), monkeypatch)


def test_nnz_zero_header(cuda_lib, tmp_path, monkeypatch):
    both(tmp_path, "zero", mm_text(5, 3, []), monkeypatch, expect_device=False)


# ---- block and tile boundaries ----------------------------------------------------------------------
@pytest.mark.parametrize("block", [256, 333, 3 * 4096 + 100])
def test_block_and_tile_boundaries(cuda_lib, tmp_path, monkeypatch, block):
    """Line lengths cycle through 29 values, so the blocks (each cut after its last complete line) end at ever
    different offsets, and lines start and end all over the 4 KiB tiles and cross their edges."""
    rng = np.random.default_rng(block)
    lines = []
    for i in range(30000):
        pad = " " * int(i % 29)
        lines.append("%d %d%s %d" % (rng.integers(1, 500), rng.integers(1, 400), pad, rng.integers(1, 6)))
    text = mm_text(500, 400, lines)
    both(tmp_path, "blk", text, monkeypatch, block=block)


# ---- validation and value pre-processing --------------------------------------------------------
@pytest.mark.parametrize("validation", [True, False])
@pytest.mark.parametrize("prepro", [None, "OneBased", "MinMaxScalar", "ImplicitALS"])
def test_validation_and_prepro(cuda_lib, tmp_path, monkeypatch, validation, prepro):
    rng = np.random.default_rng(6)
    lines = random_lines(rng, 300, 200, 20000, lambda a, b, r: "%d %d %s" % (a, b, ["1", "2", "3.5", "0.25", "5"][r.integers(5)]))
    popt = None
    if prepro == "MinMaxScalar":
        popt = {"name": prepro, "min": 1.0, "max": 5.0}
    elif prepro == "ImplicitALS":
        popt = {"name": prepro, "epsilon": 0.5}
    elif prepro:
        popt = {"name": prepro}
    host, dev = both(tmp_path, "vp", mm_text(300, 200, lines), monkeypatch, validation=validation, prepro=popt, seed=11)
    if validation:
        assert dev.handle["vali"].attrs["num_samples"] == 200


def test_large_file(cuda_lib, tmp_path, monkeypatch):
    """20 M entries: many 64 MiB blocks, thousands of CTAs per block, the scans and both CSR builds at size."""
    U, I, n = 400000, 60000, 20_000_000
    rng = np.random.default_rng(8)
    r = rng.integers(1, U + 1, n)
    c = rng.integers(1, I + 1, n)
    v = rng.integers(1, 6, n)
    path = tmp_path / "big.mtx"
    write_mm(path, U, I, r, c, v)
    assert os.path.getsize(path) > 3 * (64 << 20)
    _, dev = both(tmp_path, "big", None, monkeypatch)
    assert dev.get_header()["num_nnz"] == n - 500


# ---- fallback and errors ---------------------------------------------------------------------------
REJECTED = {
    "mixed_2_and_3_tokens": ["1 2 3", "2 2", "3 1 1"],
    "float_index": ["1 2 3", "2.0 2 1", "3 1 1"],
    "signed_index": ["1 2 3", "+2 2 1", "3 1 1"],
    "bare_cr": ["1 2 3", "2 2 1\r3 1 1", "1 1 2"],
    "overlong_line": ["1 2 3", "2 2 1 % " + "x" * 1100, "3 1 1"],
    "control_char": ["1 2 3", "2 2 1\v", "3 1 1"],
    "more_lines_than_header": None,
}


@pytest.mark.parametrize("case", sorted(REJECTED))
def test_rejected_constructs_fall_back(cuda_lib, tmp_path, monkeypatch, case):
    rng = np.random.default_rng(9)
    body = random_lines(rng, 3, 3, 400, lambda a, b, r: "%d %d %d" % (a, b, r.integers(1, 6)))
    lines = REJECTED[case]
    if lines is None:
        text = mm_text(3, 3, body, nnz=len(body) - 10)
    else:
        text = mm_text(3, 3, body[:200] + lines + body[200:])
    both(tmp_path, case, text, monkeypatch, expect_device=False)


@pytest.mark.parametrize("bad", ["0 1 1", "4 1 1", "1 0 2", "2 6 1", "99999999999 1 1"])
def test_out_of_range_raises_with_line(cuda_lib, tmp_path, monkeypatch, bad):
    lines = ["1 1 1", "2 2 2", "3 3 3"] * 50
    lines.insert(77, bad)
    text = mm_text(3, 5, lines)
    with pytest.raises(ValueError, match=r"line %d\b" % (77 + 3)):    # banner and size lines come first
        _build(tmp_path, "oor", text, True, monkeypatch)

"""Device Stream parser (csrc/stream_ingest.cu, data/stream.py::_device_ingest): every case builds the same session
file through the host loop and the device path, with NumPy seeded identically before each, and compares every array
and attr of the two databases bitwise.  Files the device path declines must fall back to the host loop and still
match, or raise what the host loop raises."""
import numpy as np
import pytest

from tests.test_mm_ingest_gpu import assert_same_db

pytestmark = pytest.mark.gpu

KNOWN = [("apple mango mango apple pie juice coke\npie\njuice coke grape", "kim\nlee\npark"),
         ("사과 망고 망고 사과 파이 주스 콜라\n파이\n주스 콜라 포도", "김씨\n이씨\n박씨")]


def _build(tmp_path, name, text, device, monkeypatch, uid=None, iid=None, matrix=False, validation="newest-1",
           block=None, hash_bits=None, seed=7):
    from buffalo_b200.data import stream as smod
    from buffalo import Stream, StreamOptions
    files = {"main": text, "uid": uid, "iid": iid}
    opt = StreamOptions().get_default_option()
    for k, v in files.items():
        if v is None:
            continue
        p = tmp_path / ("%s.%s" % (name, k))
        if not p.exists():
            p.write_bytes(v if isinstance(v, bytes) else v.encode())
        opt.input[k] = str(p)
    monkeypatch.setattr(smod, "DEVICE_INGEST_MIN_BYTES", 0 if device else 1 << 62)
    if block:
        monkeypatch.setattr(smod, "DEVICE_INGEST_BLOCK_BYTES", block)
    if hash_bits:
        monkeypatch.setattr(smod, "_HASH_BITS", hash_bits)
    opt.data.tmp_dir = str(tmp_path)
    opt.data.path = str(tmp_path / ("%s_%s.h5py" % (name, "dev" if device else "host")))
    opt.data.internal_data_type = "matrix" if matrix else "stream"
    if validation is None:
        opt.data.validation = {}
    elif validation.startswith("newest"):
        opt.data.validation.update(name="newest", n=int(validation.split("-")[1]))
    else:                                     # sample-p-max
        _, p, mx = validation.split("-")
        opt.data.validation.update(name="sample", p=float(p), max_samples=int(mx))
    np.random.seed(seed)
    db = Stream(opt)
    db.create()
    return db


def both(tmp_path, name, text, monkeypatch, expect_device=True, **kw):
    host = _build(tmp_path, name, text, False, monkeypatch, **kw)
    dev = _build(tmp_path, name, text, True, monkeypatch, **kw)
    assert hasattr(dev, "ingest_stats") == expect_device, "device path %s" % ("expected" if expect_device else "not expected")
    assert_same_db(host, dev)
    return host, dev


def zipf_sessions(seed, users, vocab, mean_len, sep=" ", empty=0.05, max_len=None):
    rng = np.random.default_rng(seed)
    toks = ["t%d" % i for i in range(vocab)]
    lines = []
    for _ in range(users):
        n = 0 if rng.random() < empty else int(rng.geometric(1.0 / mean_len))
        n = n if max_len is None else min(n, max_len)
        ids = np.minimum(rng.zipf(1.3, n) - 1, vocab - 1)
        lines.append(sep.join(toks[i] for i in ids))
    return "\n".join(lines) + "\n"


@pytest.mark.parametrize("matrix", [False, True], ids=["stream", "matrix"])
@pytest.mark.parametrize("k", [0, 1], ids=["ascii", "korean"])
def test_known_answer(cuda_lib, tmp_path, monkeypatch, k, matrix):
    text, uids = KNOWN[k]
    _, dev = both(tmp_path, "ka", text, monkeypatch, uid=uids, matrix=matrix)
    h = dev.get_header()
    assert (h["num_users"], h["num_items"], h["num_nnz"]) == (3, 6, 7 if matrix else 9)


@pytest.mark.parametrize("matrix", [False, True], ids=["stream", "matrix"])
@pytest.mark.parametrize("validation", ["newest-1", "newest-2", "newest-5", "sample-0.05-100", "sample-0.0001-10", None])
def test_validation(cuda_lib, tmp_path, monkeypatch, validation, matrix):
    text = zipf_sessions(3, 700, 300, 12)
    _, dev = both(tmp_path, "v", text, monkeypatch, validation=validation, matrix=matrix)
    if validation == "sample-0.05-100":
        assert dev.get_group("vali").attrs["num_samples"] > 0
    if validation == "sample-0.0001-10":
        assert dev.get_group("vali").attrs["num_samples"] == 0


@pytest.mark.parametrize("matrix", [False, True], ids=["stream", "matrix"])
@pytest.mark.parametrize("case", ["uid", "iid", "iid_dup", "iid_unused", "uid_longer", "uid_iid"])
def test_uid_iid(cuda_lib, tmp_path, monkeypatch, case, matrix):
    text = zipf_sessions(4, 300, 50, 8)
    lines = text.count("\n")
    vocab = sorted({t for ln in text.split("\n") for t in ln.split()}, key=lambda t: int(t[1:]))
    kw = {}
    if "uid" in case:
        kw["uid"] = "\n".join("user%d" % i for i in range(lines + (40 if case == "uid_longer" else 0))) + "\n"
    if "iid" in case:
        names = list(reversed(vocab))
        if case == "iid_dup":
            names = names[:10] + names[3:8] + names[10:] + names[:2]      # repeated names take their last index
        if case == "iid_unused":
            names = ["never%d" % i for i in range(25)] + names + ["unused"]
        kw["iid"] = "\n".join(names) + "\n"
    both(tmp_path, "u", text, monkeypatch, matrix=matrix, **kw)


TEXTS = {
    "empty_lines": "\n\na b\n\n\nc a a\n\n",
    "one_token": "x\ny\nx\nz\n",
    "repeats": "a a a a b a b b\nb b b\n",
    "long_session": " ".join("w%d" % (i % 997) for i in range(6000)) + "\nshort\n" + " ".join("w%d" % i for i in range(3000)),
    "no_final_newline": "a b c\nd e\nf",
    "crlf": "a b c\r\nd e a\r\n\r\nf\r\n",
    "separators": "a\tb\x0bc\x0cd\x1ce\x1df\x1eg\x1fh\n \t\x0b\x0c a  \t\t b\x1c\x1c\x1cc  \n\t\n",
    "unicode_tokens": "café naïve 日本 😀 café\n😀 x\n",
}


@pytest.mark.parametrize("matrix", [False, True], ids=["stream", "matrix"])
@pytest.mark.parametrize("name", sorted(TEXTS))
def test_texts(cuda_lib, tmp_path, monkeypatch, name, matrix):
    both(tmp_path, name, TEXTS[name], monkeypatch, matrix=matrix, validation="newest-2")


@pytest.mark.parametrize("block", [64, 100, 4099])
def test_tiny_blocks(cuda_lib, tmp_path, monkeypatch, block):
    text = zipf_sessions(5, 400, 200, 5, max_len=10)          # lines of at most 49 bytes straddle the blocks
    for matrix in (False, True):
        both(tmp_path, "b%d" % block, text, monkeypatch, block=block, matrix=matrix)


def test_line_longer_than_block_declines(cuda_lib, tmp_path, monkeypatch):
    text = "a b\n" + " ".join("tok%d" % i for i in range(40)) + "\nc\n"
    both(tmp_path, "long", text, monkeypatch, expect_device=False, block=64)


@pytest.mark.parametrize("seed", [11, 12, 13])
def test_random_zipf(cuda_lib, tmp_path, monkeypatch, seed):
    text = zipf_sessions(seed, 40000, 30000, 15)
    assert len(text) > 2 << 20
    for matrix in (False, True):
        _, dev = both(tmp_path, "z%d" % seed, text, monkeypatch, matrix=matrix, block=1 << 20,
                      validation="sample-0.01-300" if matrix else "newest-1")
        assert dev.ingest_stats["device_ms"]["parse"] > 0


def test_table_growth(cuda_lib, tmp_path, monkeypatch):
    """~90k new tokens in the first 1 MiB block overflow the initial 65536-slot table (claim retried after a rehash);
    later blocks push the load past 1/2 (rehash between blocks)."""
    rng = np.random.default_rng(21)
    ids = rng.integers(0, 150000, 400000)
    text = "\n".join(" ".join("t%d" % i for i in ids[k:k + 20]) for k in range(0, len(ids), 20)) + "\n"
    for matrix in (False, True):
        _, dev = both(tmp_path, "grow", text, monkeypatch, matrix=matrix, block=1 << 20)
        assert dev.get_header()["num_items"] > 130000      # about 139.6k distinct of 150k ids


@pytest.mark.parametrize("text", ["a b\rc d\n", "a b\nc d\r", "a\r\rb\n"], ids=["inner", "final", "double"])
def test_bare_cr_declines(cuda_lib, tmp_path, monkeypatch, text):
    both(tmp_path, "cr", text, monkeypatch, expect_device=False)


@pytest.mark.parametrize("bad", [b"\xff", b"\xc0\xaf", b"\xe0\x80\xaf", b"\xed\xa0\x80", b"\xf4\x90\x80\x80", b"\x80", b"\xc3",
                                 b"\xe6\x97"], ids=["ff", "overlong2", "overlong3", "surrogate", "above_max", "lone_cont",
                                                    "cut2", "cut3"])
def test_invalid_utf8_raises_like_host(cuda_lib, tmp_path, monkeypatch, bad):
    text = b"a b\nc " + bad + b" d\ne\n"
    for device in (False, True):
        with pytest.raises(UnicodeDecodeError):
            _build(tmp_path, "bad", text, device, monkeypatch)


@pytest.mark.parametrize("cp", [0x85, 0xA0, 0x1680, 0x2000, 0x200A, 0x2028, 0x2029, 0x202F, 0x205F, 0x3000])
def test_multibyte_space_declines(cuda_lib, tmp_path, monkeypatch, cp):
    text = "a b\nc" + chr(cp) + "d e\nf\n"
    both(tmp_path, "sp", text, monkeypatch, expect_device=False, matrix=True)


def test_token_missing_from_iid_raises_like_host(cuda_lib, tmp_path, monkeypatch):
    for device in (False, True):
        with pytest.raises(KeyError):
            _build(tmp_path, "miss", "a b\nc\n", device, monkeypatch, iid="a\nb\n")


def test_hash_collision_declines(cuda_lib, tmp_path, monkeypatch):
    text = zipf_sessions(6, 200, 100, 6)
    both(tmp_path, "hc", text, monkeypatch, expect_device=False, hash_bits=2)
    both(tmp_path, "hc1", "a a a\na\n", monkeypatch, hash_bits=2)      # one distinct token: no collision


def test_memory_decline(cuda_lib, tmp_path, monkeypatch):
    from buffalo_b200 import backend
    monkeypatch.setattr(backend, "device_free_bytes", lambda: 0)
    both(tmp_path, "mem", "a b\nc\n", monkeypatch, expect_device=False)


def test_als_on_device_built_db(cuda_lib, tmp_path, monkeypatch):
    from buffalo import ALS, ALSOption
    text = zipf_sessions(8, 3000, 800, 10)
    host, dev = both(tmp_path, "als", text, monkeypatch, matrix=True)
    out = []
    for db in (host, dev):
        opt = ALSOption().get_default_option()
        opt.update(d=32, num_iters=1, random_seed=3)
        als = ALS(opt)
        als.set_data(db)
        np.random.seed(9)
        als.initialize()
        als.train()
        out.append((als.P.copy(), als.Q.copy()))
    for a, b in zip(out[0], out[1]):
        assert np.abs(a - b).max() <= 1e-5 * np.abs(a).max()

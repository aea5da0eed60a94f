"""Batch recommendations without each user's seen items (ParALS / ParBPRMF.topk_recommendation(exclude_seen=...)) where
no GPU is needed: the NumPy path against an fp64 reference, the argument errors, the unchanged default, and the C ABI
of bfl_seen_topk*."""
import ctypes
import os
import re

import numpy as np
import pytest
import scipy.sparse

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Opt(dict):
    __getattr__ = dict.get


class _Ids(object):
    def __init__(self, U, I):
        self.userids = ["u%d" % i for i in range(U)]
        self.itemids = ["i%d" % i for i in range(I)]


class _Data(object):
    """The part of a database exclude_seen=True reads: the "rowwise" group (END offsets, keys)."""

    def __init__(self, indptr, keys):
        self.groups = {"rowwise": {"indptr": np.asarray(indptr, np.int64), "key": np.asarray(keys, np.int32)}}

    def get_group(self, name):
        return self.groups[name]


class FakeAlgo(object):
    def __init__(self, U=40, I=230, d=12, bias=False, seed=3, data=None):
        rng = np.random.default_rng(seed)
        self.P = rng.normal(size=(U, d)).astype(np.float32)
        self.Q = rng.normal(size=(I, d)).astype(np.float32)
        self.Qb = rng.normal(size=(I, 1)).astype(np.float32)
        self.opt = _Opt(num_workers=1, _nrz_P=False, _nrz_Q=False, use_bias=bias)
        self._idmanager = _Ids(U, I)
        self.data = data

    def get_index_pool(self, keys, group="item"):
        names = self._idmanager.itemids if group == "item" else self._idmanager.userids
        pos = {n: i for i, n in enumerate(names)}
        return [pos.get(k) for k in keys] if isinstance(keys, list) else keys


def fp64_reference(algo, bias, users, k, seen, pool=None):
    """Keys of the fp64 ranking: score descending, then candidate position, seen items removed, -1 padded."""
    cand = np.arange(algo.Q.shape[0]) if pool is None else np.asarray(pool)
    s = algo.P[users].astype(np.float64) @ algo.Q[cand].astype(np.float64).T
    if bias:
        s = s + algo.Qb[cand, 0].astype(np.float64)[None, :]
    out = np.full((len(users), k), -1, np.int32)
    for r, u in enumerate(users):
        keep = np.array([c not in seen[u] for c in cand])
        pos = np.nonzero(keep)[0]
        order = pos[np.argsort(-s[r, pos], kind="stable")][:k]
        out[r, :len(order)] = cand[order]
    return out


@pytest.fixture
def no_device(monkeypatch):
    from buffalo_b200 import backend
    monkeypatch.setattr(backend, "device_available", lambda: False)


def random_seen(U, I, seed, unsorted=True):
    """Rows of 0..60 items with duplicates, in random order; the dict of sets and the CSR (END offsets, keys)."""
    rng = np.random.default_rng(seed)
    rows = [rng.integers(0, I, size=rng.integers(0, 60)) for _ in range(U)]
    if not unsorted:
        rows = [np.unique(r) for r in rows]
    indptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
    keys = np.concatenate(rows).astype(np.int32)
    return {u: set(r.tolist()) for u, r in enumerate(rows)}, indptr, keys


@pytest.mark.parametrize("cls,bias", [("ParALS", False), ("ParBPRMF", True)])
def test_numpy_path_matches_fp64_reference(no_device, cls, bias):
    from buffalo_b200.parallel import base
    U, I = 40, 230
    seen, indptr, keys = random_seen(U, I, 1)
    algo = FakeAlgo(U, I, bias=bias, data=_Data(indptr, keys))
    par = getattr(base, cls)(algo)
    users = [3, 0, 39, 17, 17, 8]
    names = ["u%d" % u for u in users]
    lens = np.diff(indptr, prepend=0)
    coo = scipy.sparse.coo_matrix((np.ones(len(keys)), (np.repeat(np.arange(U), lens), keys)), shape=(U, I))
    pool_ids = np.random.default_rng(2).permutation(I)[:90]
    pool = ["i%d" % p for p in pool_ids]
    for k in (1, 10, 200):
        want = fp64_reference(algo, bias, users, k, seen)
        for ex in (True, coo.tocsr(), coo):
            kept, got, scores = par.topk_recommendation(names, topk=k, exclude_seen=ex)
            assert kept == names and np.array_equal(got, want), (k, type(ex))
            assert (scores[got == -1] == 0).all()
        want_p = fp64_reference(algo, bias, users, k, seen, pool=pool_ids)
        _, got, _ = par.topk_recommendation(names, topk=k, pool=pool, exclude_seen=True)
        assert np.array_equal(got, want_p), k
    # repr drops the padding
    _, rnames, _ = par.topk_recommendation(names, topk=200, pool=pool, exclude_seen=True, repr=True)
    assert [len(r) for r in rnames] == [len(set(pool_ids.tolist()) - seen[u]) for u in users]


def test_history_covering_all_but_three_items(no_device):
    from buffalo_b200.parallel import base
    U, I = 5, 50
    row = np.setdiff1d(np.arange(I), [7, 31, 44])[::-1]
    indptr = np.array([0, 0, len(row), len(row), len(row)], np.int64)
    algo = FakeAlgo(U, I, bias=True, data=_Data(indptr, row))
    par = base.ParBPRMF(algo)
    _, keys, scores = par.topk_recommendation(["u2", "u1"], topk=6, exclude_seen=True)
    s = algo.P[2] @ algo.Q[[7, 31, 44]].T + algo.Qb[[7, 31, 44], 0]
    assert keys[0, :3].tolist() == np.array([7, 31, 44])[np.argsort(-s, kind="stable")].tolist()
    assert (keys[0, 3:] == -1).all() and (scores[0, 3:] == 0).all()
    assert (keys[1] >= 0).all()                   # u1 has no history
    # a pool inside the history leaves nothing
    _, keys, scores = par.topk_recommendation(["u2"], topk=4, pool=["i0", "i1"], exclude_seen=True)
    assert (keys == -1).all() and (scores == 0).all()


def test_stream_database_rows_unsorted_with_duplicates(no_device, tmp_path):
    from buffalo import Stream, StreamOptions
    from buffalo_b200.parallel import base
    rng = np.random.default_rng(5)
    sessions = [[int(x) for x in rng.integers(0, 60, size=rng.integers(1, 25))] for _ in range(30)]
    (tmp_path / "main").write_text("\n".join(" ".join("t%d" % t for t in s) for s in sessions) + "\n")
    opt = StreamOptions().get_default_option()
    opt.input.main = str(tmp_path / "main")
    opt.data.path = str(tmp_path / "s.h5py")
    opt.data.tmp_dir = str(tmp_path)
    opt.data.validation = {}
    db = Stream(opt)
    db.create()
    h = db.get_header()
    grp = db.get_group("rowwise")
    indptr = np.asarray(grp["indptr"][:], np.int64)
    keys = np.asarray(grp["key"][:int(indptr[-1])])
    rows = np.split(keys, indptr[:-1])
    assert any((np.diff(r) < 0).any() for r in rows) and any(len(np.unique(r)) < len(r) for r in rows)
    algo = FakeAlgo(int(h["num_users"]), int(h["num_items"]), data=db)
    par = base.ParALS(algo)
    users = list(range(0, algo.P.shape[0], 2))
    seen = {u: set(r.tolist()) for u, r in enumerate(rows)}
    _, got, _ = par.topk_recommendation(["u%d" % u for u in users], topk=15, exclude_seen=True)
    assert np.array_equal(got, fp64_reference(algo, False, users, 15, seen))
    db.close()


def test_default_is_todays_result(no_device):
    from buffalo_b200.parallel import base
    seen, indptr, keys = random_seen(40, 230, 4)
    algo = FakeAlgo(bias=True, data=_Data(indptr, keys))
    par = base.ParBPRMF(algo)
    names = ["u1", "u30", "nobody"]
    a = par.topk_recommendation(names, topk=9)
    b = par.topk_recommendation(names, topk=9, exclude_seen=False)
    assert a[0] == b[0] and np.array_equal(a[1], b[1]) and np.array_equal(a[2].view(np.uint32), b[2].view(np.uint32))
    idx = np.array([1, 30])
    k = np.zeros((2, 9), np.int32)
    v = np.zeros((2, 9), np.float32)
    base.dot_topn(idx, algo.P, algo.Q, algo.Qb, k, v, None, 9)
    assert np.array_equal(a[1], k) and np.array_equal(a[2].view(np.uint32), v.view(np.uint32))


def test_bad_exclude_seen_raises(no_device):
    from buffalo_b200.parallel import base
    algo = FakeAlgo(10, 30)
    par = base.ParALS(algo)
    with pytest.raises(ValueError, match="pass a scipy"):
        par.topk_recommendation(["u1"], topk=3, exclude_seen=True)
    with pytest.raises(ValueError, match="must be a"):
        par.topk_recommendation(["u1"], topk=3, exclude_seen=scipy.sparse.csr_matrix((10, 31)))
    with pytest.raises(ValueError, match="must be a"):
        par.topk_recommendation(["u1"], topk=3, exclude_seen=scipy.sparse.csr_matrix((9, 30)))
    m = scipy.sparse.csr_matrix((np.ones(2), np.array([1, 2]), np.array([0, 2] + [2] * 9)), shape=(10, 30))
    m.indices[1] = 30
    with pytest.raises(ValueError, match="outside"):
        par.topk_recommendation(["u1"], topk=3, exclude_seen=m)


def _declared_seen():
    text = open(os.path.join(ROOT, "include", "buffalo_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return {name: args.count(",") + 1 for name, args in re.findall(r"\b(bfl_seen_[a-z0-9_]+)\s*\(([^)]*)\)", text)}


def test_seen_symbols_exported_with_declared_arity():
    from buffalo_b200 import _cabi
    handle = ctypes.CDLL(_cabi.LIB_PATH)
    decl = _declared_seen()
    assert set(decl) == {"bfl_seen_topk", "bfl_seen_topk_device"}
    for name, arity in decl.items():
        assert hasattr(handle, name), name
        assert len(_cabi.PROTOTYPES[name][1]) == arity, name


def test_wrapper_checks_seen_rows_before_the_device():
    from buffalo_b200 import backend
    h = backend.Serve()
    h.num_items, h.num_queries = 10, 4          # as after set_items / set_queries; no device call below
    q = np.arange(3, dtype=np.int32)
    good = np.array([1, 1, 3], np.int64), np.array([0, 9, 2], np.int32)
    for ptr, keys, msg in [(good[0].astype(np.int32), good[1], "dtype"), (good[0], good[1].astype(np.int64), "dtype"),
                           (np.array([[1, 1, 3]], np.int64), good[1], "dtype"),
                           (np.array([1, 1, 3, 3, 3, 3], np.int64)[::2], good[1], "C-contiguous"),
                           (good[0][:2], good[1], "one END offset per query"),
                           (np.array([2, 1, 3], np.int64), good[1], "non-decreasing"),
                           (np.array([-1, 1, 3], np.int64), good[1], "non-decreasing"),
                           (np.array([1, 1, 4], np.int64), good[1], "ends past"),
                           (good[0], np.array([0, 10, 2], np.int32), "out of range"),
                           (good[0], np.array([0, -1, 2], np.int32), "out of range")]:
        with pytest.raises(ValueError, match=msg):
            h.topk_seen(q, 3, ptr, keys)
    with pytest.raises(ValueError, match="k must be in"):
        h.topk_seen(q, 0, *good)
    with pytest.raises(ValueError, match="query index out of range"):
        h.topk_seen(np.array([4], np.int32), 3, good[0][:1], good[1])
    h.close()


def test_native_seen_call_checks_state_and_rows():
    from buffalo_b200 import _cabi
    lib = _cabi.lib()
    h = lib.bfl_serve_create()
    q = np.zeros(2, np.int32)
    out = np.zeros((2, 3), np.int32)
    ptr = np.array([1, 2], np.int64)
    keys = np.array([0, 1], np.int32)
    assert lib.bfl_seen_topk(h, q.ctypes.data, 2, 3, ptr.ctypes.data, keys.ctypes.data, out.ctypes.data, None) == 3
    assert lib.bfl_seen_topk(None, q.ctypes.data, 2, 3, ptr.ctypes.data, keys.ctypes.data, out.ctypes.data, None) == 4
    lib.bfl_serve_destroy(h)

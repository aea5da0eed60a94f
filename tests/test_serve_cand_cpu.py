"""Per-user candidate pools (ParALS / ParBPRMF.topk_recommendation(pool=<sparse matrix>)) where no GPU is needed: the
NumPy path against an fp64 per-row reference, empty rows and padding, non-canonical rows, the argument errors raised
before any device work, and the C ABI of bfl_cand_topk*."""
import numpy as np
import pytest
import scipy.sparse

from tests.test_ivf_cpu import cpu_model


def fp64_rows(P, Q, Qb, users, rows, k, seen=None):
    """Per row: the candidates of its list ranked by the fp64 score, ties to the earlier position, seen items removed,
    -1 padded."""
    out = np.full((len(users), k), -1, np.int32)
    for i, (u, cand) in enumerate(zip(users, rows)):
        cand = np.asarray(cand, np.int64)
        if not cand.size:
            continue
        s = Q[cand].astype(np.float64) @ P[u].astype(np.float64)
        if Qb is not None:
            s = s + Qb.reshape(-1)[cand].astype(np.float64)
        order = sorted(range(len(cand)), key=lambda j: (-s[j], j))
        if seen is not None:
            order = [j for j in order if cand[j] not in seen[i]]
        order = order[:k]
        out[i, :len(order)] = cand[order]
    return out


def pool_matrix(rows, U, I):
    """CSR (U, I) whose row u lists rows[u] in the given order (duplicates kept, indices unsorted)."""
    indptr = np.concatenate([[0], np.cumsum([len(r) for r in rows])]).astype(np.int64)
    indices = np.concatenate([np.asarray(r, np.int32) for r in rows]) if indptr[-1] else np.zeros(0, np.int32)
    return scipy.sparse.csr_matrix((np.ones(len(indices), np.float32), indices, indptr), shape=(U, I))


def random_rows(U, I, seed, lens=None):
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 40, size=U) if lens is None else lens
    return [rng.integers(0, I, size=int(n)) for n in lens]


@pytest.fixture
def numpy_path(monkeypatch):
    """The NumPy path: no device, whatever the machine has."""
    from buffalo_b200 import backend
    monkeypatch.setattr(backend, "device_available", lambda: False)


@pytest.fixture
def no_device_work(monkeypatch):
    """Any serve-handle step fails the test."""
    from buffalo_b200 import backend

    def refuse(*a, **k):
        raise AssertionError("device work before the checks finished")
    for name in ("set_items", "set_queries", "topk_candidates", "topk_candidates_device", "topk", "topk_seen"):
        monkeypatch.setattr(backend.Serve, name, refuse)
    monkeypatch.setattr(backend, "device_available", lambda: True)


@pytest.mark.parametrize("kind", ["als", "bpr"])
@pytest.mark.parametrize("k", [1, 7, 50])
def test_numpy_path_matches_fp64(numpy_path, kind, k):
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    m = cpu_model(kind, U=60, I=200, d=12, use_bias=True)
    par = (ParALS if kind == "als" else ParBPRMF)(m)
    rows = random_rows(60, 200, 1)
    users = np.array([5, 0, 59, 17, 17, 33], np.int32)
    kept, keys, scores = par.topk_recommendation(users, topk=k, pool=pool_matrix(rows, 60, 200))
    Qb = m.Qb if kind == "bpr" else None
    want = fp64_rows(m.P, m.Q, Qb, users, [rows[u] for u in users], k)
    np.testing.assert_array_equal(keys, want)
    # scores are the fp32 dot products (+ bias) of the chosen items, 0.0 on the padding
    for i, u in enumerate(users):
        got = keys[i] >= 0
        s = m.Q[keys[i][got]] @ m.P[u] + (0 if Qb is None else Qb.reshape(-1)[keys[i][got]])
        np.testing.assert_allclose(scores[i][got], s, rtol=1e-5, atol=1e-5)
        assert (scores[i][~got] == 0).all()


def test_empty_rows_padding_and_unqueried_users(numpy_path):
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als", U=10, I=30, d=4)
    rows = [[], [3], [1, 2, 3, 4], list(range(30)), [], [7, 7, 7], [], [], [], [29, 0]]
    M = pool_matrix(rows, 10, 30)
    users = np.array([0, 1, 2, 5, 9], np.int32)
    _, keys, scores = ParALS(m).topk_recommendation(users, topk=3, pool=M)
    assert (keys[0] == -1).all() and (scores[0] == 0).all()
    assert keys[1, 0] == 3 and (keys[1, 1:] == -1).all() and (scores[1, 1:] == 0).all()
    assert (keys[3] == 7).all()                                       # duplicates are distinct candidates
    np.testing.assert_array_equal(keys, fp64_rows(m.P, m.Q, None, users, [rows[u] for u in users], 3))
    # rows of users not asked for are ignored, whatever they hold
    rows2 = list(rows)
    rows2[3], rows2[4] = [5, 6], [0]
    _, keys2, _ = ParALS(m).topk_recommendation(users, topk=3, pool=pool_matrix(rows2, 10, 30))
    np.testing.assert_array_equal(keys2, keys)


def test_non_canonical_rows_and_exclude_seen(numpy_path):
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als", U=8, I=40, d=6)
    rows = [[30, 2, 2, 17, 5, 30, 0], [39, 1, 38, 1], [], [4], [5, 6, 7, 8, 9, 10], [0], [1], [2]]
    M = pool_matrix(rows, 8, 40)
    assert not M.has_sorted_indices
    seen_rows = [[2, 30], [1], [0], [4], [6, 9, 11], [], [], []]
    S = pool_matrix(seen_rows, 8, 40)
    users = np.arange(8, dtype=np.int32)
    _, keys, _ = ParALS(m).topk_recommendation(users, topk=5, pool=M, exclude_seen=S)
    want = fp64_rows(m.P, m.Q, None, users, rows, 5, seen=[set(r) for r in seen_rows])
    np.testing.assert_array_equal(keys, want)
    assert keys[0, 0] in (17, 5, 0) and (keys[3] == -1).all()


def test_list_keys_and_repr(numpy_path):
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als", U=6, I=20, d=4)
    rows = [[1, 2], [3, 4, 5], [], [6], [7, 8], [9]]
    kept, names, _ = ParALS(m).topk_recommendation(["u1", "u2", "u4"], topk=2, pool=pool_matrix(rows, 6, 20),
                                                   repr=True)
    assert kept == ["u1", "u2", "u4"]
    want = fp64_rows(m.P, m.Q, None, [1, 2, 4], [rows[1], rows[2], rows[4]], 2)
    assert names == [["i%d" % t for t in row if t != -1] for row in want]
    assert names[1] == []


def test_argument_errors_before_device_work(no_device_work):
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als", U=10, I=30, d=4)
    par = ParALS(m)
    users = np.arange(4, dtype=np.int32)
    good = pool_matrix(random_rows(10, 30, 2), 10, 30)
    with pytest.raises(ValueError, match=r"pool must be a \(10, 30\) matrix"):
        par.topk_recommendation(users, pool=scipy.sparse.csr_matrix((9, 30), dtype=np.float32))
    with pytest.raises(ValueError, match=r"pool must be a \(10, 30\) matrix"):
        par.topk_recommendation(users, pool=scipy.sparse.csr_matrix((10, 31), dtype=np.float32))
    bad = good.copy()
    bad.indices[0] = 30
    with pytest.raises(ValueError, match=r"column outside \[0, 30\)"):
        par.topk_recommendation(users, pool=bad)
    for k in (0, 4097):
        with pytest.raises(ValueError, match=r"k must be in \[1, 4096\]"):
            par.topk_recommendation(users, topk=k, pool=good)
    with pytest.raises(ValueError, match="nprobe does not take a pool"):
        par.topk_recommendation(users, pool=good, nprobe=4)
    with pytest.raises(ValueError, match="exclude_seen must be"):
        par.topk_recommendation(users, pool=good, exclude_seen=scipy.sparse.csr_matrix((3, 30), dtype=np.float32))
    # a list pool keeps meaning one pool for every user, and an empty one still raises
    with pytest.raises(RuntimeError, match="pool is empty"):
        par.topk_recommendation(users, pool=[])


def test_fold_in_argument_errors_before_device_work(no_device_work, monkeypatch):
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als", U=10, I=30, d=4)

    def refuse(*a, **k):
        raise AssertionError("fold-in before the checks finished")
    m._fold_in_device = refuse
    par = ParALS(m)
    hist = scipy.sparse.csr_matrix(np.eye(3, 30, dtype=np.float32))
    with pytest.raises(ValueError, match=r"pool must be a \(3, 30\) matrix"):
        par.fold_in_recommendation(hist, topk=5, pool=scipy.sparse.csr_matrix((10, 30), dtype=np.float32))
    with pytest.raises(ValueError, match=r"pool must be a \(2, 30\) matrix"):
        par.fold_in_recommendation([[], []], topk=5, pool=scipy.sparse.csr_matrix((3, 30), dtype=np.float32))
    bad = pool_matrix([[1], [2], [3]], 3, 30)
    bad.indices[1] = -1
    with pytest.raises(ValueError, match="column outside"):
        par.fold_in_recommendation(hist, topk=5, pool=bad)
    with pytest.raises(ValueError, match="histories must be"):
        par.fold_in_recommendation(np.eye(3, 30), topk=5, pool=bad)


def test_serve_argument_errors_before_native_call(monkeypatch):
    """backend.Serve.topk_candidates checks the lists before calling the library (no handle work needed)."""
    from buffalo_b200 import backend
    s = backend.Serve.__new__(backend.Serve)
    s.num_items, s.num_queries, s._h, s._lib = 30, 5, None, None
    q = np.arange(3, dtype=np.int32)
    with pytest.raises(ValueError, match="cand_indptr must hold one END offset per query"):
        s.topk_candidates(q, 4, np.array([1, 2], np.int64), np.zeros(2, np.int32))
    with pytest.raises(ValueError, match="non-decreasing"):
        s.topk_candidates(q, 4, np.array([2, 1, 3], np.int64), np.zeros(3, np.int32))
    with pytest.raises(ValueError, match=r"cand key out of range \[0, 30\)"):
        s.topk_candidates(q, 4, np.array([1, 2, 3], np.int64), np.array([0, 30, 1], np.int32))
    with pytest.raises(ValueError, match="Buffer dtype"):
        s.topk_candidates(q, 4, np.array([1, 2, 3], np.int32), np.zeros(3, np.int32))
    with pytest.raises(ValueError, match="seen key out of range"):
        s.topk_candidates(q, 4, np.array([1, 2, 3], np.int64), np.zeros(3, np.int32),
                          seen=(np.array([0, 0, 1], np.int64), np.array([-1], np.int32)))
    with pytest.raises(ValueError, match="query index out of range"):
        s.topk_candidates(np.array([5], np.int32), 4, np.array([1], np.int64), np.zeros(1, np.int32))


def test_abi_declared():
    import os
    import re
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    text = open(os.path.join(root, "include", "buffalo_b200.h")).read()
    for name in ("bfl_cand_topk", "bfl_cand_topk_device", "bfl_cand_set_budget"):
        assert re.search(r"\b%s\(" % name, text), name
    from buffalo_b200 import _cabi
    assert {"bfl_cand_topk", "bfl_cand_topk_device", "bfl_cand_set_budget"} <= set(_cabi.PROTOTYPES)

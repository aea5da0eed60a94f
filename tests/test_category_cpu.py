"""Per-category caps (topk_recommendation / fold_in_recommendation / most_similar with categories and category_cap,
cap_categories) where no GPU is needed: every argument error and the nprobe / diversify refusals before any device
work, and the NumPy path and cap_categories against the plain walk of tests/category_ref.py over the complete
ranking."""
import numpy as np
import pytest
import scipy.sparse

from tests import category_ref
from tests.test_ivf_cpu import cpu_model
from tests.test_serve_cand_cpu import pool_matrix


@pytest.fixture
def numpy_path(monkeypatch):
    """The NumPy path: no device, whatever the machine has."""
    from buffalo_b200 import backend
    monkeypatch.setattr(backend, "device_available", lambda: False)


@pytest.fixture
def no_device_work(monkeypatch):
    """Any serve-handle step, the walk on either side, or a fold-in fails the test."""
    from buffalo_b200 import backend
    from buffalo_b200.algo.als import ALS
    from buffalo_b200.parallel import base

    def refuse(*a, **k):
        raise AssertionError("device work before the checks finished")
    for name in ("set_items", "set_queries", "bind_queries", "set_pool", "topk", "topk_device", "topk_seen",
                 "topk_seen_device", "topk_candidates", "topk_candidates_device", "__init__"):
        monkeypatch.setattr(backend.Serve, name, refuse)
    monkeypatch.setattr(backend, "category_walk_device", refuse)
    monkeypatch.setattr(base, "category_walk_numpy", refuse)
    monkeypatch.setattr(ALS, "_fold_in_device", refuse, raising=False)
    monkeypatch.setattr(backend, "device_available", lambda: True)


class _Data(object):
    def __init__(self, m):
        self.m = m.tocsr()

    def get_group(self, name):
        assert name == "rowwise"
        return {"indptr": np.asarray(self.m.indptr[1:], np.int64), "key": np.asarray(self.m.indices, np.int32)}


def model(kind="als", U=30, I=50, d=8, seed=5):
    m = cpu_model(kind, U=U, I=I, d=d, use_bias=True)
    rng = np.random.default_rng(seed)
    m.P = rng.integers(-3, 4, (U, d)).astype(np.float32)     # small integers: many exact ties
    m.Q = rng.integers(-3, 4, (I, d)).astype(np.float32)
    if kind == "bpr":
        m.Qb = rng.integers(-2, 3, (I, 1)).astype(np.float32)
    m.data = _Data(scipy.sparse.random(U, I, density=0.1, format="csr", random_state=rng))
    return m


def par_of(m, kind):
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    return (ParALS if kind == "als" else ParBPRMF)(m)


# --- argument errors, before any device work ------------------------------------------------------------------------

def test_argument_errors(no_device_work):
    m = model(I=50)
    par = par_of(m, "als")
    users = np.arange(3, dtype=np.int32)
    cats = np.zeros(50, np.int64)
    bad = [
        (dict(categories=cats), "together"),
        (dict(category_cap=1), "together"),
        (dict(categories=np.zeros(49, np.int32), category_cap=1), "one entry per item"),
        (dict(categories=np.zeros((50, 1), np.int32), category_cap=1), "1-d integer"),
        (dict(categories=np.zeros(50, np.float32), category_cap=1), "1-d integer"),
        (dict(categories=np.full(50, -2), category_cap=1), r"\[-1"),
        (dict(categories=cats, category_cap=-1), ">= 0"),
        (dict(categories=cats, category_cap=1.5), "category_cap"),
        (dict(categories=cats, category_cap=True), "category_cap"),
        (dict(categories=cats, category_cap=np.array([1, -1])), "category_cap"),
        (dict(categories=cats, category_cap=np.array([1.0])), "category_cap"),
        (dict(categories=np.arange(50) % 3, category_cap=np.array([1, 1])), r"\[-1, 2\)"),
        (dict(categories=cats, category_cap=1, nprobe=2), "nprobe"),
        (dict(categories=cats, category_cap=1, diversify=0.5), "diversify"),
        (dict(categories=cats, category_cap=1, pool=np.array([1, 2, 1], np.int32)), "twice"),
        (dict(categories=cats, category_cap=1, pool=pool_matrix([[1, 2, 1]] + [[]] * 29, 30, 50)), "twice"),
    ]
    for kw, msg in bad:
        with pytest.raises(ValueError, match=msg):
            par.topk_recommendation(users, 5, **kw)
    for k in (0, 4097, 2.0):
        with pytest.raises(ValueError, match="topk"):
            par.topk_recommendation(users, k, categories=cats, category_cap=1)
    with pytest.raises(ValueError, match="nprobe"):
        par.most_similar(np.arange(2, dtype=np.int32), 5, categories=cats, category_cap=1, nprobe=2)
    with pytest.raises(ValueError, match="one entry per item"):
        par.most_similar(np.arange(2, dtype=np.int32), 5, group="user", categories=cats, category_cap=1)
    with pytest.raises(ValueError, match="diversify"):
        par.fold_in_recommendation([[1, 2]], 5, categories=cats, category_cap=1, diversify=0.1)
    with pytest.raises(ValueError, match="together"):
        par.fold_in_recommendation([[1, 2]], 5, categories=cats)
    with pytest.raises(ValueError, match="twice"):
        par.fold_in_recommendation([[1, 2]], 5, categories=cats, category_cap=1, pool=np.array([3, 3], np.int32))


def test_cap_categories_argument_errors(no_device_work):
    from buffalo_b200.parallel.base import cap_categories
    idx, val = np.array([[0, 1, -1]], np.int32), np.zeros((1, 3), np.float32)
    cats = np.array([0, 1], np.int32)
    with pytest.raises(ValueError, match="cand_idx"):
        cap_categories(idx[0], val[0], cats, 1, 2)
    with pytest.raises(ValueError, match="cand_idx"):
        cap_categories(idx.astype(np.float32), val, cats, 1, 2)
    with pytest.raises(ValueError, match="outside"):
        cap_categories(np.array([[0, 2]], np.int32), val[:, :2], cats, 1, 2)
    with pytest.raises(ValueError, match="topk"):
        cap_categories(idx, val, cats, 1, 0)
    with pytest.raises(ValueError, match="category_cap"):
        cap_categories(idx, val, cats, np.array([1]), 2)
    with pytest.raises(ValueError, match="categories"):
        cap_categories(idx, val, cats.astype(np.float64), 1, 2)


# --- the NumPy path against the reference ---------------------------------------------------------------------------

def full_then_walk(par, users, cats, cap, topk, depth, **kw):
    _, keys, scores = par.topk_recommendation(users, depth, **kw)
    return category_ref.walk(keys, scores, cats, cap, topk)


@pytest.mark.parametrize("kind", ["als", "bpr"])
def test_numpy_path_against_reference(numpy_path, kind):
    U, I = 30, 60
    m = model(kind, U, I)
    par = par_of(m, kind)
    rng = np.random.default_rng(2)
    users = np.array([0, 3, 4, 4, 17, 29], np.int32)
    cats = rng.integers(-1, 5, I)
    per_cat = np.array([0, 1, 2, 3, 1])
    rows = [rng.choice(I, int(n), replace=False) for n in rng.integers(0, 30, U)]
    rows[3] = np.zeros(0, np.int64)                              # an empty pool row
    pool = rng.choice(I, 25, replace=False).astype(np.int32)
    seen = scipy.sparse.random(U, I, density=0.2, format="csr", random_state=rng)
    for kw, depth in [(dict(), I), (dict(pool=pool), len(pool)), (dict(exclude_seen=True), I),
                      (dict(exclude_seen=seen), I), (dict(pool=pool_matrix(rows, U, I)), 30),
                      (dict(pool=pool_matrix(rows, U, I), exclude_seen=True), 30)]:
        for cap in (0, 1, 2, per_cat):
            for topk in (1, 4, 10, 100):                         # 100: more than the catalogue
                _, keys, scores = par.topk_recommendation(users, topk, categories=cats, category_cap=cap, **kw)
                want = full_then_walk(par, users, cats, cap, topk, depth, **kw)
                np.testing.assert_array_equal(keys, want[0])
                np.testing.assert_array_equal(scores, want[1])
                if np.ndim(cap) == 0 and cap == 0:
                    assert set(cats[keys[keys >= 0]]) <= {-1}     # every capped category banned
    # most_similar on the normalized rows
    m2 = model(kind, U, I)
    par2 = par_of(m2, kind)
    items = np.array([1, 5, 9], np.int32)
    got = par2.most_similar(items, 7, categories=cats, category_cap=1)
    keys, scores = par2.most_similar(items, I)
    want = category_ref.walk(keys, scores, cats, 1, 7)
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(got[1], want[1])


def test_all_uncapped_is_the_plain_result(numpy_path):
    m = model(I=40)
    par = par_of(m, "als")
    users = np.arange(10, dtype=np.int32)
    got = par.topk_recommendation(users, 8, categories=np.full(40, -1), category_cap=0)
    plain = par.topk_recommendation(users, 8)
    np.testing.assert_array_equal(got[1], plain[1])
    np.testing.assert_array_equal(got[2], plain[2])


def test_cap_categories_against_reference(numpy_path):
    from buffalo_b200.parallel.base import cap_categories
    rng = np.random.default_rng(9)
    I, n, m = 70, 40, 25
    cats = rng.integers(-1, 6, I)
    idx = rng.integers(0, I, (n, m)).astype(np.int32)
    idx[rng.random((n, m)) < 0.2] = -1
    val = rng.standard_normal((n, m)).astype(np.float32)
    for cap in (0, 1, 3, np.array([0, 1, 2, 1, 5, 2])):
        for topk in (1, 5, 25, 40):
            got = cap_categories(idx, val, cats, cap, topk)
            want = category_ref.walk(idx, val, cats, cap, topk)
            np.testing.assert_array_equal(got[0], want[0])
            np.testing.assert_array_equal(got[1], want[1])


def test_reference_by_hand():
    cats = np.array([0, 0, 1, -1, 0, 1])
    keys = np.array([[0, 1, 2, 3, 4, 5]])
    vals = np.arange(6, 0, -1, dtype=np.float32)[None]
    assert category_ref.walk(keys, vals, cats, 1, 4)[0].tolist() == [[0, 2, 3, -1]]
    assert category_ref.walk(keys, vals, cats, 2, 4)[0].tolist() == [[0, 1, 2, 3]]
    assert category_ref.walk(keys, vals, cats, np.array([0, 2]), 6)[0].tolist() == [[2, 3, 5, -1, -1, -1]]
    assert category_ref.walk(np.array([[-1, 4, -1, 0]]), vals[:, :4], cats, 1, 2)[0].tolist() == [[4, -1]]

"""ALS.explain / ParALS.explain where no GPU is needed: every input check raises before any device work, item lists map
to the index form, models without least-squares rows are refused, without a GPU a valid call raises the backend's
"no CPU fallback" error, and the fp64 reference (tests/explain_ref.py) keeps its own identities."""
import numpy as np
import pytest
import scipy.sparse

from tests import explain_ref
from tests.test_fold_in_cpu import cpu_model, history


@pytest.fixture
def no_device_work(monkeypatch):
    """Any step past the input checks (holder creation, upload) fails the test."""
    from buffalo_b200.algo import fold_in

    def refuse(*a, **k):
        raise AssertionError("device work before the input checks finished")
    monkeypatch.setattr(fold_in.ItemState, "refresh", refuse)
    monkeypatch.setattr(fold_in, "to_device", refuse)
    monkeypatch.setattr(fold_in, "csr_to_device", refuse)


class _Data(object):
    def __init__(self, U, I, seed=0):
        m = history(U, I, seed)
        self.groups = {"rowwise": {"indptr": m.indptr[1:].astype(np.int64), "key": m.indices.astype(np.int32),
                                   "val": m.data.astype(np.float32)}}

    def get_group(self, name):
        return self.groups[name]


def test_input_checks_before_device_work(no_device_work):
    m = cpu_model("als")
    I = m.Q.shape[0]
    H = history(4, I)
    good = np.zeros((4, 3), np.int32)
    with pytest.raises(ValueError, match="matrix"):
        m.explain(history(4, I + 1), good)
    with pytest.raises(ValueError, match="histories"):
        m.explain(np.zeros((4, I)), good)
    for bad in (np.zeros((3, 3), np.int32), np.zeros((4, 3, 1), np.int32), np.zeros(4, np.int32),
                np.zeros((4, 3), np.float32)):
        with pytest.raises(ValueError, match="items"):
            m.explain(H, bad)
    for bad in (-2, I):
        items = good.copy()
        items[1, 2] = bad
        with pytest.raises(ValueError, match="outside"):
            m.explain(H, items)
    with pytest.raises(ValueError, match="items"):
        m.explain(H, [["i1"]] * 3)                 # one list per row
    with pytest.raises(ValueError, match="items"):
        m.explain(H, [["i1"], "i2", ["i3"], []])
    with pytest.raises(ValueError, match="items"):
        m.explain(H, "i1")
    with pytest.raises(ValueError, match="targets"):
        m.explain(H, np.zeros((4, 4097), np.int32))
    for topm in (0, 65, -1, 2.0, True):
        with pytest.raises(ValueError, match="topm"):
            m.explain(H, good, topm=topm)
    wide = cpu_model("als", d=257)
    with pytest.raises(ValueError, match="d <= 256"):
        wide.explain(H, good)


def test_normalized_items_refused(no_device_work):
    m = cpu_model("als", _nrz_Q=True)
    with pytest.raises(RuntimeError, match="normalized"):
        m.explain(history(2, m.Q.shape[0]), np.zeros((2, 1), np.int32))


def test_item_lists_map_to_the_index_form():
    from buffalo_b200.algo import fold_in
    m = cpu_model("als", I=12)
    lists = [["i7", "nope", "i2"], [], ["i11"]]
    T = fold_in.target_matrix(m, lists, 3, 12, 4096)
    assert T.dtype == np.int32 and T.tolist() == [[7, -1, 2], [-1, -1, -1], [11, -1, -1]]
    idx = np.array([[7, -1, 2], [-1, -1, -1], [11, -1, -1]], dtype=np.int64)
    assert np.array_equal(fold_in.target_matrix(m, idx, 3, 12, 4096), T)
    assert fold_in.target_matrix(m, [[], []], 2, 12, 4096).shape == (2, 0)


def test_par_als_checks_before_device_work(no_device_work):
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als", U=30)
    par = ParALS(m)
    items = np.zeros((2, 3), np.int32)
    with pytest.raises(ValueError, match="training data"):
        par.explain(np.array([0, 1]), items)
    m.data = _Data(30, m.Q.shape[0])
    with pytest.raises(ValueError, match="unknown user"):
        par.explain(["u1", "nobody"], items)
    with pytest.raises(ValueError, match="outside"):
        par.explain(np.array([0, 30]), items)
    with pytest.raises(ValueError, match="items"):
        par.explain(["u1", "u2"], np.zeros((3, 3), np.int32))
    with pytest.raises(ValueError, match="topm"):
        par.explain(["u1", "u2"], items, topm=65)


@pytest.mark.parametrize("kind", ["bpr", "warp", "plsi"])
def test_models_without_explain_refused(kind, no_device_work):
    from buffalo_b200.algo.bpr import BPRMF
    from buffalo_b200.algo.warp import WARP
    from buffalo_b200.misc import aux
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    if kind == "plsi":
        par = ParALS(cpu_model("plsi"))
    else:
        cls = BPRMF if kind == "bpr" else WARP
        m = cls.__new__(cls)
        m.opt = aux.Option(num_workers=1, use_bias=True)
        par = ParBPRMF(m)
    with pytest.raises(NotImplementedError, match="least-squares"):
        par.explain(["u1"], np.zeros((1, 1), np.int32))


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from buffalo_b200 import _cabi
    m = cpu_model("als")
    with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
        m.explain(history(3, m.Q.shape[0]), np.zeros((3, 2), np.int32))


@pytest.mark.parametrize("adaptive_reg", [False, True])
def test_reference_identities(adaptive_reg):
    """score == q_i' solve(A, b), and all contributions of a row-target sum to its score, both in fp64"""
    rng = np.random.default_rng(3)
    I, d = 60, 7
    Q = rng.normal(scale=0.3, size=(I, d)).astype(np.float32)
    rows = [np.sort(rng.integers(0, I, n)) for n in (1, 5, 40)] + [np.array([], np.int64)]   # duplicates included
    indptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
    keys = np.concatenate(rows).astype(np.int32)
    vals = rng.random(len(keys)).astype(np.float32) * 3
    targets = rng.integers(-1, I, (len(rows), 6)).astype(np.int32)
    got = explain_ref.explain_rows(Q, indptr, keys, vals, targets, 3, 2.0, 0.5, adaptive_reg)
    G = Q.astype(np.float64).T @ Q.astype(np.float64)
    beg = np.concatenate([[0], indptr[:-1]])
    for r, res in enumerate(got):
        rk, rv = keys[beg[r]:indptr[r]], vals[beg[r]:indptr[r]]
        if not len(rk):
            assert res["x"] is None and (res["keys"] == -1).all() and (res["scores"] == 0).all()
            continue
        A, b = explain_ref.row_system(G, Q, rk, rv, 2.0, 0.5, adaptive_reg)
        for t, i in enumerate(targets[r]):
            if i < 0:
                assert res["scores"][t] == 0 and (res["keys"][t] == -1).all()
                continue
            want = Q[i].astype(np.float64) @ np.linalg.solve(A, b)
            items, c = res["ranked"][t]
            assert np.isclose(res["scores"][t], want, rtol=1e-12, atol=1e-12)
            assert np.isclose(c.sum(), want, rtol=1e-9, atol=1e-12)
            assert len(items) == len(np.unique(rk)) and (np.diff(c) <= 0).all()
            m = min(3, len(items))
            assert (res["keys"][t, m:] == -1).all() and (res["contrib"][t, m:] == 0).all()


def test_reference_tie_rule():
    """equal contributions go to the smaller item"""
    items, c = explain_ref.ranked(np.array([2, 5, 9, 11]), np.array([1.0, 3.0, 3.0, 1.0]))
    assert items.tolist() == [5, 9, 2, 11] and c.tolist() == [3.0, 3.0, 1.0, 1.0]

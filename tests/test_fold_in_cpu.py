"""Fold-in (ALS.fold_in, PLSI.fold_in, ParALS.fold_in_recommendation) where no GPU is needed: every input check raises
before any device work, the history input is read as documented, BPRMF / WARP are refused, and without a GPU a valid
call raises the backend's "no CPU fallback" error."""
import numpy as np
import pytest
import scipy.sparse


def cpu_model(kind="als", U=30, I=50, d=8, **opt):
    """A model object with factors and an item-id map, built without the backend holder (no GPU needed)."""
    from buffalo_b200.algo.als import ALS
    from buffalo_b200.algo.options import ALSOption, PLSIOption
    from buffalo_b200.algo.plsi import PLSI
    from buffalo_b200.misc import aux
    cls, opt_cls = (ALS, ALSOption) if kind == "als" else (PLSI, PLSIOption)
    m = cls.__new__(cls)
    m.opt = aux.Option(opt_cls().get_default_option())
    m.opt.update(dict(d=d, **opt))
    rng = np.random.default_rng(1)
    m.P = rng.random((U, d)).astype(np.float32)
    m.Q = rng.random((I, d)).astype(np.float32)
    m._idmanager = aux.Option({"userids": ["u%d" % i for i in range(U)], "itemids": ["i%d" % i for i in range(I)],
                               "userid_mapped": True, "itemid_mapped": True})
    m._idmanager.userid_map = {v: i for i, v in enumerate(m._idmanager.userids)}
    m._idmanager.itemid_map = {v: i for i, v in enumerate(m._idmanager.itemids)}
    return m


@pytest.fixture
def no_device_work(monkeypatch):
    """Any step past the input checks (holder creation, upload) fails the test."""
    from buffalo_b200.algo import fold_in

    def refuse(*a, **k):
        raise AssertionError("device work before the input checks finished")
    monkeypatch.setattr(fold_in.ItemState, "refresh", refuse)
    monkeypatch.setattr(fold_in, "to_device", refuse)


def history(n, I, seed=0):
    rng = np.random.default_rng(seed)
    return scipy.sparse.random(n, I, density=0.1, format="csr", random_state=rng, dtype=np.float32)


@pytest.mark.parametrize("kind", ["als", "plsi"])
def test_input_checks_before_device_work(no_device_work, kind):
    m = cpu_model(kind)
    I, d = m.Q.shape[0], m.opt.d
    good = history(4, I)
    with pytest.raises(ValueError, match="matrix"):
        m.fold_in(history(4, I + 1))
    bad = good.copy()
    bad.indices[0] = I + 3                    # scipy does not check index ranges after construction
    with pytest.raises(ValueError, match="outside"):
        m.fold_in(bad)
    bad.indices[0] = -1
    with pytest.raises(ValueError, match="outside"):
        m.fold_in(bad)
    for init in (np.zeros((3, d)), np.zeros((4, d + 1)), np.zeros(4 * d)):
        with pytest.raises(ValueError, match="init"):
            m.fold_in(good, init=init)
    with pytest.raises(ValueError, match="histories"):
        m.fold_in(np.zeros((4, I)))
    with pytest.raises(ValueError, match="history"):
        m.fold_in([[0, 1], 5])
    name = "sweeps" if kind == "als" else "iters"
    for bad_count in (0, -1, 1.5, True):
        with pytest.raises(ValueError, match=name):
            m.fold_in(good, **{name: bad_count})


def test_normalized_items_refused(no_device_work):
    m = cpu_model("als", _nrz_Q=True)
    with pytest.raises(RuntimeError, match="normalized"):
        m.fold_in(history(2, m.Q.shape[0]))


def test_history_csr_matrix_and_lists():
    from buffalo_b200.algo import fold_in
    m = cpu_model("als", I=12)
    # unsorted rows, read in ascending item order, without changing the caller's matrix
    indptr, indices = np.array([0, 3, 3, 5]), np.array([7, 2, 5, 11, 0])
    data = np.array([1, 2, 3, 4, 5], np.float64)
    mat = scipy.sparse.csr_matrix((data, indices, indptr), shape=(3, 12))
    ends, keys, vals = fold_in.history_csr(m, mat, 12)
    assert ends.dtype == np.int64 and keys.dtype == np.int32 and vals.dtype == np.float32
    assert ends.tolist() == [3, 3, 5] and keys.tolist() == [2, 5, 7, 0, 11] and vals.tolist() == [2, 3, 1, 5, 4]
    assert mat.indices.tolist() == [7, 2, 5, 11, 0]
    # lists: unknown ids dropped, value 1.0, ascending; equal to the matrix without the unknown ids
    lists = [["i7", "nope", "i2"], [], ["i11", "i0", "zzz"]]
    le, lk, lv = fold_in.history_csr(m, lists, 12)
    me, mk, mv = fold_in.history_csr(m, scipy.sparse.csr_matrix((np.ones(4), [7, 2, 11, 0], [0, 2, 2, 4]),
                                                                shape=(3, 12)), 12)
    assert le.tolist() == me.tolist() == [2, 2, 4]
    assert lk.tolist() == mk.tolist() == [2, 7, 0, 11]
    assert lv.tolist() == mv.tolist() == [1.0] * 4


def test_start_rows():
    from buffalo_b200.algo import fold_in
    assert (fold_in.start_rows(None, 3, 4, 0.25) == 0.25).all()
    X = np.arange(12, dtype=np.float64).reshape(3, 4)
    out = fold_in.start_rows(X, 3, 4, 0.0)
    assert out.dtype == np.float32 and (out == X).all()


@pytest.mark.parametrize("kind", ["bpr", "warp"])
def test_fold_in_recommendation_refuses_sgd_models(kind, no_device_work):
    from buffalo_b200.algo.bpr import BPRMF
    from buffalo_b200.algo.warp import WARP
    from buffalo_b200.misc import aux
    from buffalo_b200.parallel.base import ParBPRMF
    cls = BPRMF if kind == "bpr" else WARP
    m = cls.__new__(cls)
    m.opt = aux.Option(num_workers=1, use_bias=True)
    with pytest.raises(NotImplementedError, match="ALS, PLSI"):
        ParBPRMF(m).fold_in_recommendation([["a"]])


def test_fold_in_recommendation_checks_before_device_work(no_device_work):
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als")
    par = ParALS(m)
    with pytest.raises(ValueError, match="k must be"):
        par.fold_in_recommendation(history(2, m.Q.shape[0]), topk=0)
    with pytest.raises(RuntimeError, match="pool is empty"):
        par.fold_in_recommendation(history(2, m.Q.shape[0]), pool=np.zeros(0, np.int32))
    with pytest.raises(ValueError, match="matrix"):
        par.fold_in_recommendation(history(2, m.Q.shape[0] + 1))


@pytest.mark.parametrize("kind", ["als", "plsi"])
def test_no_cpu_fallback(kind):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from buffalo_b200 import _cabi
    m = cpu_model(kind)
    P0, Q0 = m.P.copy(), m.Q.copy()
    with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
        m.fold_in(history(3, m.Q.shape[0]))
    assert (m.P == P0).all() and (m.Q == Q0).all()

"""IVF index (ParALS.build_index, topk_recommendation / most_similar with nprobe) where no GPU is needed: every argument
error, the missing index and the stale index are raised before any device work, and without a GPU build_index and a
valid nprobe call raise the backend's "no CPU fallback" error."""
import numpy as np
import pytest
import scipy.sparse


def cpu_model(kind="als", U=30, I=50, d=8, **opt):
    """A model object with factors and an id map, built without the backend holder (no GPU needed)."""
    from buffalo_b200.algo.als import ALS
    from buffalo_b200.algo.bpr import BPRMF
    from buffalo_b200.algo.options import ALSOption, BPRMFOption
    from buffalo_b200.misc import aux
    cls, opt_cls = (ALS, ALSOption) if kind == "als" else (BPRMF, BPRMFOption)
    m = cls.__new__(cls)
    m.opt = aux.Option(opt_cls().get_default_option())
    m.opt.update(dict(d=d, **opt))
    rng = np.random.default_rng(1)
    m.P = rng.random((U, d)).astype(np.float32)
    m.Q = rng.random((I, d)).astype(np.float32)
    if kind == "bpr":
        m.Qb = rng.random((I, 1)).astype(np.float32)
    m._idmanager = aux.Option({"userids": ["u%d" % i for i in range(U)], "itemids": ["i%d" % i for i in range(I)],
                               "userid_mapped": True, "itemid_mapped": True})
    m._idmanager.userid_map = {v: i for i, v in enumerate(m._idmanager.userids)}
    m._idmanager.itemid_map = {v: i for i, v in enumerate(m._idmanager.itemids)}
    return m


@pytest.fixture
def no_device_work(monkeypatch):
    """Any step past the checks (index build, attach, search) fails the test."""
    from buffalo_b200 import backend

    def refuse(*a, **k):
        raise AssertionError("device work before the checks finished")
    for name in ("build", "search", "search_device", "_attach"):
        monkeypatch.setattr(backend.IVF, name, refuse)


def fake_index(par, group, nlist, with_bias=False):
    """An index object as build_index leaves it, for the factors as they are now (no device work)."""
    from buffalo_b200 import backend
    ivf = backend.IVF()
    F = np.ascontiguousarray(par.algo.Q if group == "item" else par.algo.P, dtype=np.float32)
    Fb = par._index_bias(group)
    ivf.nlist, ivf.num_rows, ivf.d, ivf.has_bias = nlist, F.shape[0], F.shape[1], Fb is not None
    ivf.keys = par._fingerprint(F, Fb)
    par._indexes = dict(getattr(par, "_indexes", None) or {}, **{group: ivf})
    return ivf


def test_build_index_argument_errors(no_device_work):
    from buffalo_b200.parallel.base import ParALS
    par = ParALS(cpu_model(I=50))
    for bad in (0, -1, 51, 2.0, True, None):
        with pytest.raises(ValueError, match="nlist"):
            par.build_index(bad)
    with pytest.raises(ValueError, match="nlist"):
        ParALS(cpu_model(U=10)).build_index(11, group="user")
    for bad in (0, -3, 1.5):
        with pytest.raises(ValueError, match="iters"):
            par.build_index(4, iters=bad)
    with pytest.raises(ValueError, match="group"):
        par.build_index(4, group="context")


def test_nprobe_argument_errors(no_device_work):
    from buffalo_b200.parallel.base import ParALS
    par = ParALS(cpu_model())
    users = np.arange(3, dtype=np.int32)
    with pytest.raises(ValueError, match="pool"):
        par.topk_recommendation(users, nprobe=1, pool=np.arange(5, dtype=np.int32))
    with pytest.raises(ValueError, match="exclude_seen"):
        par.topk_recommendation(users, nprobe=1, exclude_seen=True)
    with pytest.raises(ValueError, match="exclude_seen"):
        par.topk_recommendation(users, nprobe=1, exclude_seen=scipy.sparse.csr_matrix((30, 50), dtype=np.float32))
    with pytest.raises(ValueError, match="pool"):
        par.most_similar(np.arange(2, dtype=np.int32), nprobe=1, pool=np.arange(5, dtype=np.int32))
    # no index yet
    with pytest.raises(RuntimeError, match="build_index"):
        par.topk_recommendation(users, nprobe=1)
    fake_index(par, "item", 8)
    for bad in (0, 9, -1, 1.0, True):
        with pytest.raises(ValueError, match="nprobe"):
            par.topk_recommendation(users, nprobe=bad)
    with pytest.raises(ValueError, match="k must be"):
        par.topk_recommendation(users, nprobe=2, topk=0)
    # the item index does not serve the user group
    with pytest.raises(RuntimeError, match="no user index"):
        par.most_similar(np.arange(2, dtype=np.int32), group="user", nprobe=1)


def test_stale_index_edited_in_place(no_device_work):
    from buffalo_b200.parallel.base import ParALS
    par = ParALS(cpu_model())
    fake_index(par, "item", 8)
    par.algo.Q[3, 2] += 1.0
    with pytest.raises(RuntimeError, match="stale.*build_index again"):
        par.topk_recommendation(np.arange(3, dtype=np.int32), nprobe=2)


def test_stale_bias(no_device_work):
    from buffalo_b200.parallel.base import ParBPRMF
    par = ParBPRMF(cpu_model("bpr", use_bias=True))
    assert par._index_bias("item") is not None
    fake_index(par, "item", 8)
    par.algo.Qb[5, 0] += 1.0
    with pytest.raises(RuntimeError, match="stale"):
        par.topk_recommendation(np.arange(3, dtype=np.int32), nprobe=2)


def test_stale_after_normalize(no_device_work):
    """most_similar normalises first (as without nprobe), so an index built on the raw factors is stale; the message
    says to build again after normalize."""
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model()
    m.normalize = lambda group="item": setattr(m, "Q", m.Q / np.linalg.norm(m.Q, axis=1, keepdims=True))
    par = ParALS(m)
    fake_index(par, "item", 8)
    with pytest.raises(RuntimeError, match=r"stale.*after algo.normalize\('item'\)"):
        par.most_similar(np.arange(2, dtype=np.int32), nprobe=2)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from buffalo_b200 import _cabi
    from buffalo_b200.parallel.base import ParALS
    par = ParALS(cpu_model())
    Q0 = par.algo.Q.copy()
    with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
        par.build_index(4)
    assert (par.algo.Q == Q0).all()
    fake_index(par, "item", 8)
    with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
        par.topk_recommendation(np.arange(3, dtype=np.int32), nprobe=2)

"""Batch serving (buffalo.parallel ParALS / ParBPRMF, backend.Serve) without a GPU: the NumPy path is what runs when no
device is available, the bfl_serve_* C ABI is exported as declared, and the wrapper rejects bad arguments before any
device call."""
import ctypes
import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


class _Opt(dict):
    __getattr__ = dict.get


class _Ids(object):
    def __init__(self, U, I):
        self.userids = ["u%d" % i for i in range(U)]
        self.itemids = ["i%d" % i for i in range(I)]


class FakeAlgo(object):
    """The part of Algo that Par* touches, around seeded factors."""

    def __init__(self, U=37, I=211, d=12, bias=False, seed=3):
        rng = np.random.default_rng(seed)
        self.P = rng.normal(size=(U, d)).astype(np.float32)
        self.Q = rng.normal(size=(I, d)).astype(np.float32)
        self.Qb = rng.normal(size=(I, 1)).astype(np.float32)
        self.opt = _Opt(num_workers=1, _nrz_P=False, _nrz_Q=False, use_bias=bias)
        self._idmanager = _Ids(U, I)

    def get_index_pool(self, keys, group="item"):
        names = self._idmanager.itemids if group == "item" else self._idmanager.userids
        pos = {n: i for i, n in enumerate(names)}
        return [pos.get(k) for k in keys] if isinstance(keys, list) else keys

    def normalize(self, group="item"):
        if group == "item" and not self.opt._nrz_Q:
            self.Q = (self.Q / np.linalg.norm(self.Q, axis=1, keepdims=True)).astype(np.float32)
            self.opt["_nrz_Q"] = True


def exact(A, B, Bb, idx, k, pool):
    """Stable best-first top-k of fp32 NumPy scores, -1 / 0 padded (the dot_topn result)."""
    cand = B if pool is None else B[pool]
    s = A[idx].dot(cand.T)
    if Bb is not None:
        s = s + (Bb if pool is None else Bb[pool]).reshape(1, -1)
    kk = min(k, s.shape[1])
    order = np.argsort(-s, axis=1, kind="stable")[:, :kk]
    keys = np.full((len(idx), k), -1, dtype=np.int32)
    vals = np.zeros((len(idx), k), dtype=np.float32)
    keys[:, :kk] = order if pool is None else np.asarray(pool)[order]
    vals[:, :kk] = np.take_along_axis(s, order, axis=1)
    return keys, vals


@pytest.fixture
def no_device(monkeypatch):
    from buffalo_b200 import backend
    monkeypatch.setattr(backend, "device_available", lambda: False)


@pytest.mark.parametrize("cls,bias", [("ParALS", False), ("ParBPRMF", True), ("ParBPRMF", False)])
def test_numpy_path_without_device(no_device, cls, bias):
    from buffalo_b200.parallel import base
    algo = FakeAlgo(bias=bias)
    par = getattr(base, cls)(algo)
    users = ["u3", "u0", "nobody", "u36"]
    idx = np.array([3, 0, 36], dtype=np.int32)
    Qb = algo.Qb if (cls == "ParBPRMF" and bias) else None
    kept, keys, scores = par.topk_recommendation(users, topk=7)
    assert kept == ["u3", "u0", "u36"] and keys.dtype == np.int32 and scores.dtype == np.float32
    want_k, want_s = exact(algo.P, algo.Q, Qb, idx, 7, None)
    assert np.array_equal(keys, want_k) and np.array_equal(scores, want_s)
    # pool smaller than topk: -1 / 0 padding; repr drops the padding
    pool_names = ["i5", "i200", "i17"]
    kept, keys, scores = par.topk_recommendation(users, topk=5, pool=pool_names)
    want_k, want_s = exact(algo.P, algo.Q, Qb, idx, 5, [5, 200, 17])
    assert np.array_equal(keys, want_k) and np.array_equal(scores, want_s) and (keys[:, 3:] == -1).all()
    _, names, _ = par.topk_recommendation(users, topk=5, pool=pool_names, repr=True)
    assert [sorted(n) for n in names] == [sorted(pool_names)] * 3
    with pytest.raises(RuntimeError, match="pool is empty"):
        par.topk_recommendation(users, topk=5, pool=["missing"][:0])
    # most_similar normalises and returns the query item first
    keys, scores = par.most_similar(["i9", "i100"], topk=4)
    assert keys[:, 0].tolist() == [9, 100] and np.allclose(scores[:, 0], 1.0, atol=1e-6)
    want_k, _ = exact(algo.Q, algo.Q, None, np.array([9, 100]), 4, None)
    assert np.array_equal(keys, want_k)
    with pytest.raises(RuntimeError, match="normalized"):
        par.topk_recommendation(users, topk=3)


def _declared_serve():
    text = open(os.path.join(ROOT, "include", "buffalo_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    out = {}
    for name, args in re.findall(r"\b(bfl_serve_[a-z0-9_]+)\s*\(([^)]*)\)", text):
        args = args.strip()
        out[name] = 0 if args in ("", "void") else args.count(",") + 1
    return out


def test_serve_symbols_exported_with_declared_arity():
    from buffalo_b200 import _cabi
    handle = ctypes.CDLL(_cabi.LIB_PATH)
    decl = _declared_serve()
    assert set(decl) == {"bfl_serve_" + n for n in ("create", "destroy", "set_items", "bind_items_device", "set_queries",
                                                   "bind_queries_device", "set_pool", "topk", "topk_device")}
    for name, arity in decl.items():
        assert hasattr(handle, name), name
        assert len(_cabi.PROTOTYPES[name][1]) == arity, name


def test_wrapper_rejects_bad_arguments_before_the_device():
    from buffalo_b200 import backend
    h = backend.Serve()
    for k in (0, -1, backend.SERVE_KMAX + 1):
        with pytest.raises(ValueError, match="k must be in"):
            h.topk(np.zeros(3, np.int32), k)
    with pytest.raises(ValueError, match="pool is empty"):
        h.set_pool(np.zeros(0, np.int32))
    with pytest.raises(ValueError, match="dtype/ndim"):
        h.set_items(np.zeros((4, 8), np.float64))
    with pytest.raises(ValueError, match="dtype/ndim"):
        h.set_items(np.zeros(8, np.float32))
    with pytest.raises(ValueError, match="C-contiguous"):
        h.set_items(np.zeros((8, 8), np.float32)[:, ::2])
    with pytest.raises(ValueError, match="one value per item"):
        h.set_items(np.zeros((4, 8), np.float32), np.zeros(3, np.float32))
    with pytest.raises(ValueError, match="set the items before the queries"):
        h.set_queries(np.zeros((4, 8), np.float32))
    with pytest.raises(ValueError, match="query index out of range"):
        h.topk(np.array([0], np.int32), 3)
    h.close()
    h.close()


def test_native_state_and_argument_errors():
    """The C entry points check the call order and their arguments before they touch the device."""
    from buffalo_b200 import _cabi
    lib = _cabi.lib()
    h = lib.bfl_serve_create()
    q = np.zeros(2, np.int32)
    out = np.zeros((2, 3), np.int32)
    assert lib.bfl_serve_topk(h, q.ctypes.data, 2, 3, out.ctypes.data, None) == 3          # BFL_ERR_STATE
    assert lib.bfl_serve_set_queries(h, out.ctypes.data, 2, 3) == 3
    assert lib.bfl_serve_set_pool(h, q.ctypes.data, 2) == 3
    assert lib.bfl_serve_set_items(h, None, 4, 8, 8, None) == 4                            # BFL_ERR_ARG
    assert lib.bfl_serve_set_items(h, out.ctypes.data, 4, 4, 8, None) == 4                 # ld < d
    lib.bfl_serve_destroy(h)

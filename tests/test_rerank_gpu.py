"""MMR re-ranking on the device (csrc/rerank.cu, bfl_mmr_rerank_device, topk_recommendation(diversify=w), rerank_mmr)
against the fp64 reference (tests/rerank_ref.py): exact lists where every step has an objective gap, greedy validity
everywhere else, w = 0 bitwise equal to the plain result for every candidate stage, a known diversity answer, padding,
independence from the batch, and a production-size call."""
import functools

import numpy as np
import pytest
import scipy.sparse

from tests.rerank_ref import check_greedy, gap_inputs, mmr_ref, random_inputs
from tests.test_serve_cand_cpu import pool_matrix

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module", autouse=True)
def _release_cached_memory():
    """The production-size case leaves memory in torch's caching allocator: hand it back for the tests after this
    module."""
    yield
    import torch
    torch.cuda.empty_cache()


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def device_rerank(idx, val, F, k, w):
    import torch
    from buffalo_b200 import backend
    h = backend.Serve()
    try:
        h.set_items(np.ascontiguousarray(F, np.float32))
        ki, kv = h.rerank_mmr_device(torch.from_numpy(idx).cuda(), torch.from_numpy(val).cuda(), k, w)
        return ki.cpu().numpy(), kv.cpu().numpy()
    finally:
        h.close()


@functools.lru_cache(maxsize=None)
def _gap_case(d, M, w):
    return gap_inputs(2 if M > 200 else 4, M, d, w, seed=1000 * d + M)


@functools.lru_cache(maxsize=None)
def _random_case(d, M):
    return random_inputs(24, M, d, seed=7 * d + M)


DS = [4, 20, 100, 128, 200, 256]
MS = [1, 2, 31, 32, 33, 255, 256]
WS = [0.0, 0.3, 1.0]
CASES = [(M, k) for M in MS for k in sorted({1, min(10, M), M})]


@pytest.mark.parametrize("w", WS)
@pytest.mark.parametrize("M,k", CASES)
@pytest.mark.parametrize("d", DS)
def test_against_reference(cuda_lib, d, M, k, w):
    w = float(np.float32(w))
    idx, val, F = _gap_case(d, M, w)
    got = device_rerank(idx, val, F, k, w)
    want = mmr_ref(idx, val, F, k, w)
    np.testing.assert_array_equal(got[0], want[0])
    assert np.array_equal(bits(got[1]), bits(want[1]))
    idx, val, F = _random_case(d, M)
    keys, scores = device_rerank(idx, val, F, k, w)
    check_greedy(idx, val, F, w, keys, scores)
    # a shorter k is the prefix of the longer one: the steps do not look ahead
    full = device_rerank(idx, val, F, M, w)
    assert np.array_equal(keys, full[0][:, :k]) and np.array_equal(bits(scores), bits(full[1][:, :k]))


class _Data(object):
    """The "rowwise" group of a model's training data, as exclude_seen=True reads it."""

    def __init__(self, m):
        self.m = m.tocsr()

    def get_group(self, name):
        assert name == "rowwise"
        return {"indptr": np.asarray(self.m.indptr[1:], np.int64), "key": np.asarray(self.m.indices, np.int32)}


def _model(kind, U, I, d=32, seed=21):
    from tests.test_ivf_cpu import cpu_model
    m = cpu_model(kind, U=U, I=I, d=d, use_bias=True)
    rng = np.random.default_rng(seed)
    m.P = rng.standard_normal((U, d)).astype(np.float32)
    m.Q = rng.standard_normal((I, d)).astype(np.float32)
    m.data = _Data(scipy.sparse.random(U, I, density=0.02, format="csr", random_state=rng))
    return m


@pytest.mark.parametrize("kind", ["als", "bpr"])
def test_w0_is_the_plain_result_bitwise(cuda_lib, kind):
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    U, I = 3000, 4000
    m = _model(kind, U, I)
    par = (ParALS if kind == "als" else ParBPRMF)(m)
    rng = np.random.default_rng(3)
    rows = [rng.integers(0, I, size=int(x)).astype(np.int32) for x in rng.integers(0, 120, size=U)]
    rows[5] = np.zeros(0, np.int32)
    rows[6] = np.concatenate([rows[6][:4]] * 3)            # duplicates
    seen = scipy.sparse.random(U, I, density=0.05, format="csr", random_state=rng)
    users = np.concatenate([np.arange(0, U, 3), [5, 6]]).astype(np.int32)
    stages = [dict(), dict(pool=["i%d" % i for i in range(0, I, 7)]), dict(exclude_seen=True), dict(exclude_seen=seen),
              dict(pool=pool_matrix(rows, U, I)), dict(pool=pool_matrix(rows, U, I), exclude_seen=True)]
    for kw in stages:
        for k, M in ((10, None), (1, 7), (64, 256)):
            _, pk, ps = par.topk_recommendation(users, topk=k, **kw)
            _, dk, ds = par.topk_recommendation(users, topk=k, diversify=0.0, diversify_candidates=M, **kw)
            assert np.array_equal(dk, pk), kw
            assert np.array_equal(bits(ds), bits(ps)), kw


def _fold_model(I=3000, d=20):
    from tests.helpers import full_opt, init_factors
    from tests.test_fold_in_gpu import als_model
    return als_model(full_opt(d=d), np.zeros((1, d), np.float32), init_factors(I, d, d, 3, scale=0.1, signed=True))


def test_fold_in_w0_and_greedy(cuda_lib):
    from buffalo_b200.parallel.base import ParALS
    from tests.helpers import csr_from_lengths
    from tests.test_fold_in_gpu import history_lengths, to_matrix
    I, n = 3000, 200
    rng = np.random.default_rng(9)
    indptr, keys, vals = csr_from_lengths(history_lengths(rng, n, empty=3), I, rng)
    H = to_matrix(indptr, keys, vals, I)
    m = _fold_model(I)
    par = ParALS(m)
    rows = [rng.integers(0, I, size=int(x)).astype(np.int32) for x in rng.integers(0, 80, size=n)]
    rows[2] = np.zeros(0, np.int32)
    pool = rng.choice(I, 500, replace=False).astype(np.int32)
    for kw in (dict(exclude_seen=True), dict(exclude_seen=False), dict(pool=pool),
               dict(pool=pool_matrix(rows, n, I), exclude_seen=True)):
        pk, ps = par.fold_in_recommendation(H, topk=10, **kw)
        dk, ds = par.fold_in_recommendation(H, topk=10, diversify=0, **kw)
        assert np.array_equal(dk, pk) and np.array_equal(bits(ds), bits(ps)), kw
        assert "queries" not in par._serve._bound and par._serve.num_queries == 0
    # diversified: greedy over the plain candidates at k = M
    ck, cv = par.fold_in_recommendation(H, topk=40, exclude_seen=True)
    dk, ds = par.fold_in_recommendation(H, topk=10, exclude_seen=True, diversify=0.5, diversify_candidates=40)
    check_greedy(ck, cv, m.Q, 0.5, dk, ds)


def test_known_diversity_answer(cuda_lib):
    import buffalo_b200.evaluate as ev
    from buffalo_b200.parallel.base import ParALS
    from tests.test_ivf_cpu import cpu_model
    rng = np.random.default_rng(4)
    d, per, U = 8, 10, 16
    centers = np.eye(d, dtype=np.float32)[:4]
    Q = (np.repeat(centers, per, axis=0) + 0.01 * rng.standard_normal((4 * per, d))).astype(np.float32)
    m = cpu_model("als", U=U, I=4 * per, d=d)
    m.Q = Q
    m.P = np.tile(np.array([1.0, 0.8, 0.8, 0.8, 0, 0, 0, 0], np.float32), (U, 1))
    m.P += (0.01 * rng.standard_normal(m.P.shape)).astype(np.float32)
    par = ParALS(m)
    users = np.arange(U, dtype=np.int32)
    _, plain, _ = par.topk_recommendation(users, topk=4)
    _, div, _ = par.topk_recommendation(users, topk=4, diversify=0.7, diversify_candidates=4 * per)
    cluster = lambda k: k // per
    assert (cluster(plain) == 0).all()
    assert all(sorted(cluster(row).tolist()) == [0, 1, 2, 3] for row in div)
    test = scipy.sparse.csr_matrix(np.ones((U, 4 * per), np.float32))
    a = ev.evaluate_lists(plain, test, cutoffs=(4,), item_factors=Q)
    b = ev.evaluate_lists(div, test, cutoffs=(4,), item_factors=Q)
    assert b["ild@4"] > a["ild@4"] + 0.5


def test_padding_from_seen_rows_and_small_pools(cuda_lib):
    from buffalo_b200.parallel.base import ParALS
    from tests.test_ivf_cpu import cpu_model
    m = cpu_model("als", U=6, I=12, d=4)
    par = ParALS(m)
    seen = scipy.sparse.csr_matrix((np.ones(8), np.arange(8), [0, 8, 8, 8, 8, 8, 8]), shape=(6, 12))
    users = np.arange(6, dtype=np.int32)
    _, k1, s1 = par.topk_recommendation(users, topk=6, exclude_seen=seen, diversify=0.5, diversify_candidates=10)
    assert (k1[0, 4:] == -1).all() and (bits(s1[0, 4:]) == 0).all() and (k1[0, :4] >= 8).all()
    assert (k1[1:] >= 0).all()
    _, k2, s2 = par.topk_recommendation(users, topk=5, pool=["i1", "i4", "i9"], diversify=0.3)
    assert (k2[:, 3:] == -1).all() and (bits(s2[:, 3:]) == 0).all()
    assert all(sorted(r[:3].tolist()) == [1, 4, 9] for r in k2)


def test_independent_of_batch_position_and_run(cuda_lib, monkeypatch):
    from buffalo_b200.parallel import base, rerank_mmr
    from buffalo_b200 import backend
    idx, val, F = random_inputs(100000, 64, 32, seed=5, n_items=20000)
    w = float(np.float32(0.3))
    full = rerank_mmr(idx, val, F, 10, w)
    again = rerank_mmr(idx, val, F, 10, w)
    assert np.array_equal(full[0], again[0]) and np.array_equal(bits(full[1]), bits(again[1]))
    for r in (0, 1, 4242, 99999):
        one = rerank_mmr(idx[r:r + 1], val[r:r + 1], F, 10, w)
        assert np.array_equal(one[0][0], full[0][r]) and np.array_equal(bits(one[1][0]), bits(full[1][r]))
    monkeypatch.setattr(base, "RERANK_BATCH_BYTES", 8 * 64 * 777)          # 777 rows per batch
    small = rerank_mmr(idx, val, F, 10, w)
    assert np.array_equal(small[0], full[0]) and np.array_equal(bits(small[1]), bits(full[1]))
    # the device and NumPy paths agree on inputs whose every step has an objective gap
    gi, gv, gF = gap_inputs(6, 48, 20, w, seed=3)
    dev = rerank_mmr(gi, gv, gF, 20, w)
    monkeypatch.setattr(backend, "device_available", lambda: False)
    host = rerank_mmr(gi, gv, gF, 20, w)
    assert np.array_equal(dev[0], host[0]) and np.array_equal(bits(dev[1]), bits(host[1]))


def test_small_python_batches_in_topk_recommendation(cuda_lib, monkeypatch):
    from buffalo_b200.parallel import base
    m = _model("bpr", 5000, 3000)
    par = base.ParBPRMF(m)
    users = np.arange(5000, dtype=np.int32)
    want = par.topk_recommendation(users, topk=10, diversify=0.4, exclude_seen=True)
    monkeypatch.setattr(base, "RERANK_BATCH_BYTES", 8 * 40 * 333)
    got = par.topk_recommendation(users, topk=10, diversify=0.4, exclude_seen=True)
    assert np.array_equal(got[1], want[1]) and np.array_equal(bits(got[2]), bits(want[2]))


def test_production_size(cuda_lib):
    from buffalo_b200.parallel.base import ParALS
    from tests.test_ivf_cpu import cpu_model
    U, I, d = 131072, 100000, 128
    m = cpu_model("als", U=U, I=I, d=d)
    rng = np.random.default_rng(12)
    m.P = rng.standard_normal((U, d)).astype(np.float32)
    m.Q = rng.standard_normal((I, d)).astype(np.float32)
    par = ParALS(m)
    users = np.arange(U, dtype=np.int32)
    w = float(np.float32(0.3))
    _, keys, scores = par.topk_recommendation(users, topk=10, diversify=w, diversify_candidates=256)
    assert keys.shape == (U, 10) and (keys >= 0).all()
    sample = np.sort(rng.choice(U, 512, replace=False)).astype(np.int32)
    _, ck, cv = par.topk_recommendation(sample, topk=256)
    check_greedy(ck, cv, m.Q, w, keys[sample], scores[sample])

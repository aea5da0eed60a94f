"""Per-user candidate pools on the device (csrc/candidates.cu, bfl_cand_topk*, backend.Serve.topk_candidates*,
ParALS / ParBPRMF.topk_recommendation(pool=<sparse matrix>), fold_in_recommendation(pool=<sparse matrix>)): every row
is bitwise what the existing path returns for that row alone with its list as the pool (Serve.set_pool + topk, or
topk_seen with seen rows): same item ids, same score bits, same order."""
import numpy as np
import pytest
import scipy.sparse

from tests.test_serve_cand_cpu import pool_matrix
from tests.test_serve_gpu import bits, factors, make

pytestmark = pytest.mark.gpu


def csr(rows):
    ends = np.cumsum([len(r) for r in rows]).astype(np.int64)
    keys = np.concatenate([np.asarray(r, np.int32) for r in rows]) if ends.size and ends[-1] else np.zeros(0, np.int32)
    return ends, np.ascontiguousarray(keys, dtype=np.int32)


def per_row(h, qidx, rows, k, seen_rows=None):
    """The existing path, one call per row with the row as the pool; an empty row is -1 / 0.0."""
    keys = np.full((len(qidx), k), -1, np.int32)
    vals = np.zeros((len(qidx), k), np.float32)
    for i, (q, row) in enumerate(zip(qidx, rows)):
        if not len(row):
            continue
        h.set_pool(np.asarray(row, np.int32))
        if seen_rows is None:
            keys[i], vals[i] = (a[0] for a in h.topk(np.array([q], np.int32), k))
        else:
            s = np.ascontiguousarray(seen_rows[i], dtype=np.int32)
            keys[i], vals[i] = (a[0] for a in h.topk_seen(np.array([q], np.int32), k, np.array([s.size], np.int64), s))
    h.set_pool(None)
    return keys, vals


def assert_same(got, want):
    np.testing.assert_array_equal(got[0], want[0])
    np.testing.assert_array_equal(bits(got[1]), bits(want[1]))


def lengths_rows(I, k, seed):
    rng = np.random.default_rng(seed)
    lens = [0, 1, max(k - 1, 0), k, 1023, 1024, 1025, 2049]
    return [rng.integers(0, I, size=n).astype(np.int32) for n in lens]


@pytest.mark.parametrize("d", [1, 3, 4, 20, 64, 128, 200, 256, 300])
@pytest.mark.parametrize("k", [1, 10, 1024, 4096])
def test_bitwise_per_row(cuda_lib, d, k):
    I, n = 3000, 8
    P, Q, Qb = factors(n, I, d, d, seed=d * 7 + k, bias=(d + k) % 2 == 0)
    h = make(P, Q, Qb)
    rows = lengths_rows(I, k, d + k)
    qidx = np.arange(n, dtype=np.int32)[::-1].copy()
    got = h.topk_candidates(qidx, k, *csr(rows))
    assert_same(got, per_row(h, qidx, rows, k))
    rng = np.random.default_rng(d)
    seen = [np.concatenate([r[:len(r) // 3], rng.integers(0, I, size=5)]).astype(np.int32) for r in rows]
    got = h.topk_candidates(qidx, k, *csr(rows), seen=csr(seen))
    assert_same(got, per_row(h, qidx, rows, k, seen))


@pytest.mark.parametrize("k", [10, 1024])
def test_skewed_long_row(cuda_lib, k):
    I, d = 1_200_000, 128
    P, Q, Qb = factors(6, I, d, d, seed=5, bias=True)
    h = make(P, Q, Qb)
    rng = np.random.default_rng(6)
    rows = [rng.integers(0, I, size=3), rng.integers(0, I, size=1_000_000), rng.integers(0, I, size=3), [],
            rng.integers(0, I, size=2), rng.integers(0, I, size=3)]
    qidx = np.arange(6, dtype=np.int32)
    assert_same(h.topk_candidates(qidx, k, *csr(rows)), per_row(h, qidx, rows, k))


def test_ties_inf_and_unaligned_pitch(cuda_lib):
    I, d, ld = 4000, 20, 21
    P, Q, Qb = factors(5, I, ld, d, seed=9, bias=True)
    Q[1::2] = Q[0::2]                                # pairs of equal rows: ties broken by list position
    Qb[1::2] = Qb[0::2]
    Qb[::7] = -np.inf                                # -inf scores
    h = make(P, Q, Qb, d=d)
    rng = np.random.default_rng(10)
    rows = [rng.integers(0, I, size=n).astype(np.int32) for n in (40, 900, 1024, 3000, 7)]
    rows[0][1::2] = rows[0][0::2] ^ 1                # both rows of each pair in one list
    qidx = np.arange(5, dtype=np.int32)
    for k in (5, 64):
        assert_same(h.topk_candidates(qidx, k, *csr(rows)), per_row(h, qidx, rows, k))
        seen = [r[:3] for r in rows]
        assert_same(h.topk_candidates(qidx, k, *csr(rows), seen=csr(seen)), per_row(h, qidx, rows, k, seen))


@pytest.mark.parametrize("budget", [1, 1023, 1024, 1025, 5000])
def test_batch_edges_host_equals_device(cuda_lib, budget):
    import torch
    I, d, n, k = 5000, 64, 300, 16
    P, Q, Qb = factors(n, I, d, d, seed=11, bias=False)
    h = make(P, Q, Qb)
    rng = np.random.default_rng(12)
    rows = [rng.integers(0, I, size=int(m)).astype(np.int32) for m in rng.integers(0, 60, size=n)]
    rows[17] = rng.integers(0, I, size=3000).astype(np.int32)
    seen = [r[::4] for r in rows]
    qidx = rng.permutation(n).astype(np.int32)
    want = h.topk_candidates(qidx, k, *csr(rows), seen=csr(seen))
    h._set_cand_budget(budget)
    try:
        assert_same(h.topk_candidates(qidx, k, *csr(rows), seen=csr(seen)), want)
    finally:
        h._set_cand_budget(0)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    # the device entry reads rows through cand_row / seen_row: reversed CSRs, row n - 1 - i for query i
    cptr, ckeys = csr(rows[::-1])
    sptr, skeys = csr(seen[::-1])
    rrow = t(np.arange(n - 1, -1, -1, dtype=np.int32))
    idx, val = h.topk_candidates_device(t(qidx), k, t(cptr), t(ckeys), cand_row=rrow, seen=(t(sptr), t(skeys), rrow))
    torch.cuda.synchronize()
    assert_same((idx.cpu().numpy(), val.cpu().numpy()), want)
    assert_same(per_row(h, qidx[:20], rows[:20], k, seen[:20]), (want[0][:20], want[1][:20]))


def _model(kind, U, I, d=32):
    from tests.test_ivf_cpu import cpu_model
    m = cpu_model(kind, U=U, I=I, d=d, use_bias=True)
    rng = np.random.default_rng(21)
    m.P = rng.standard_normal((U, d)).astype(np.float32)
    m.Q = rng.standard_normal((I, d)).astype(np.float32)
    return m


@pytest.mark.parametrize("kind", ["als", "bpr"])
def test_par_many_users_equal_per_user_calls(cuda_lib, kind):
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    U, I = 131072, 20000
    par = (ParALS if kind == "als" else ParBPRMF)(_model(kind, U, I))
    rng = np.random.default_rng(22)
    lens = np.minimum(rng.zipf(1.5, size=U) * 10, 5000)
    lens[::97] = 0
    ptr = np.concatenate([[0], np.cumsum(lens)]).astype(np.int64)
    M = scipy.sparse.csr_matrix((np.ones(ptr[-1], np.float32), rng.integers(0, I, size=ptr[-1]).astype(np.int32), ptr),
                                shape=(U, I))
    S = pool_matrix([rng.integers(0, I, size=40) for _ in range(U)], U, I)
    users = np.arange(U, dtype=np.int32)
    for seen in (False, S):
        kept, keys, vals = par.topk_recommendation(users, topk=10, pool=M, exclude_seen=seen)
        assert keys.shape == (U, 10)
        for u in rng.choice(U, size=64, replace=False).tolist() + [0, 97]:
            row = M.indices[M.indptr[u]:M.indptr[u + 1]]
            if not row.size:
                assert (keys[u] == -1).all() and (bits(vals[u]) == 0).all()
                continue
            _, k1, v1 = par.topk_recommendation(np.array([u], np.int32), topk=10, pool=row.astype(np.int32),
                                                exclude_seen=seen)
            np.testing.assert_array_equal(keys[u], k1[0])
            np.testing.assert_array_equal(bits(vals[u]), bits(v1[0]))
    ids = ["u%d" % u for u in (3, 5, 97)]
    _, names, _ = par.topk_recommendation(ids, topk=10, pool=M, repr=True)
    _, want, _ = par.topk_recommendation(np.array([3, 5, 97], np.int32), topk=10, pool=M)
    assert names == [["i%d" % t for t in row if t != -1] for row in want]


def test_fold_in_recommendation_pool_matrix(cuda_lib):
    from buffalo_b200 import backend
    from buffalo_b200.parallel.base import ParALS
    from tests.helpers import csr_from_lengths, full_opt, init_factors
    from tests.test_fold_in_gpu import als_model, history_lengths, to_matrix
    d, I, n, topk = 20, 5000, 300, 50
    rng = np.random.default_rng(5)
    indptr, keys, vals = csr_from_lengths(history_lengths(rng, n, empty=3), I, rng)
    H = to_matrix(indptr, keys, vals, I)
    m = als_model(full_opt(d=d), np.zeros((1, d), np.float32), init_factors(I, d, d, 3, scale=0.1, signed=True))
    rows = [rng.integers(0, I, size=int(x)).astype(np.int32) for x in rng.integers(0, 900, size=n)]
    rows[4] = np.zeros(0, np.int32)
    par = ParALS(m)
    for excl in (True, False):
        got = par.fold_in_recommendation(H, topk=topk, pool=pool_matrix(rows, n, I), exclude_seen=excl)
        assert "queries" not in par._serve._bound and par._serve.num_queries == 0
        # fold_in followed by per-row calls on a host copy of the folded rows (padded to the device row pitch)
        X = m.fold_in(H)
        h = backend.Serve()
        h.set_items(np.ascontiguousarray(m.Q, dtype=np.float32))
        vdim = m._fold_state.holder.get_vdim()
        Xp = np.zeros((n, vdim), np.float32)
        Xp[:, :d] = X
        h.set_queries(Xp)
        beg = np.concatenate([[0], indptr[:-1]])
        seen = [keys[beg[r]:indptr[r]] for r in range(n)] if excl else None
        assert_same(got, per_row(h, np.arange(n, dtype=np.int32), rows, topk, seen))
    m._idmanager.itemids = ["i%d" % i for i in range(I)]
    names, _ = par.fold_in_recommendation(H, topk=topk, pool=pool_matrix(rows, n, I), exclude_seen=False,
                                          repr=True)
    assert names[4] == [] and names[0] == [m._idmanager.itemids[t] for t in got[0][0] if t != -1]


def test_close_returns_memory(cuda_lib):
    import torch
    I, d = 200000, 128
    P, Q, _ = factors(4096, I, d, d, seed=41, bias=False)
    rng = np.random.default_rng(42)
    rows = [rng.integers(0, I, size=500).astype(np.int32) for _ in range(4096)]
    warm = make(P, Q, None)
    warm.topk_candidates(np.arange(4096, dtype=np.int32), 10, *csr(rows))
    warm.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    h = make(P, Q, None)
    h.topk_candidates(np.arange(4096, dtype=np.int32), 10, *csr(rows), seen=csr([r[:5] for r in rows]))
    h.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert torch.cuda.mem_get_info()[0] >= free0 - (4 << 20)

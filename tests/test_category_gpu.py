"""Per-category caps on the device (csrc/category.cu, bfl_category_walk_device, topk_recommendation /
fold_in_recommendation / most_similar with categories, cap_categories): bitwise the plain walk of tests/category_ref.py
over the same call's complete unconstrained ranking in every serving mode, exact through several deepening rounds on
adversarial layouts, independent of the first depth, the batch split and the other rows, items of add_items capped,
and the plain call unchanged around a capped one."""
import copy

import numpy as np
import pytest
import scipy.sparse

from tests import category_ref
from tests.test_serve_cand_cpu import pool_matrix

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


def same(got, want):
    return np.array_equal(got[0], want[0]) and np.array_equal(bits(got[1]), bits(want[1]))


class _Data(object):
    def __init__(self, m):
        self.m = m.tocsr()

    def get_group(self, name):
        assert name == "rowwise"
        return {"indptr": np.asarray(self.m.indptr[1:], np.int64), "key": np.asarray(self.m.indices, np.int32)}


def int_model(kind, U, I, d=8, seed=3, hi=3):
    """Small-integer factors (and bias): every fp32 score is exact, so NumPy's stable order is the device order."""
    from tests.test_ivf_cpu import cpu_model
    m = cpu_model(kind, U=U, I=I, d=d, use_bias=True)
    rng = np.random.default_rng(seed)
    m.P = rng.integers(-hi, hi + 1, (U, d)).astype(np.float32)
    m.Q = rng.integers(-hi, hi + 1, (I, d)).astype(np.float32)
    if kind == "bpr":
        m.Qb = rng.integers(-2, 3, (I, 1)).astype(np.float32)
    m.data = _Data(scipy.sparse.random(U, I, density=0.02, format="csr", random_state=rng))
    return m


def par_of(m, kind):
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    return (ParALS if kind == "als" else ParBPRMF)(m)


def capped_vs_full(call, cats, cap, topk, depth, **kw):
    """call(topk, **kw) -> (keys, scores); the capped call against the walk of the unconstrained call at depth."""
    got = call(topk, categories=cats, category_cap=cap, **kw)
    full = call(depth, **kw)
    want = category_ref.walk(full[0], full[1], cats, cap, topk)
    assert same(got, want), (kw, cap, topk)
    return got


@pytest.mark.parametrize("kind", ["als", "bpr"])
def test_bitwise_against_the_complete_ranking(cuda_lib, kind):
    U, I = 400, 3000
    m = int_model(kind, U, I, d=16, seed=11)
    m.P = np.random.default_rng(1).standard_normal((U, 16)).astype(np.float32)   # general fp32 scores too
    par = par_of(m, kind)
    rng = np.random.default_rng(5)
    users = np.concatenate([rng.choice(U, 90, replace=False), [7, 7]]).astype(np.int32)
    cats = rng.integers(-1, 40, I)
    cats[rng.choice(I, 600, replace=False)] = 3                 # one large category
    per_cat = rng.integers(0, 4, 40)
    rows = [rng.choice(I, int(n), replace=False) for n in rng.integers(0, 900, U)]
    rows[users[0]] = np.zeros(0, np.int64)
    per_user = pool_matrix(rows, U, I)
    pool = rng.choice(I, 1500, replace=False).astype(np.int32)
    seen = scipy.sparse.random(U, I, density=0.05, format="csr", random_state=rng)

    def call(k, **kw):
        _, keys, scores = par.topk_recommendation(users, k, **kw)
        return keys, scores
    for kw, depth in [(dict(), I), (dict(pool=pool), len(pool)), (dict(exclude_seen=True), I),
                      (dict(exclude_seen=seen), I), (dict(pool=per_user), 900),
                      (dict(pool=per_user, exclude_seen=True), 900), (dict(pool=pool, exclude_seen=seen), len(pool))]:
        for cap, topk in [(1, 10), (2, 50), (per_cat, 10), (0, 20), (1, 1000)]:
            capped_vs_full(call, cats, cap, topk, depth, **kw)
    # most_similar on the normalized item rows
    items = rng.choice(I, 40, replace=False).astype(np.int32)
    capped_vs_full(lambda k, **kw: par.most_similar(items, k, **kw), cats, 1, 10, I)
    capped_vs_full(lambda k, **kw: par.most_similar(items, k, **kw), cats, per_cat, 30, I, pool=pool)


def trained_als(seed=31):
    from tests.test_explore_gpu import trained
    return trained(seed=seed)


def test_explore_and_fold_in_against_the_complete_ranking(cuda_lib):
    from buffalo_b200.parallel.base import ParALS
    from tests.helpers import csr_from_lengths
    from tests.test_explain_gpu import to_matrix
    m, rng, R = trained_als()
    U, I = m.P.shape[0], m.Q.shape[0]
    par = ParALS(m)
    cats = rng.integers(-1, 25, I)
    users = rng.choice(U, 100, replace=False).astype(np.int32)
    per_user = scipy.sparse.random(U, I, density=0.3, format="csr", random_state=rng)
    for kw, depth in [(dict(), I), (dict(exclude_seen=True), I), (dict(pool=per_user), int(np.diff(per_user.indptr).max()))]:
        def call(k, **kw2):
            _, keys, scores = par.topk_recommendation(users, k, explore=0.7, explore_seed=99, **kw2)
            return keys, scores
        capped_vs_full(call, cats, 1, 10, depth, **kw)
        capped_vs_full(call, cats, 2, 40, depth, **kw)
    hi, hk, hv = csr_from_lengths(rng.integers(0, 40, 70), I, rng)
    H = to_matrix(hi, hk, hv, I)
    pool = rng.choice(I, 800, replace=False).astype(np.int32)
    for kw, depth in [(dict(), I), (dict(exclude_seen=False), I), (dict(pool=pool), len(pool)),
                      (dict(explore=0.5, explore_seed=3), I)]:
        capped_vs_full(lambda k, **kw2: par.fold_in_recommendation(H, k, **kw2), cats, 1, 10, depth, **kw)


def adversarial(kind, U=48, I=20000, seed=7):
    """Items 0..2999 score highest for every user (category 0, cap 1), the next 6000 next (category 1, banned); the
    rest in categories 2..49 with cap 2, a tenth uncapped.  A capped row walks past 9000 items: several rounds."""
    m = int_model(kind, U, I, d=8, seed=seed, hi=2)
    m.P[:, 0] = 4
    m.Q[:3000, 0] = 9
    m.Q[3000:9000, 0] = 6
    rng = np.random.default_rng(seed)
    cats = rng.integers(2, 50, I)
    cats[rng.random(I) < 0.1] = -1
    cats[:3000], cats[3000:9000] = 0, 1
    caps = np.full(50, 2)
    caps[0], caps[1] = 1, 0
    return m, cats, caps


def numpy_full(m, users, kind, seen=None, pool=None):
    """(keys, scores) of the complete ranking in NumPy: exact integer scores, stable order (ties to the smaller id or the
    earlier pool entry)."""
    cand = np.arange(m.Q.shape[0]) if pool is None else np.asarray(pool)
    s = m.P[users] @ m.Q[cand].T
    if kind == "bpr":
        s = s + m.Qb[cand, 0][None]
    s = s.astype(np.float32)
    keys = np.empty(s.shape, np.int64)
    vals = np.empty(s.shape, np.float32)
    for r in range(len(users)):
        o = np.argsort(-s[r], kind="stable")
        if seen is not None:
            o = o[~np.isin(cand[o], seen[r])]
        keys[r, :len(o)], vals[r, :len(o)] = cand[o], s[r, o]
        keys[r, len(o):], vals[r, len(o):] = -1, 0
    return keys, vals


@pytest.mark.parametrize("kind", ["als", "bpr"])
def test_deepening_on_adversarial_layouts(cuda_lib, kind):
    from buffalo_b200.parallel import base
    m, cats, caps = adversarial(kind)
    par = par_of(m, kind)
    U, I = m.P.shape[0], m.Q.shape[0]
    users = np.arange(U, dtype=np.int32)
    rng = np.random.default_rng(2)
    seen = scipy.sparse.random(U, I, density=0.05, format="csr", random_state=rng)
    seen_rows = [seen.indices[seen.indptr[u]:seen.indptr[u + 1]] for u in range(U)]
    pool = rng.choice(I, 15000, replace=False).astype(np.int32)
    stats = []
    real = base._capped_batches
    base._capped_batches = lambda *a, **k: real(*a, **dict(k, stats=stats))
    try:
        for kw, full in [(dict(), numpy_full(m, users, kind)),
                         (dict(exclude_seen=seen), numpy_full(m, users, kind, seen=seen_rows)),
                         (dict(pool=pool), numpy_full(m, users, kind, pool=pool))]:
            for cap, topk in [(caps, 10), (caps, 60), (1, 10)]:
                _, keys, scores = par.topk_recommendation(users, topk, categories=cats, category_cap=cap, **kw)
                want = category_ref.walk(full[0], full[1], cats, cap, topk)
                assert same((keys, scores), want), (kw, topk)
    finally:
        base._capped_batches = real
    assert max(r for r, _, _ in stats) >= 3                   # the layouts forced several rounds


def test_independent_of_depth_batch_and_neighbours(cuda_lib, monkeypatch):
    from buffalo_b200.parallel import base
    m, cats, caps = adversarial("bpr", U=12)
    par = par_of(m, "bpr")
    users = np.array([3, 0, 11, 5, 5, 8, 1], np.int32)
    ref = par.topk_recommendation(users, 12, categories=cats, category_cap=caps, exclude_seen=True)
    for m0, batch in [(1, 1), (7, 3 << 16), (None, 1), (7, 1 << 40)]:
        monkeypatch.setattr(base, "CATEGORY_M0", m0)
        monkeypatch.setattr(base, "CATEGORY_BATCH_BYTES", batch)
        got = par.topk_recommendation(users, 12, categories=cats, category_cap=caps, exclude_seen=True)
        assert same(got[1:], ref[1:]), (m0, batch)
    monkeypatch.setattr(base, "CATEGORY_M0", None)
    monkeypatch.setattr(base, "CATEGORY_BATCH_BYTES", 1 << 30)
    for i, u in enumerate(users):
        alone = par.topk_recommendation(np.array([u], np.int32), 12, categories=cats, category_cap=caps,
                                        exclude_seen=True)
        assert same((alone[1][0], alone[2][0]), (ref[1][i], ref[2][i])), u


def test_add_items_are_capped(cuda_lib):
    m = int_model("als", 60, 500, seed=4)
    par = par_of(m, "als")
    users = np.arange(60, dtype=np.int32)
    new = np.tile(np.full((1, 8), 3, np.float32), (40, 1))      # score high for users with a positive row sum
    m.add_items(["n%d" % i for i in range(40)], new)
    rng = np.random.default_rng(0)
    cats = np.concatenate([rng.integers(-1, 10, 500), np.full(40, 10)])
    with pytest.raises(ValueError, match="one entry per item"):
        par.topk_recommendation(users, 10, categories=cats[:500], category_cap=1)
    got = capped_vs_full(lambda k, **kw: par.topk_recommendation(users, k, **kw)[1:], cats, 1, 10, 540)
    assert (np.isin(got[0], np.arange(500, 540)).sum(axis=1) <= 1).all()
    assert np.isin(got[0], np.arange(500, 540)).any()


def test_plain_call_unchanged_around_a_capped_one(cuda_lib):
    m = int_model("bpr", 200, 2000, seed=8)
    par = par_of(m, "bpr")
    users = np.arange(0, 200, 3, dtype=np.int32)
    cats = np.random.default_rng(1).integers(-1, 30, 2000)
    for kw in (dict(), dict(exclude_seen=True), dict(pool=np.arange(0, 2000, 3, dtype=np.int32))):
        before = par.topk_recommendation(users, 25, **kw)
        par.topk_recommendation(users, 25, categories=cats, category_cap=1, **kw)
        after = par.topk_recommendation(users, 25, **kw)
        assert same(before[1:], after[1:]), kw


def test_cap_categories_on_the_device(cuda_lib, monkeypatch):
    from buffalo_b200 import backend
    from buffalo_b200.parallel.base import cap_categories
    rng = np.random.default_rng(12)
    I, n, M = 5000, 700, 300
    cats = rng.integers(-1, 40, I)
    idx = rng.integers(0, I, (n, M)).astype(np.int32)
    idx[rng.random((n, M)) < 0.1] = -1
    val = rng.standard_normal((n, M)).astype(np.float32)
    for cap, topk in [(1, 10), (0, 5), (3, 100), (rng.integers(0, 5, 40), 50), (2, 400)]:
        got = cap_categories(idx, val, cats, cap, topk)
        assert same(got, category_ref.walk(idx, val, cats, cap, topk)), (topk,)
    # the kernel's walk state carries over between calls on consecutive parts of a list
    import torch
    topk, slots = 64, backend.category_table_slots(64)
    state = torch.zeros((n, 1 + 2 * slots), dtype=torch.int32, device="cuda")
    oi = torch.full((n, topk), -1, dtype=torch.int32, device="cuda")
    ov = torch.zeros((n, topk), dtype=torch.float32, device="cuda")
    tc = torch.from_numpy(cats.astype(np.int32)).cuda()
    for a, b in [(0, 1), (1, 33), (33, 100), (100, M)]:
        backend.category_walk_device(torch.from_numpy(np.ascontiguousarray(idx[:, a:b])).cuda(),
                                     torch.from_numpy(np.ascontiguousarray(val[:, a:b])).cuda(), None, tc, 2, topk,
                                     state, oi, ov)
    assert same((oi.cpu().numpy(), ov.cpu().numpy()), category_ref.walk(idx, val, cats, 2, topk))

"""ALS explanations on the GPU (DESIGN.md 4.11): ALS.explain against the fp64 reference (tests/explain_ref.py), the sum
identity, agreement with the llt fold-in, batch independence, ParALS.explain on trained users, failure isolation, the
item-factor cache rules and a production-sized call."""
import numpy as np
import pytest
import scipy.sparse

from tests import explain_ref
from tests.helpers import csr_from_lengths, full_opt, init_factors

pytestmark = pytest.mark.gpu


def to_matrix(indptr, keys, vals, num_items):
    return scipy.sparse.csr_matrix((vals, keys, np.concatenate([[0], indptr])), shape=(len(indptr), num_items))


def als_model(opt, Q):
    from buffalo_b200.algo.als import ALS
    from buffalo_b200.algo.options import ALSOption
    o = ALSOption().get_default_option()
    o.update(opt)
    m = ALS(o)
    m.P, m.Q = np.zeros((1, Q.shape[1]), np.float32), Q.copy()
    return m


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def same(a, b):
    return all(x.shape == y.shape and np.array_equal(bits(x), bits(y)) for x, y in zip(a, b))


def random_targets(rng, n, k, num_items, none=0.2):
    T = rng.integers(0, num_items, (n, k)).astype(np.int32)
    T[rng.random((n, k)) < none] = -1
    return T


def check_rows(got, ref, Q, targets, rows=None):
    """Scores within 1e-3 |x_ref| |q_i|; contributions within 1e-3 of the row-target's largest |contribution|; keys equal
    wherever the reference contribution is more than that apart from its neighbours; -1 / 0.0 padding exact."""
    scores, keys, contrib = got
    topm = keys.shape[2]
    for j, res in enumerate(ref):
        r = j if rows is None else rows[j]
        for t, i in enumerate(targets[r]):
            if res["x"] is None or i < 0:
                assert scores[r, t] == 0 and (keys[r, t] == -1).all() and (contrib[r, t] == 0).all(), (r, t)
                continue
            qn = np.linalg.norm(Q[i].astype(np.float64))
            assert abs(scores[r, t] - res["scores"][t]) <= 1e-3 * np.linalg.norm(res["x"]) * qn + 1e-30, (r, t)
            items, c = res["ranked"][t]
            tol = 1e-3 * np.abs(c).max()
            m = min(topm, len(items))
            assert (keys[r, t, m:] == -1).all() and (contrib[r, t, m:] == 0).all(), (r, t)
            assert np.abs(contrib[r, t, :m] - c[:m]).max() <= tol, (r, t)
            gap = np.abs(np.diff(c))
            for p in range(m):
                clear = (p == 0 or gap[p - 1] > tol) and (p + 1 >= len(c) or gap[p] > tol)
                if clear:
                    assert keys[r, t, p] == items[p], (r, t, p, keys[r, t], items[:m])


def problem(d, seed, n=48, I=8000, vals="ints", long_rows=(5200,)):
    """histories of 1..300 entries plus `long_rows`, three empty rows; signed item factors of moderate size (DESIGN §2)"""
    rng = np.random.default_rng(seed)
    lengths = np.concatenate([[1, 2], rng.integers(1, 300, n - 5 - len(long_rows)), long_rows, [0, 0, 0]])
    rng.shuffle(lengths)
    fractional = lambda g, m: g.random(m) * 4.0 + 0.05
    indptr, keys, vals = csr_from_lengths(lengths, I, rng, vals=fractional if vals == "fractional" else "ints")
    Q = init_factors(I, d, d, seed + 1, scale=0.1, signed=True)
    return rng, indptr, keys, vals, Q, I


@pytest.mark.parametrize("alpha", [8.0, 0.5])
@pytest.mark.parametrize("adaptive_reg", [False, True])
@pytest.mark.parametrize("d", [5, 20, 32, 64, 100, 128, 200, 256])
def test_against_fp64_reference(cuda_lib, d, adaptive_reg, alpha):
    rng, indptr, keys, vals, Q, I = problem(d, d + int(adaptive_reg) * 7, vals="fractional" if alpha < 1 else "ints")
    opt = full_opt(d=d, optimizer="llt" if d < 128 else "ialspp", alpha=alpha, adaptive_reg=adaptive_reg)
    targets = random_targets(rng, len(indptr), 10, I)
    topm = 5 if d % 2 else 8
    got = als_model(opt, Q).explain(to_matrix(indptr, keys, vals, I), targets, topm=topm)
    assert got[0].dtype == np.float32 and got[1].dtype == np.int32 and got[2].dtype == np.float32
    assert got[0].shape == targets.shape and got[1].shape == got[2].shape == targets.shape + (topm,)
    ref = explain_ref.explain_rows(Q, indptr, keys, vals, targets, topm, alpha, opt["reg_u"], adaptive_reg)
    check_rows(got, ref, Q, targets)


@pytest.mark.parametrize("d", [20, 128])
def test_list_input_with_duplicates(cuda_lib, d):
    """items and histories as id lists: duplicate history items are summed into one contribution, unknown targets -1"""
    rng = np.random.default_rng(40 + d)
    I = 2000
    Q = init_factors(I, d, d, 9, scale=0.1, signed=True)
    m = als_model(full_opt(d=d), Q)
    ids = ["item%d" % i for i in range(I)]
    m._idmanager.itemids, m._idmanager.itemid_map, m._idmanager.itemid_mapped = ids, {v: i for i, v in enumerate(ids)}, True
    rows = [rng.integers(0, 40, rng.integers(1, 90)).tolist() for _ in range(30)]   # many repeats
    rows[4] = []
    hist = [[ids[i] for i in r] for r in rows]
    tlists = [[ids[i] for i in rng.integers(0, I, rng.integers(0, 7))] + (["nope"] if j % 4 == 0 else [])
              for j in range(30)]
    got = m.explain(hist, tlists, topm=6)
    lens = np.array([len(r) for r in rows])
    indptr = np.cumsum(lens).astype(np.int64)
    keys = np.concatenate([np.sort(r) for r in rows]).astype(np.int32)
    from buffalo_b200.algo import fold_in
    targets = fold_in.target_matrix(m, tlists, 30, I, 4096)
    assert targets.shape[1] == max(len(t) for t in tlists)
    assert got[0].shape == targets.shape
    ref = explain_ref.explain_rows(Q, indptr, keys, np.ones(len(keys), np.float32), targets, 6, 8.0, 0.1, False)
    check_rows(got, ref, Q, targets)
    # no item appears twice among a row-target's keys
    for kk in got[1].reshape(-1, 6):
        kk = kk[kk >= 0]
        assert len(kk) == len(set(kk.tolist()))


@pytest.mark.parametrize("d", [32, 128])
def test_contributions_sum_to_the_score(cuda_lib, d):
    rng = np.random.default_rng(70 + d)
    I = 4000
    indptr, keys, vals = csr_from_lengths(rng.integers(1, 65, 60), I, rng)
    Q = init_factors(I, d, d, 5, scale=0.1, signed=True)
    targets = random_targets(rng, 60, 12, I, none=0.0)
    scores, out_keys, contrib = als_model(full_opt(d=d), Q).explain(to_matrix(indptr, keys, vals, I), targets, topm=64)
    assert (out_keys >= 0).sum(axis=2).min() >= 1
    total = contrib.astype(np.float64).sum(axis=2)
    assert (np.abs(total - scores) <= 1e-4 * np.abs(contrib.astype(np.float64)).sum(axis=2)).all()


@pytest.mark.parametrize("d", [5, 20, 64, 100])
def test_agrees_with_llt_fold_in(cuda_lib, d):
    rng, indptr, keys, vals, Q, I = problem(d, 300 + d, n=80, long_rows=(1500,))
    m = als_model(full_opt(d=d, optimizer="llt"), Q)
    H = to_matrix(indptr, keys, vals, I)
    targets = random_targets(rng, len(indptr), 10, I, none=0.0)
    scores, _, _ = m.explain(H, targets)
    X = m.fold_in(H, sweeps=1).astype(np.float64)
    lens = np.diff(np.concatenate([[0], indptr]))
    for r in np.flatnonzero(lens):
        q = Q[targets[r]].astype(np.float64)
        want = q @ X[r]
        tol = 1e-4 * np.linalg.norm(X[r]) * np.linalg.norm(q, axis=1)
        assert (np.abs(scores[r] - want) <= tol).all(), r


def test_batch_independence(cuda_lib):
    """a row's outputs are bitwise the same whatever rows share its call and in whatever order"""
    d = 64
    rng, indptr, keys, vals, Q, I = problem(d, 11, n=90)
    m = als_model(full_opt(d=d), Q)
    H = to_matrix(indptr, keys, vals, I)
    targets = random_targets(rng, H.shape[0], 20, I)
    whole = m.explain(H, targets, topm=7)
    cuts = [0, 1, 37, 60, H.shape[0]]
    parts = [m.explain(H[a:b], targets[a:b], topm=7) for a, b in zip(cuts[:-1], cuts[1:])]
    assert same(whole, [np.concatenate(x) for x in zip(*parts)])
    perm = rng.permutation(H.shape[0])
    shuffled = m.explain(H[perm], targets[perm], topm=7)
    assert same([x[perm] for x in whole], shuffled)


class _Data(object):
    """The part of a database ALS.train() and ParALS.explain read: header and the two CSR groups."""

    def __init__(self, U, I, indptr, keys, vals):
        from tests.helpers import transpose_csr
        cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
        self.header = {"num_users": U, "num_items": I, "num_nnz": len(keys)}
        self.groups = {"rowwise": {"indptr": indptr, "key": keys, "val": vals},
                       "colwise": {"indptr": cind, "key": ckeys, "val": cvals}}

    def get_header(self):
        return self.header

    def get_group(self, name):
        return self.groups[name]


def test_par_als_explain_matches_als_explain(cuda_lib):
    from buffalo_b200.misc import aux
    from buffalo_b200.parallel.base import ParALS
    U, I, d = 400, 1500, 20
    rng = np.random.default_rng(21)
    indptr, keys, vals = csr_from_lengths(rng.integers(1, 120, U), I, rng)
    m = als_model(full_opt(d=d, num_iters=2, random_seed=3), np.zeros((1, d), np.float32))
    m.data = _Data(U, I, indptr, keys, vals)
    m.initialize()
    m.train()
    m._idmanager = aux.Option({"userids": ["u%d" % i for i in range(U)], "itemids": ["i%d" % i for i in range(I)],
                               "userid_mapped": True, "itemid_mapped": True})
    m._idmanager.userid_map = {v: i for i, v in enumerate(m._idmanager.userids)}
    m._idmanager.itemid_map = {v: i for i, v in enumerate(m._idmanager.itemids)}
    par = ParALS(m)
    users = ["u0"] + ["u%d" % u for u in rng.choice(np.arange(1, U), 49, replace=False)]
    pool = keys[:min(6, int(indptr[0]))].tolist() + rng.choice(I, 6, replace=False).tolist()
    kept, topks, _ = par.topk_recommendation(users, 10, pool=["i%d" % p for p in pool], exclude_seen=True)
    assert kept == users and (topks[0] == -1).any()        # u0's seen pool items leave -1 padding
    got = par.explain(kept, topks)
    H = to_matrix(indptr, keys, vals, I)[[int(u[1:]) for u in users]]
    want = m.explain(H, topks)
    assert same(got, want)
    assert (got[1][topks < 0] == -1).all() and (got[0][topks < 0] == 0).all()
    # index keys and item ids without the padding
    s, named, c = par.explain(np.array([int(u[1:]) for u in users]), topks, repr=True)
    assert same((s, c), (want[0], want[2]))
    assert named == [[["i%d" % x for x in kk if x != -1] for kk in row] for row in want[1]]


def test_failed_factorisation_is_isolated(cuda_lib):
    """reg_u = 0 and an exactly zero last column of Q: every history row meets the pivot 0 exactly and gets NaN scores
    and -1 keys; a row made indefinite by negative values fails alone while its neighbours match the reference"""
    d, I = 20, 1000
    rng = np.random.default_rng(5)
    indptr, keys, vals = csr_from_lengths(rng.integers(1, 50, 12), I, rng)
    indptr = np.concatenate([indptr[:3], [indptr[2]], indptr[3:]])            # an empty row at 3
    H = to_matrix(indptr, keys, vals, I)
    targets = random_targets(rng, H.shape[0], 5, I)
    targets[0, 0] = -1
    Q = init_factors(I, d, d, 6, scale=0.1, signed=True)
    Q0 = Q.copy()
    Q0[:, -1] = 0
    scores, out_keys, contrib = als_model(full_opt(d=d, reg_u=0.0), Q0).explain(H, targets)
    valid = targets >= 0
    valid[3] = False
    assert np.isnan(scores[valid]).all() and (scores[~valid] == 0).all()
    assert (out_keys == -1).all() and (contrib == 0).all()
    # negative values make one row's A indefinite
    v = vals.copy()
    v[indptr[5] - 1] = -500.0
    H = to_matrix(indptr, keys, v, I)
    got = als_model(full_opt(d=d), Q).explain(H, targets)
    assert np.isnan(got[0][5][targets[5] >= 0]).all() and (got[1][5] == -1).all()
    rows = [r for r in range(H.shape[0]) if r != 5]
    ref = explain_ref.explain_rows(Q, indptr, keys, v, targets, 5, 8.0, 0.1, False, rows=rows)
    check_rows(got, ref, Q, targets, rows=rows)


def test_item_factor_cache_rules(cuda_lib):
    d = 32
    rng, indptr, keys, vals, Q, I = problem(d, 17, n=30, long_rows=())
    m = als_model(full_opt(d=d), Q)
    H = to_matrix(indptr, keys, vals, I)
    targets = random_targets(rng, H.shape[0], 8, I)
    before = m.explain(H, targets)
    m.Q[::7] *= 1.5                                   # in place: the next call uploads Q and recomputes its Gram
    after = m.explain(H, targets)
    assert not same(before, after)
    check_rows(after, explain_ref.explain_rows(m.Q, indptr, keys, vals, targets, 5, 8.0, 0.1, False), m.Q, targets)
    m.normalize("item")
    with pytest.raises(RuntimeError, match="normalized"):
        m.explain(H, targets)


def test_production_scale(cuda_lib):
    """131072 Pareto-length histories (mean about 50) x k = 10 x topm = 5 at 1M items and d = 128; a seeded sample of
    256 rows against the reference"""
    n, I, d = 131072, 1000000, 128
    rng = np.random.default_rng(2026)
    lengths = np.minimum(np.ceil((rng.pareto(2.0, n) + 1.0) * 25.0), 5000).astype(np.int64)
    keys = rng.integers(0, I, int(lengths.sum()), dtype=np.int32)
    vals = rng.integers(1, 6, len(keys)).astype(np.float32)
    H = scipy.sparse.csr_matrix((vals, keys, np.concatenate([[0], np.cumsum(lengths)])), shape=(n, I))
    Q = (rng.standard_normal((I, d), dtype=np.float32) * 0.1).astype(np.float32)
    targets = rng.integers(0, I, (n, 10)).astype(np.int32)
    got = als_model(full_opt(d=d), Q).explain(H, targets)
    assert np.isfinite(got[0]).all() and (got[1] >= 0).any(axis=2).all()
    rows = np.sort(rng.choice(n, 256, replace=False))
    S = H[rows]
    S.sort_indices()
    ref = explain_ref.explain_rows(Q, S.indptr[1:].astype(np.int64), S.indices, S.data, targets[rows], 5, 8.0, 0.1, False)
    check_rows(tuple(x[rows] for x in got), ref, Q, targets[rows])

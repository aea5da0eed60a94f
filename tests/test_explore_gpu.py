"""Exploration on the GPU (DESIGN.md 4.17): ALS.posterior_sample against the fp64 reference (tests/explore_ref.py),
scale 0 and explore=0 bitwise, the draw statistics, row independence and determinism, ParALS.topk_recommendation /
fold_in_recommendation with explore equal to the plain calls on the sampled rows in every ranking mode, the failure
rule, and a coverage check on a trained model."""
import copy

import numpy as np
import pytest
import scipy.sparse

from tests import explore_ref
from tests.helpers import csr_from_lengths, full_opt, init_factors
from tests.test_explain_gpu import _Data, als_model, bits, to_matrix

pytestmark = pytest.mark.gpu


def same(a, b):
    a, b = np.asarray(a), np.asarray(b)
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def check_parity(out, mean, Y, scale, failed=None):
    """per row ||out - mean - scale y_ref|| <= 1e-3 scale ||y_ref||"""
    for r in range(out.shape[0]):
        if failed is not None and failed[r]:
            assert same(out[r], mean[r]), r
            continue
        err = np.linalg.norm(out[r].astype(np.float64) - mean[r].astype(np.float64) - scale * Y[r])
        assert err <= 1e-3 * scale * np.linalg.norm(Y[r]), (r, err, scale * np.linalg.norm(Y[r]))


@pytest.mark.parametrize("alpha", [0.0, 8.0])
@pytest.mark.parametrize("adaptive_reg", [False, True])
@pytest.mark.parametrize("d", [5, 20, 32, 100, 128, 256])
def test_against_fp64_reference(cuda_lib, d, adaptive_reg, alpha):
    rng = np.random.default_rng(d * 10 + int(adaptive_reg) * 3 + int(alpha))
    I = 8000
    lengths = np.concatenate([[0, 1, 2, 31, 32, 33, 5000], rng.integers(1, 300, 20)])
    rng.shuffle(lengths)
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    # a row of one item repeated, and one of two items each repeated: duplicates stay separate entries of A_r
    r = int(np.flatnonzero(lengths == 31)[0])
    b = 0 if r == 0 else int(indptr[r - 1])
    keys[b:b + 31] = 17
    r = int(np.flatnonzero(lengths == 33)[0])
    b = 0 if r == 0 else int(indptr[r - 1])
    keys[b:b + 33] = np.sort(np.resize([5, 4000], 33))
    Q = init_factors(I, d, d, d + 1, scale=0.1, signed=True)
    opt = full_opt(d=d, optimizer="llt" if d < 128 else "ialspp", alpha=alpha, adaptive_reg=adaptive_reg)
    m = als_model(opt, Q)
    n = len(indptr)
    mean = (rng.standard_normal((n, d)) * 0.1).astype(np.float32)
    draw_keys = rng.choice(2 ** 40, n, replace=False)
    seed, scale = int(rng.integers(0, 2 ** 32)), 0.5
    out = m.posterior_sample(to_matrix(indptr, keys, vals, I), mean, scale=scale, seed=seed, draw_keys=draw_keys)
    assert out.dtype == np.float32 and out.shape == (n, d)
    _, Y, failed = explore_ref.sample_rows(Q, indptr, keys, vals, mean, draw_keys, seed, scale, alpha, opt["reg_u"],
                                           adaptive_reg)
    assert not failed.any()
    check_parity(out, mean, Y, scale)


@pytest.mark.parametrize("ld", [5, 16])
def test_row_pitch_of_mean_and_out(cuda_lib, ld):
    """the C entry point with mean / out rows ld floats apart, narrower (d = 5) or wider than the pitch at which Q is
    stored (8): the same draws as the padded rows of ALS.posterior_sample, the reference's within 1e-3, and columns
    d..ld-1 of out not written"""
    import torch
    from buffalo_b200.algo import fold_in
    from buffalo_b200.backend import CuALS
    d, I = 5, 2000
    rng = np.random.default_rng(50 + ld)
    indptr, keys, vals = csr_from_lengths(np.concatenate([[0, 1, 40, 300], rng.integers(1, 60, 40)]), I, rng)
    n = len(indptr)
    Q = init_factors(I, d, d, 12, scale=0.1, signed=True)
    m = als_model(full_opt(d=d, optimizer="llt"), Q)
    mean = (rng.standard_normal((n, d)) * 0.1).astype(np.float32)
    dk = rng.choice(2 ** 33, n, replace=False)
    want = m.posterior_sample(to_matrix(indptr, keys, vals, I), mean, scale=0.6, seed=77, draw_keys=dk)
    st, h = fold_in.resident_state(m, CuALS)
    assert h.get_vdim() == 8
    dev = torch.device("cuda")
    M = torch.zeros((n, ld), dtype=torch.float32, device=dev)
    M[:, :d] = torch.from_numpy(mean).to(dev)
    out = torch.full((n, ld), 7.0, dtype=torch.float32, device=dev)
    ind_t, keys_t, vals_t = fold_in.csr_to_device(indptr, keys, vals)
    try:
        m._bind_fold_items(st, h, torch.zeros((1, h.get_vdim()), dtype=torch.float32, device=dev))
        out, failed = h.posterior_sample_device(ind_t, keys_t, vals_t, M, torch.from_numpy(dk).to(dev), 77, 0.6,
                                                out=out)
    finally:
        h._keep = []
    got = out.cpu().numpy()
    assert int(failed.item()) == 0
    assert same(got[:, :d], want)
    assert (got[:, d:] == 7.0).all()
    _, Y, failed = explore_ref.sample_rows(Q, indptr, keys, vals, mean, dk, 77, 0.6, 8.0, 0.1, False)
    check_parity(got[:, :d], mean, Y, 0.6)


def test_zero_scale_returns_the_mean(cuda_lib):
    d, I = 16, 500
    rng = np.random.default_rng(2)
    indptr, keys, vals = csr_from_lengths(rng.integers(0, 40, 30), I, rng)
    m = als_model(full_opt(d=d), init_factors(I, d, d, 3, scale=0.1, signed=True))
    mean = rng.standard_normal((30, d)).astype(np.float32)
    mean[0, :3] = [-0.0, np.nan, np.inf]
    out = m.posterior_sample(to_matrix(indptr, keys, vals, I), mean, scale=0.0, seed=5)
    assert same(out, mean)


def test_statistics(cuda_lib):
    """20000 draw keys on one history: the empirical mean within 4 standard errors of the mean row, the empirical
    covariance within 0.05 (relative Frobenius) of the fp64 scale^2 A^-1"""
    for d in (8, 32):
        rng = np.random.default_rng(70 + d)
        I, n, scale = 300, 20000, 0.8
        # columns scaled from 1 down to 1/8: a spread of posterior variances
        Q = init_factors(I, d, d, 9, scale=0.3, signed=True) * (0.125 ** (np.arange(d) / (d - 1)))[None, :]
        Q = Q.astype(np.float32)
        row = np.sort(rng.choice(I, 25, replace=False)).astype(np.int32)
        v = rng.integers(1, 5, 25).astype(np.float32)
        m = als_model(full_opt(d=d, alpha=4.0, reg_u=0.2), Q)
        H = to_matrix(np.arange(1, n + 1, dtype=np.int64) * 25, np.tile(row, n), np.tile(v, n), I)
        mu = rng.standard_normal(d).astype(np.float32)
        out = m.posterior_sample(H, np.tile(mu, (n, 1)), scale=scale, seed=123).astype(np.float64)
        G = Q.astype(np.float64).T @ Q.astype(np.float64)
        want = scale ** 2 * np.linalg.inv(explore_ref.row_matrix(G, Q, row, v, 4.0, 0.2, False))
        se = np.sqrt(np.diag(want) / n)
        assert (np.abs(out.mean(axis=0) - mu) <= 4 * se).all(), d
        C = np.cov(out.T)
        assert np.linalg.norm(C - want) <= 0.05 * np.linalg.norm(want), (d, np.linalg.norm(C - want) / np.linalg.norm(want))


def test_independence_and_determinism(cuda_lib):
    import torch
    d, I = 32, 3000
    rng = np.random.default_rng(8)
    indptr, keys, vals = csr_from_lengths(rng.integers(0, 80, 300), I, rng)
    H = to_matrix(indptr, keys, vals, I)
    m = als_model(full_opt(d=d), init_factors(I, d, d, 4, scale=0.1, signed=True))
    mean = (rng.standard_normal((300, d)) * 0.1).astype(np.float32)
    dk = rng.choice(10 ** 6, 300, replace=False)
    whole = m.posterior_sample(H, mean, 0.7, 99, dk)
    assert same(m.posterior_sample(H, mean, 0.7, 99, dk), whole)                # repeated call
    for r in (0, 57, 299):                                                        # alone
        assert same(m.posterior_sample(H[r], mean[r:r + 1], 0.7, 99, dk[r:r + 1]), whole[r:r + 1])
    cuts = [0, 1, 120, 121, 300]                                                  # split over several calls
    parts = [m.posterior_sample(H[a:b], mean[a:b], 0.7, 99, dk[a:b]) for a, b in zip(cuts[:-1], cuts[1:])]
    assert same(np.concatenate(parts), whole)
    # inside a 100k-row call, at shuffled positions
    N = 100000
    blen = rng.integers(0, 60, N - 300)
    bkeys = rng.integers(0, I, int(blen.sum())).astype(np.int32)
    brow = np.repeat(np.arange(N - 300), blen)
    bkeys = bkeys[np.lexsort((bkeys, brow))]                                     # ascending within a row
    other = to_matrix(np.cumsum(blen), bkeys, rng.integers(1, 4, len(bkeys)).astype(np.float32), I)
    big = scipy.sparse.vstack([H, other]).tocsr()
    perm = rng.permutation(N)
    bmean = np.concatenate([mean, np.zeros((N - 300, d), np.float32)])
    bdk = np.concatenate([dk, 10 ** 6 + np.arange(N - 300)])
    got = m.posterior_sample(big[perm], bmean[perm], 0.7, 99, bdk[perm])
    inv = np.argsort(perm)
    assert same(got[inv[:300]], whole)
    # on a non-default stream
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        on_s = m.posterior_sample(H, mean, 0.7, 99, dk)
    s.synchronize()
    assert same(on_s, whole)
    # another seed moves every row
    other = m.posterior_sample(H, mean, 0.7, 100, dk)
    assert (np.abs(other - whole).max(axis=1) > 0).all()


def test_failed_factorisation_leaves_the_mean(cuda_lib):
    """adaptive_reg and an empty history: A = Q'Q, exactly singular for two items at d = 8; the row comes back as its
    mean and is counted, its neighbour with a history is sampled"""
    d = 8
    Q = np.zeros((2, d), np.float32)
    Q[0, :2] = 1.0
    Q[1, 2:4] = 1.0
    m = als_model(full_opt(d=d, adaptive_reg=True), Q)
    warnings = []
    m.logger = type("L", (), {"warning": lambda self, msg: warnings.append(msg)})()
    H = to_matrix(np.array([0, 2], np.int64), np.array([0, 1], np.int32), np.ones(2, np.float32), 2)
    mean = np.arange(2 * d, dtype=np.float32).reshape(2, d)
    out = m.posterior_sample(H, mean, scale=1.0, seed=3)
    assert same(out[0], mean[0]) and not same(out[1], mean[1])
    assert len(warnings) == 1 and "1 of 2 rows" in warnings[0]
    _, Y, failed = explore_ref.sample_rows(Q, np.array([0, 2], np.int64), np.array([0, 1], np.int32),
                                           np.ones(2, np.float32), mean, [0, 1], 3, 1.0, 8.0, 0.1, True)
    assert failed.tolist() == [True, False]
    check_parity(out, mean, Y, 1.0, failed)


def clustered(U, I, rng, clusters=10, per_user=30):
    """Rows of per_user distinct items: 80 % from the user's cluster (u % clusters, items i % clusters) at Zipf(1.2)
    popularity within it, the rest uniform over the catalogue."""
    members = [np.arange(c, I, clusters) for c in range(clusters)]
    rows = []
    for u in range(U):
        own = members[u % clusters]
        p = 1.0 / np.arange(1, len(own) + 1) ** 1.2
        picks = set(rng.choice(own, int(0.8 * per_user), replace=False, p=p / p.sum()).tolist())
        while len(picks) < per_user:
            picks.add(int(rng.integers(0, I)))
        rows.append(np.sort(np.fromiter(picks, np.int64)))
    keys = np.concatenate(rows).astype(np.int32)
    return np.cumsum([len(r) for r in rows]).astype(np.int64), keys, rng.integers(1, 4, len(keys)).astype(np.float32)


def trained(U=600, I=2000, d=24, seed=31, structured=False):
    from buffalo_b200.misc import aux
    rng = np.random.default_rng(seed)
    if structured:
        indptr, keys, vals = clustered(U, I, rng)
    else:
        indptr, keys, vals = csr_from_lengths(rng.integers(1, 60, U), I, rng)
    m = als_model(full_opt(d=d, num_iters=3, random_seed=3), np.zeros((1, d), np.float32))
    m.data = _Data(U, I, indptr, keys, vals)
    m.initialize()
    m.train()
    m._idmanager = aux.Option({"userids": ["u%d" % i for i in range(U)], "itemids": ["i%d" % i for i in range(I)],
                               "userid_mapped": True, "itemid_mapped": True})
    m._idmanager.userid_map = {v: i for i, v in enumerate(m._idmanager.userids)}
    m._idmanager.itemid_map = {v: i for i, v in enumerate(m._idmanager.itemids)}
    return m, rng, to_matrix(indptr, keys, vals, I)


def modes(rng, n_rows, U, I):
    pool = rng.choice(I, 300, replace=False)
    per_user = scipy.sparse.random(n_rows, I, density=0.05, format="csr", random_state=rng)
    seen = scipy.sparse.random(U, I, density=0.02, format="csr", random_state=rng)
    return pool, per_user, seen


def test_topk_recommendation_explores_the_sampled_rows(cuda_lib):
    from buffalo_b200.parallel.base import ParALS
    m, rng, R = trained()
    U, I = m.P.shape[0], m.Q.shape[0]
    par = ParALS(m)
    par.build_index(16)
    idx = np.sort(rng.choice(U, 120, replace=False)).astype(np.int32)
    pool, per_user, seen = modes(rng, U, U, I)
    calls = [dict(), dict(pool=["i%d" % p for p in pool]), dict(pool=per_user), dict(exclude_seen=True),
             dict(exclude_seen=seen), dict(diversify=0.4), dict(pool=per_user, exclude_seen=True, diversify=0.3),
             dict(nprobe=4)]
    sigma, s = 0.6, 2024
    sampled = m.P.copy()
    sampled[idx] = m.posterior_sample(R[idx], m.P[idx], scale=sigma, seed=s, draw_keys=idx)
    assert not np.array_equal(sampled[idx], m.P[idx])
    m2 = copy.copy(m)
    m2.P = sampled
    par2 = ParALS(m2)
    par2._indexes = par._indexes                         # the same index of the same Q
    for kw in calls:
        got = par.topk_recommendation(idx, 10, explore=sigma, explore_seed=s, **kw)
        want = par2.topk_recommendation(idx, 10, **kw)
        assert same(got[1], want[1]) and same(got[2], want[2]), kw
        # explore = 0 is the plain call, bit for bit
        zero, plain = par.topk_recommendation(idx, 10, explore=0.0, **kw), par.topk_recommendation(idx, 10, **kw)
        assert same(zero[1], plain[1]) and same(zero[2], plain[2]), kw
    # user ids resolve to the same rows and draw keys
    got = par.topk_recommendation(["u%d" % u for u in idx[:7]], 10, explore=sigma, explore_seed=s)
    assert same(got[1], par2.topk_recommendation(idx[:7], 10)[1])
    # a user listed twice, in any order, gets its one draw at both places
    dup = np.concatenate([idx[5:9], idx[:3], idx[6:8], idx[:1]]).astype(np.int32)
    for kw in (dict(), dict(exclude_seen=True), dict(nprobe=4)):
        got = par.topk_recommendation(dup, 10, explore=sigma, explore_seed=s, **kw)
        want = par2.topk_recommendation(dup, 10, **kw)
        assert same(got[1], want[1]) and same(got[2], want[2]), kw
    got = par.topk_recommendation(["u%d" % idx[0], "u%d" % idx[1], "u%d" % idx[0]], 10, explore=sigma, explore_seed=s)
    assert same(got[1][0], got[1][2]) and same(got[1], par2.topk_recommendation(idx[[0, 1, 0]], 10)[1])


def test_fold_in_recommendation_explores_the_sampled_rows(cuda_lib):
    from buffalo_b200.parallel.base import ParALS
    m, rng, R = trained(seed=33)
    I = m.Q.shape[0]
    n = 90
    lengths = rng.integers(0, 40, n)
    hi, hk, hv = csr_from_lengths(lengths, I, rng)
    H = to_matrix(hi, hk, hv, I)
    pool, per_user, _ = modes(rng, n, n, I)
    sigma, s = 0.9, 7
    X = m.fold_in(H)
    Xs = m.posterior_sample(H, X, scale=sigma, seed=s)
    m3 = copy.copy(m)
    m3.P = np.ascontiguousarray(Xs)
    par, par3 = ParALS(m), ParALS(m3)
    rows = np.arange(n, dtype=np.int32)
    calls = [(dict(exclude_seen=False), dict()), (dict(), dict(exclude_seen=H)),
             (dict(pool=["i%d" % p for p in pool]), dict(pool=["i%d" % p for p in pool], exclude_seen=H)),
             (dict(pool=per_user), dict(pool=per_user, exclude_seen=H)),
             (dict(diversify=0.5), dict(diversify=0.5, exclude_seen=H))]
    for kw, kw3 in calls:
        got = par.fold_in_recommendation(H, 10, explore=sigma, explore_seed=s, **kw)
        _, keys3, scores3 = par3.topk_recommendation(rows, 10, **kw3)
        assert same(got[0], keys3) and same(got[1], scores3), kw
        zero, plain = par.fold_in_recommendation(H, 10, explore=0.0, **kw), par.fold_in_recommendation(H, 10, **kw)
        assert same(zero[0], plain[0]) and same(zero[1], plain[1]), kw


def test_exploration_widens_coverage(cuda_lib):
    """on clustered data with popular items in every cluster the plain lists concentrate on them; Thompson draws spread
    each user's list over directions its history leaves uncertain"""
    from buffalo_b200.evaluate import evaluate_lists
    from buffalo_b200.parallel.base import ParALS
    m, rng, R = trained(U=1500, I=3000, d=32, seed=40, structured=True)
    par = ParALS(m)
    users = np.arange(m.P.shape[0], dtype=np.int32)
    test = R[users]
    plain = par.topk_recommendation(users, 10)[1]
    explored = par.topk_recommendation(users, 10, explore=1.0, explore_seed=1)[1]
    cov = lambda ranked: evaluate_lists(ranked, test, cutoffs=(10,))["coverage@10"]
    assert cov(explored) > cov(plain), (cov(explored), cov(plain))
    # another seed gives other lists, a repeated seed the same
    assert same(par.topk_recommendation(users, 10, explore=1.0, explore_seed=1)[1], explored)
    assert not same(par.topk_recommendation(users, 10, explore=1.0, explore_seed=2)[1], explored)

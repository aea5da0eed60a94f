"""Fold-in on the GPU (DESIGN.md 4.10): ALS.fold_in is the user half-epoch's row solve (bitwise with deterministic=True),
converges to the exact least-squares row, and leaves the model alone; PLSI.fold_in matches an fp64 mirror of Hofmann's
folding-in and one deterministic EM iteration of training; ParALS.fold_in_recommendation ranks the folded rows as the
serve handle ranks a host copy of them."""
import numpy as np
import pytest
import scipy.sparse

from tests.helpers import csr_from_lengths, full_opt, init_factors, rel_err, row_rel_err

pytestmark = pytest.mark.gpu


def bits(a):
    return np.ascontiguousarray(a, dtype=np.float32).view(np.uint32)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def to_matrix(indptr, keys, vals, num_items):
    return scipy.sparse.csr_matrix((vals, keys, np.concatenate([[0], indptr])), shape=(len(indptr), num_items))


def history_lengths(rng, n, split_rows=0, empty=0):
    """mostly short rows, `split_rows` of 1537..4000 entries (the split-row path at d >= 128), `empty` empty rows"""
    lengths = np.concatenate([rng.integers(1, 300, n - split_rows - empty), rng.integers(1537, 4001, split_rows),
                              np.zeros(empty, np.int64)])
    rng.shuffle(lengths)
    return lengths


def als_model(opt, P, Q):
    from buffalo_b200.algo.als import ALS
    from buffalo_b200.algo.options import ALSOption
    o = ALSOption().get_default_option()
    o.update(opt)
    m = ALS(o)
    m.P, m.Q = P.copy(), Q.copy()
    return m


def plsi_model(opt, P, Q):
    from buffalo_b200.algo.options import PLSIOption
    from buffalo_b200.algo.plsi import PLSI
    o = PLSIOption().get_default_option()
    o.update(opt)
    m = PLSI(o)
    m.P, m.Q = P.copy(), Q.copy()
    return m


def train_user_half(opt, P, Q, indptr, keys, vals):
    """P after one user half-epoch of a training holder: the calls ALS._train_resident makes for axis 0"""
    import torch
    from buffalo_b200 import backend
    obj = backend.CuALS()
    assert obj.init(opt)
    vdim, d = obj.get_vdim(), opt["d"]
    tP = torch.zeros(P.shape[0], vdim, device="cuda")
    tQ = torch.zeros(Q.shape[0], vdim, device="cuda")
    tP[:, :d], tQ[:, :d] = torch.from_numpy(P).cuda(), torch.from_numpy(Q).cuda()
    obj.bind_factors(tP, tQ)
    obj.bind_csr(0, torch.from_numpy(indptr).cuda(), torch.from_numpy(keys).cuda(), torch.from_numpy(vals).cuda())
    loss = torch.zeros(2, dtype=torch.float64, device="cuda")
    obj.precompute_device(0)
    obj.update_device(0, 0, P.shape[0], loss)
    return tP[:, :d].cpu().numpy()


@pytest.mark.parametrize("deterministic", [True, False])
@pytest.mark.parametrize("d", [5, 20, 32, 100, 128, 256])
@pytest.mark.parametrize("optimizer", ["llt", "ldlt", "manual_cg", "ialspp"])
def test_als_equals_training_half_epoch(cuda_lib, optimizer, d, deterministic):
    rng = np.random.default_rng(d)
    lengths = history_lengths(rng, 700, split_rows=24, empty=5)
    I = 6000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    P = init_factors(len(lengths), d, d, 1, scale=0.05, signed=True)
    Q = init_factors(I, d, d, 2, scale=0.05, signed=True)
    opt = full_opt(d=d, optimizer=optimizer, deterministic=deterministic)
    want = train_user_half(opt, P, Q, indptr, keys, vals)
    m = als_model(opt, P, Q)
    got = m.fold_in(to_matrix(indptr, keys, vals, I), init=P, sweeps=1)
    assert got.shape == (len(lengths), d) and got.dtype == np.float32
    if deterministic:
        assert same_bits(got, want)
    else:
        assert rel_err(got, want) < 1e-5
    empty = lengths == 0
    assert same_bits(got[empty], P[empty])                 # empty rows keep their start row


def row_systems(Q, indptr, keys, vals, alpha, reg, ialspp=False):
    """fp64 (A, b) per row: A = Q'Q + sum (c - 1) q q' + reg I, b = sum c q, c = 1 + alpha v.  iALS++ moves toward the
    target 1 with the weights c - 1 only (its gradient, oracle/np_mirror.py), so its fixed point has b = sum (c - 1) q."""
    Q = Q.astype(np.float64)
    G = Q.T @ Q
    beg = np.concatenate([[0], indptr[:-1]])
    for r in range(len(indptr)):
        q, c = Q[keys[beg[r]:indptr[r]]], 1.0 + alpha * vals[beg[r]:indptr[r]].astype(np.float64)
        A = G + (q * (c - 1)[:, None]).T @ q + reg * np.eye(Q.shape[1])
        yield A, (q * ((c - 1) if ialspp else c)[:, None]).sum(axis=0)


def exact_rows(Q, indptr, keys, vals, alpha, reg, ialspp=False):
    return np.array([np.linalg.solve(A, b) for A, b in row_systems(Q, indptr, keys, vals, alpha, reg, ialspp)])


def rel_residual(Q, indptr, keys, vals, alpha, reg, X, ialspp=False):
    return float(max(np.linalg.norm(A @ x - b) / np.linalg.norm(b)
                     for (A, b), x in zip(row_systems(Q, indptr, keys, vals, alpha, reg, ialspp), X.astype(np.float64))))


def fresh_problem(d, seed, n=200, I=3000):
    rng = np.random.default_rng(seed)
    indptr, keys, vals = csr_from_lengths(rng.integers(1, 200, n), I, rng)
    Q = init_factors(I, d, d, seed + 1, scale=0.1, signed=True)
    return indptr, keys, vals, Q, I


@pytest.mark.parametrize("d", [5, 20, 32, 100])
@pytest.mark.parametrize("optimizer", ["llt", "ldlt"])
def test_als_direct_solvers_are_exact(cuda_lib, optimizer, d):
    indptr, keys, vals, Q, I = fresh_problem(d, 3 * d)
    opt = full_opt(d=d, optimizer=optimizer)
    X = als_model(opt, np.zeros((1, d), np.float32), Q).fold_in(to_matrix(indptr, keys, vals, I))
    want = exact_rows(Q, indptr, keys, vals, opt["alpha"], opt["reg_u"])
    assert row_rel_err(X, want).max() < 1e-3


@pytest.mark.parametrize("d", [20, 32, 100, 128])
@pytest.mark.parametrize("optimizer", ["manual_cg", "ialspp"])
def test_als_iterative_solvers_converge_with_sweeps(cuda_lib, optimizer, d):
    indptr, keys, vals, Q, I = fresh_problem(d, 5 * d)
    opt = full_opt(d=d, optimizer=optimizer)
    m = als_model(opt, np.zeros((1, d), np.float32), Q)
    H = to_matrix(indptr, keys, vals, I)
    ialspp = optimizer == "ialspp" or d >= 128            # the d >= 128 rule
    res = []
    for sweeps in (1, 2, 4, 8, d):
        X = m.fold_in(H, sweeps=sweeps)
        res.append(rel_residual(Q, indptr, keys, vals, opt["alpha"], opt["reg_u"], X, ialspp))
    print("relative residual by sweeps:", res)
    for a, b in zip(res, res[1:]):
        assert b <= a * (1 + 1e-3) + 1e-5, res          # fp32 noise once converged
    want = exact_rows(Q, indptr, keys, vals, opt["alpha"], opt["reg_u"], ialspp)
    assert row_rel_err(X, want).max() < 1e-3


class _Data(object):
    """The part of a database ALS.train() reads: header and the two CSR groups."""

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


def test_model_untouched(cuda_lib):
    d, U, I = 32, 500, 2000
    rng = np.random.default_rng(77)
    indptr, keys, vals = csr_from_lengths(rng.integers(1, 100, U), I, rng)
    H = to_matrix(*csr_from_lengths(rng.integers(0, 60, 50), I, rng), I)
    opt = full_opt(d=d, deterministic=True, num_iters=3, random_seed=4)
    models = []
    for with_fold in (True, False):
        m = als_model(opt, np.zeros((1, d), np.float32), np.zeros((1, d), np.float32))
        m.data = _Data(U, I, indptr, keys, vals)
        m.initialize()
        if with_fold:
            P0, Q0 = m.P.copy(), m.Q.copy()
            m.fold_in(H, init=None, sweeps=2)
            assert same_bits(m.P, P0) and same_bits(m.Q, Q0)
        m.train()
        models.append(m)
    assert same_bits(models[0].P, models[1].P) and same_bits(models[0].Q, models[1].Q)
    # Q edited in place: the next fold_in recomputes the Gram and equals that of a fresh model
    m = models[0]
    before = m.fold_in(H)
    m.Q[::7] *= 1.5
    after = m.fold_in(H)
    fresh = als_model(opt, m.P, m.Q).fold_in(H)
    assert same_bits(after, fresh) and not same_bits(after, before)
    m.normalize("item")                       # normalised items are refused
    with pytest.raises(RuntimeError):
        m.fold_in(H)


def plsi_fold_in_fp64(Q, indptr, keys, vals, X0, iters, alpha1):
    """Hofmann's folding-in in fp64: per iteration acc = sum v l / sum l, l = max(x q, 1e-10), then
    x = (acc + alpha1 / d) / sum(acc + alpha1 / d); empty rows keep their start row."""
    Q = Q.astype(np.float64)
    d = Q.shape[1]
    a1 = alpha1 / d
    X = X0.astype(np.float64).copy()
    beg = np.concatenate([[0], indptr[:-1]])
    for r in range(len(indptr)):
        if indptr[r] == beg[r]:
            continue
        q, v = Q[keys[beg[r]:indptr[r]]], vals[beg[r]:indptr[r]].astype(np.float64)
        x = X[r]
        for _ in range(iters):
            lat = np.maximum(x[None, :] * q, 1e-10)
            acc = (v / lat.sum(axis=1)) @ lat
            x = (acc + a1) / (acc + a1).sum()
        X[r] = x
    return X


def plsi_factors(U, I, d, seed):
    rng = np.random.default_rng(seed)
    P = rng.random((U, d)) + 0.05
    Q = rng.random((I, d)) + 0.05
    return (P / P.sum(axis=1, keepdims=True)).astype(np.float32), (Q / Q.sum(axis=0, keepdims=True)).astype(np.float32)


@pytest.mark.parametrize("d", [1, 7, 20, 128, 512])
@pytest.mark.parametrize("iters", [1, 5, 20])
def test_plsi_against_fp64(cuda_lib, d, iters):
    rng = np.random.default_rng(d * 31 + iters)
    I = 4000
    lengths = history_lengths(rng, 300, empty=4)
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    P, Q = plsi_factors(1, I, d, d)
    m = plsi_model(dict(d=d, alpha1=1.0), P, Q)
    H = to_matrix(indptr, keys, vals, I)
    X = m.fold_in(H, iters=iters)
    want = plsi_fold_in_fp64(Q, indptr, keys, vals, np.full((len(lengths), d), 1.0 / d), iters, 1.0)
    assert row_rel_err(X, want).max() < 1e-4
    assert np.abs(X.sum(axis=1) - 1.0).max() < 1e-5
    assert same_bits(X, m.fold_in(H, iters=iters))          # run to run
    assert (X[lengths == 0] == np.float32(1.0 / d)).all()


@pytest.mark.parametrize("d", [7, 20, 128])
def test_plsi_one_iteration_equals_training(cuda_lib, d):
    import torch
    from buffalo_b200 import backend
    from tests.helpers import transpose_csr
    rng = np.random.default_rng(90 + d)
    U, I = 400, 3000
    indptr, keys, vals = csr_from_lengths(rng.integers(1, 200, U), I, rng)
    P, Q = plsi_factors(U, I, d, d + 1)
    opt = dict(d=d, alpha1=1.0, alpha2=1.0, deterministic=True)
    g = backend.CuPLSI()
    assert g.init(opt)
    vdim = g.get_vdim()
    tP = torch.zeros(U, vdim, device="cuda")
    tQ = torch.zeros(I, vdim, device="cuda")
    tP[:, :d], tQ[:, :d] = torch.from_numpy(P).cuda(), torch.from_numpy(Q).cuda()
    g.bind_factors(tP, tQ)
    g.bind_csr(*[torch.from_numpy(a).cuda() for a in (indptr, keys, vals)])
    g.bind_colwise_csr(*[torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in transpose_csr(indptr, keys, vals, U, I)])
    g.update_items_device(0, I)
    g.update_device(0, U, torch.zeros(1, dtype=torch.float64, device="cuda"))
    g.normalize_device(1.0, 1.0)
    want = tP[:, :d].cpu().numpy()
    got = plsi_model(opt, P, Q).fold_in(to_matrix(indptr, keys, vals, I), init=P, iters=1)
    assert np.abs(got - want).max() < 1e-6


def serve_reference(Q, X, vdim, indptr, keys, topk, pool, exclude_seen):
    """Serve.topk_seen / topk on a host copy of the folded rows (padded to the device row pitch)"""
    from buffalo_b200 import backend
    h = backend.Serve()
    h.set_items(np.ascontiguousarray(Q, dtype=np.float32))
    Xp = np.zeros((X.shape[0], vdim), np.float32)
    Xp[:, :X.shape[1]] = X
    h.set_queries(Xp)
    h.set_pool(pool)
    q = np.arange(X.shape[0], dtype=np.int32)
    if exclude_seen:
        return h.topk_seen(q, topk, indptr, keys if len(keys) else np.zeros(1, np.int32))
    return h.topk(q, topk)


@pytest.mark.parametrize("exclude_seen", [True, False])
@pytest.mark.parametrize("with_pool", [False, True])
@pytest.mark.parametrize("kind", ["als", "plsi"])
def test_fold_in_recommendation(cuda_lib, kind, with_pool, exclude_seen):
    from buffalo_b200.parallel.base import ParALS
    d, I, n, topk = 20, 5000, 300, 50
    rng = np.random.default_rng(5)
    indptr, keys, vals = csr_from_lengths(history_lengths(rng, n, empty=3), I, rng)
    H = to_matrix(indptr, keys, vals, I)
    if kind == "als":
        m = als_model(full_opt(d=d), np.zeros((1, d), np.float32), init_factors(I, d, d, 3, scale=0.1, signed=True))
    else:
        P, Q = plsi_factors(1, I, d, 4)
        m = plsi_model(dict(d=d), P, Q)
    pool = rng.choice(I, 700, replace=False).astype(np.int32) if with_pool else None
    par = ParALS(m)
    got_k, got_s = par.fold_in_recommendation(H, topk=topk, pool=pool, exclude_seen=exclude_seen)
    # nothing of the call stays referenced: the folded rows and the history CSR are freed with its results
    assert "queries" not in par._serve._bound and par._serve.num_queries == 0
    assert m._fold_state.holder._keep == []
    X = m.fold_in(H)
    want_k, want_s = serve_reference(m.Q, X, m._fold_state.holder.get_vdim(), indptr, keys, topk, pool, exclude_seen)
    assert np.array_equal(got_k, want_k) and same_bits(got_s, want_s)
    if exclude_seen:
        beg = np.concatenate([[0], indptr[:-1]])
        for r in range(n):
            assert not set(got_k[r].tolist()) & set(keys[beg[r]:indptr[r]].tolist())
    if with_pool:
        assert set(got_k[got_k >= 0].tolist()) <= set(pool.tolist())


@pytest.mark.parametrize("kind", ["als", "plsi"])
def test_lists_and_empty_rows(cuda_lib, kind):
    d, I = 20, 400
    if kind == "als":
        m = als_model(full_opt(d=d), np.zeros((1, d), np.float32), init_factors(I, d, d, 3, scale=0.1, signed=True))
    else:
        P, Q = plsi_factors(1, I, d, 6)
        m = plsi_model(dict(d=d), P, Q)
    ids = ["item%d" % i for i in range(I)]
    m._idmanager.itemids, m._idmanager.itemid_map, m._idmanager.itemid_mapped = ids, {v: i for i, v in enumerate(ids)}, True
    rng = np.random.default_rng(8)
    rows = [sorted(rng.choice(I, rng.integers(0, 30), replace=False).tolist()) for _ in range(40)]
    rows[3] = []
    lists = [[ids[i] for i in r] + ["unknown-%d" % j for j in range(k % 3)] for k, r in enumerate(rows)]
    rng.shuffle(lists[5])
    lens = np.array([len(r) for r in rows])
    indptr = np.cumsum(lens).astype(np.int64)
    mat = to_matrix(indptr, np.concatenate(rows).astype(np.int32), np.ones(int(lens.sum()), np.float32), I)
    init = rng.random((40, d)).astype(np.float32)
    a, b = m.fold_in(lists, init=init), m.fold_in(mat, init=init)
    assert same_bits(a, b)
    assert same_bits(a[lens == 0], init[lens == 0]) and lens[3] == 0
    assert all(not same_bits(a[r], init[r]) for r in np.flatnonzero(lens))

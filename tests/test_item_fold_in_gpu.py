"""Item fold-in on the GPU (DESIGN.md 4.16): ALS.fold_in_items is the item half-epoch's row solve (bitwise with
deterministic=True) and converges to the exact least-squares row; BPRMF / WARP .fold_in_items match the NumPy reference
draw for draw; the calls are reproducible, row-independent and leave the model alone; folded held-out items land in
their own cluster; and add_items serves the new rows exactly as hand-stacked factors."""
import types

import numpy as np
import pytest

from tests import item_fold_in_ref as ref
from tests.helpers import csr_from_lengths, full_opt, init_factors, row_rel_err, transpose_csr
from tests.test_fold_in_gpu import exact_rows, history_lengths, rel_residual, same_bits, to_matrix

pytestmark = pytest.mark.gpu


class Data(object):
    """The part of a database the trainers and the fold-in read: header, both CSR groups and the batch option."""

    def __init__(self, U, I, indptr, keys, vals=None):
        vals = np.ones(len(keys), np.float32) if vals is None else vals
        cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
        self.header = {"num_users": U, "num_items": I, "num_nnz": len(keys)}
        self.groups = {"rowwise": {"indptr": indptr, "key": keys, "val": vals},
                       "colwise": {"indptr": cind, "key": ckeys, "val": cvals}}
        self.opt = types.SimpleNamespace(data=types.SimpleNamespace(batch_mb=64))

    def get_header(self):
        return self.header

    def get_group(self, name):
        return self.groups[name]


def als_model(opt, P, Q):
    from buffalo_b200.algo.als import ALS
    from buffalo_b200.algo.options import ALSOption
    o = ALSOption().get_default_option()
    o.update(opt)
    m = ALS(o)
    if P is not None:
        m.P, m.Q = P.copy(), Q.copy()
    return m


def sgd_model(kind, opt, P=None, Q=None, Qb=None, data=None):
    from buffalo_b200.algo.bpr import BPRMF
    from buffalo_b200.algo.options import BPRMFOption, WARPOption
    from buffalo_b200.algo.warp import WARP
    cls, opt_cls = (BPRMF, BPRMFOption) if kind == "bpr" else (WARP, WARPOption)
    o = opt_cls().get_default_option()
    o.update(dict(evaluation_on_learning=False, compute_loss_on_training=False))
    o.update(opt)
    m = cls(o)
    if P is not None:
        m.P, m.Q, m.Qb = P.copy(), Q.copy(), Qb.copy()
    m.data = data
    return m


def train_item_half(opt, P, Q, cind, ckeys, cvals):
    """Q after one item half-epoch of a training holder: the calls ALS._train_resident makes for axis 1"""
    import torch
    from buffalo_b200 import backend
    obj = backend.CuALS()
    assert obj.init(opt)
    vdim, d = obj.get_vdim(), opt["d"]
    tP = torch.zeros(P.shape[0], vdim, device="cuda")
    tQ = torch.zeros(Q.shape[0], vdim, device="cuda")
    tP[:, :d], tQ[:, :d] = torch.from_numpy(P).cuda(), torch.from_numpy(Q).cuda()
    obj.bind_factors(tP, tQ)
    obj.bind_csr(1, torch.from_numpy(cind).cuda(), torch.from_numpy(ckeys).cuda(), torch.from_numpy(cvals).cuda())
    loss = torch.zeros(2, dtype=torch.float64, device="cuda")
    obj.precompute_device(1)
    obj.update_device(1, 0, Q.shape[0], loss)
    return tQ[:, :d].cpu().numpy()


# ---- ALS -------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [5, 20, 32, 100, 128, 256])
@pytest.mark.parametrize("optimizer", ["llt", "ldlt", "manual_cg", "ialspp"])
def test_als_equals_training_item_half_epoch(cuda_lib, optimizer, d):
    rng = np.random.default_rng(d + 1)
    lengths = history_lengths(rng, 600, split_rows=20, empty=4)      # item rows: users per item
    U = 6000
    cind, ckeys, cvals = csr_from_lengths(lengths, U, rng)
    P = init_factors(U, d, d, 1, scale=0.05, signed=True)
    Q = init_factors(len(lengths), d, d, 2, scale=0.05, signed=True)
    opt = full_opt(d=d, optimizer=optimizer, deterministic=True, reg_i=0.3, adaptive_reg=(d == 20))
    want = train_item_half(opt, P, Q, cind, ckeys, cvals)
    m = als_model(opt, P, Q)
    P0, Q0 = m.P.copy(), m.Q.copy()
    got = m.fold_in_items(to_matrix(cind, ckeys, cvals, U), init=Q, sweeps=1)
    assert got.shape == (len(lengths), d) and got.dtype == np.float32
    assert same_bits(got, want)
    assert same_bits(m.P, P0) and same_bits(m.Q, Q0)
    empty = lengths == 0
    assert same_bits(got[empty], Q[empty])


@pytest.mark.parametrize("d", [5, 20, 32, 100])
@pytest.mark.parametrize("optimizer", ["llt", "ldlt"])
def test_als_direct_solvers_are_exact(cuda_lib, optimizer, d):
    rng = np.random.default_rng(7 * d)
    U = 3000
    cind, ckeys, cvals = csr_from_lengths(rng.integers(1, 200, 200), U, rng)
    P = init_factors(U, d, d, d + 1, scale=0.1, signed=True)
    opt = full_opt(d=d, optimizer=optimizer, reg_i=0.2)
    X = als_model(opt, P, np.zeros((1, d), np.float32)).fold_in_items(to_matrix(cind, ckeys, cvals, U))
    want = exact_rows(P, cind, ckeys, cvals, opt["alpha"], opt["reg_i"])
    assert row_rel_err(X, want).max() < 1e-4


@pytest.mark.parametrize("d", [20, 128])
@pytest.mark.parametrize("optimizer", ["manual_cg", "ialspp"])
def test_als_iterative_solvers_converge_with_sweeps(cuda_lib, optimizer, d):
    rng = np.random.default_rng(11 * d)
    U = 3000
    cind, ckeys, cvals = csr_from_lengths(rng.integers(1, 200, 200), U, rng)
    P = init_factors(U, d, d, d + 2, scale=0.1, signed=True)
    opt = full_opt(d=d, optimizer=optimizer)
    m = als_model(opt, P, np.zeros((1, d), np.float32))
    H = to_matrix(cind, ckeys, cvals, U)
    ialspp = optimizer == "ialspp" or d >= 128
    res = [rel_residual(P, cind, ckeys, cvals, opt["alpha"], opt["reg_i"], m.fold_in_items(H, sweeps=s), ialspp)
           for s in (1, 2, 4, 8, d)]
    print("relative residual by sweeps:", res)
    for a, b in zip(res, res[1:]):
        assert b <= a * (1 + 1e-3) + 1e-5, res
    assert res[-1] < res[0]


def test_als_refuses_normalized_users_and_follows_p(cuda_lib):
    d, U = 16, 500
    rng = np.random.default_rng(5)
    P = init_factors(U, d, d, 3, scale=0.1, signed=True)
    H = to_matrix(*csr_from_lengths(rng.integers(1, 50, 30), U, rng), U)
    m = als_model(full_opt(d=d, optimizer="llt"), P, np.zeros((1, d), np.float32))
    before = m.fold_in_items(H)
    m.P[::5] *= 1.5                                            # in place: the next call uploads P and its Gram again
    after = m.fold_in_items(H)
    fresh = als_model(full_opt(d=d, optimizer="llt"), m.P, m.Q).fold_in_items(H)
    assert same_bits(after, fresh) and not same_bits(after, before)
    m.normalize("user")
    with pytest.raises(RuntimeError, match="normalized"):
        m.fold_in_items(H)


# ---- BPRMF / WARP against the reference ------------------------------------------------------------------------
def sgd_problem(d, seed, U=120, I=90, n=10):
    rng = np.random.default_rng(seed)
    indptr, keys, _ = csr_from_lengths(rng.integers(1, 30, U), I, rng)
    P = init_factors(U, d, d, seed + 1, scale=0.4, signed=True)
    Q = init_factors(I, d, d, seed + 2, scale=0.4, signed=True)
    Qb = (rng.standard_normal((I, 1)) * 0.2).astype(np.float32)
    lengths = rng.integers(0, 9, n)
    lengths[0] = 0
    hind, husers, _ = csr_from_lengths(lengths, U, rng)
    return Data(U, I, indptr, keys), P, Q, Qb, hind, husers


CASES = [  # kind, d, options
    ("bpr", 8, dict(optimizer="sgd")),
    ("bpr", 20, dict(optimizer="sgd", num_negative_samples=3, verify_neg=False)),
    ("bpr", 20, dict(optimizer="adagrad", sampling_power=1.0)),
    ("bpr", 64, dict(optimizer="adam", use_bias=False)),
    ("bpr", 128, dict(optimizer="adagrad", per_coordinate_normalize=True, sampling_power=2.0, verify_neg=False)),
    ("bpr", 256, dict(optimizer="sgd", sampling_power=1.0)),
    ("warp", 8, dict(optimizer="adagrad")),
    ("warp", 20, dict(optimizer="adam", score_func="l2")),
    ("warp", 64, dict(optimizer="adagrad", score_func="l2", max_trials=5)),
    ("warp", 128, dict(optimizer="adam", threshold=0.5)),
    ("warp", 256, dict(optimizer="adagrad", per_coordinate_normalize=True)),
]


@pytest.mark.parametrize("kind,d,extra", CASES)
def test_sgd_matches_reference(cuda_lib, kind, d, extra):
    data, P, Q, Qb, hind, husers = sgd_problem(d, d + len(extra))
    opt = dict(d=d, lr=0.1, min_lr=0.01, reg_i=0.02, reg_b=0.05, random_seed=9, num_iters=3, use_bias=True)
    opt.update(extra)
    m = sgd_model(kind, opt, P, Q, Qb, data)
    U = P.shape[0]
    X0 = init_factors(len(hind), d, d, 77, scale=0.3, signed=True)
    tX, tXb, (negs, trials) = m._fold_in_items_device(to_matrix(hind, husers, np.ones(len(husers)), U), init=X0,
                                                      trace=True)
    o = dict(m.opt)
    cum = None
    if kind == "bpr" and opt.get("sampling_power", 0) > 0:
        cum = np.cumsum(np.bincount(data.groups["rowwise"]["key"], minlength=Q.shape[0]).astype(np.int64)
                        ** int(opt["sampling_power"]))
    want = ref.fold_in_items(kind, o, P, Q, Qb, data.groups["rowwise"]["indptr"], data.groups["rowwise"]["key"], cum,
                             hind, husers, X0, np.zeros(len(hind)), opt["num_iters"])
    assert np.array_equal(negs.cpu().numpy(), want[2])
    if kind == "warp":
        assert np.array_equal(trials.cpu().numpy(), want[3])
    X, Xb = tX[:, :d].cpu().numpy(), tXb.cpu().numpy()
    print("max abs difference to the reference: %.3g (largest value %.3g)" % (np.abs(X - want[0]).max(),
                                                                          np.abs(want[0]).max()))
    assert np.allclose(X, want[0], rtol=1e-5, atol=1e-5 * np.abs(want[0]).max())
    assert np.allclose(Xb, want[1], rtol=1e-5, atol=1e-6)
    if extra["optimizer"] == "sgd":                               # a row without history keeps its start there
        assert same_bits(X[0], X0[0]) and Xb[0] == 0.0


@pytest.mark.parametrize("kind", ["bpr", "warp"])
def test_sgd_reproducible_row_independent_and_side_effect_free(cuda_lib, kind):
    d = 32
    data, P, Q, Qb, hind, husers = sgd_problem(d, 3, U=400, I=300, n=300)
    opt = dict(d=d, optimizer="adagrad", random_seed=5, num_iters=4, sampling_power=1.0)
    m = sgd_model(kind, opt, P, Q, Qb, data)
    U = P.shape[0]
    H = to_matrix(hind, husers, np.ones(len(husers)), U)
    before = [a.copy() for a in (m.P, m.Q, m.Qb)]
    X1, b1 = m.fold_in_items(H)
    X2, b2 = m.fold_in_items(H)
    assert same_bits(X1, X2) and same_bits(b1, b2)
    assert all(same_bits(a, b) for a, b in zip(before, (m.P, m.Q, m.Qb)))
    H2 = H.tolil()
    H2[7, :] = 0
    H2[7, [1, 2, 3]] = 1
    X3, b3 = m.fold_in_items(H2.tocsr())
    others = np.arange(H.shape[0]) != 7
    assert same_bits(X3[others], X1[others]) and same_bits(b3[others], b1[others])
    assert not same_bits(X3[7], X1[7])
    # the training holder's factors are those of initialize_model: still what train() left
    assert all(same_bits(a, b) for a, b in zip(before, (m.P, m.Q, m.Qb)))


# ---- quality on planted clusters --------------------------------------------------------------------------------
def planted(seed=0, C=4, U_per=150, I_per=60, held=10):
    """Users and items in C clusters; each user picks 25 items of its own cluster and 2 elsewhere.  The last `held`
    items of each cluster are held out of training.  Returns (train Data, item cluster of the trained items, held-out
    user lists, their clusters)."""
    rng = np.random.default_rng(seed)
    U, I = C * U_per, C * I_per
    item_c = np.repeat(np.arange(C), I_per)
    rows = []
    for u in range(U):
        c = u // U_per
        own = rng.choice(np.where(item_c == c)[0], 25, replace=False)
        other = rng.choice(np.where(item_c != c)[0], 2, replace=False)
        rows.append(np.sort(np.concatenate([own, other])))
    held_items = np.concatenate([np.where(item_c == c)[0][-held:] for c in range(C)])
    keep = np.setdiff1d(np.arange(I), held_items)
    remap = -np.ones(I, np.int64)
    remap[keep] = np.arange(len(keep))
    train_rows = [remap[r[remap[r] >= 0]] for r in rows]
    indptr = np.cumsum([len(r) for r in train_rows]).astype(np.int64)
    keys = np.concatenate(train_rows).astype(np.int32)
    hist = [[u for u in range(U) if h in rows[u]] for h in held_items]
    return Data(U, len(keep), indptr, keys), item_c[keep], hist, item_c[held_items]


@pytest.mark.parametrize("kind", ["als", "bpr", "warp"])
def test_folded_items_land_in_their_cluster(cuda_lib, kind):
    data, train_c, hist, held_c = planted()
    if kind == "als":
        m = als_model(full_opt(d=16, optimizer="llt", num_iters=8, random_seed=1, reg_i=1.0, reg_u=1.0), *[None] * 2)
    else:
        m = sgd_model(kind, dict(d=16, optimizer="adagrad", lr=0.1, num_iters=30, random_seed=1, num_workers=1))
    m.data = data
    m.initialize()
    m.train()
    ids = [str(u) for u in range(data.header["num_users"])]
    m._idmanager.update({"userids": ids, "userid_map": {v: i for i, v in enumerate(ids)}, "userid_mapped": True})
    items = [str(i) for i in range(data.header["num_items"])]
    m._idmanager.update({"itemids": items, "itemid_map": {v: i for i, v in enumerate(items)}, "itemid_mapped": True})
    out = m.fold_in_items([[str(u) for u in h] for h in hist])
    X = out if kind == "als" else out[0]
    hits = []
    for x, c in zip(X, held_c):
        top = m.most_similar(x.astype(np.float32), topk=10)
        hits.append(np.mean([train_c[int(k)] == c for k, _ in top]))
    observed = float(np.mean(hits))
    print("%s: fraction of the top-10 in the folded item's own cluster: %.3f (floor 0.8)" % (kind, observed))
    assert observed >= 0.8


# ---- serving through add_items ----------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", ["als", "bpr"])
def test_add_items_serves_like_stacked_factors(cuda_lib, kind):
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    d, U, I, n = 16, 300, 200, 25
    rng = np.random.default_rng(4)
    P = init_factors(U, d, d, 1, scale=0.3, signed=True)
    Q = init_factors(I, d, d, 2, scale=0.3, signed=True)
    Qb = (rng.standard_normal((I, 1)) * 0.1).astype(np.float32)
    rows = init_factors(n, d, d, 3, scale=0.3, signed=True)
    bias = (rng.standard_normal(n) * 0.1).astype(np.float32)
    ids = ["new%d" % i for i in range(n)]

    def model(Qm, Qbm, names):
        m = als_model(full_opt(d=d), P, Qm) if kind == "als" else sgd_model("bpr", dict(d=d, use_bias=True), P, Qm, Qbm)
        us = [str(u) for u in range(U)]
        m._idmanager.update({"userids": us, "userid_map": {v: i for i, v in enumerate(us)}, "userid_mapped": True,
                             "itemids": list(names), "itemid_map": {v: i for i, v in enumerate(names)},
                             "itemid_mapped": True})
        return m
    base_names = [str(i) for i in range(I)]
    a = model(Q, Qb, base_names)
    par_a = (ParALS if kind == "als" else ParBPRMF)(a)
    par_a.build_index(group="item", nlist=4)
    a.add_items(ids, rows, None if kind == "als" else bias)
    b = model(np.vstack([Q, rows]), np.vstack([Qb, bias[:, None]]), base_names + ids)
    par_b = (ParALS if kind == "als" else ParBPRMF)(b)
    users = [str(u) for u in range(0, U, 3)]
    ra = par_a.topk_recommendation(users, topk=20)
    rb = par_b.topk_recommendation(users, topk=20)
    for x, y in zip(ra, rb):
        assert np.array_equal(np.asarray(x), np.asarray(y))
    with pytest.raises(RuntimeError, match="stale"):
        par_a.topk_recommendation(users, topk=10, nprobe=2)
    qa = par_a.most_similar(ids[:5] + ["3", "7"], topk=10)
    qb = par_b.most_similar(ids[:5] + ["3", "7"], topk=10)
    for x, y in zip(qa, qb):
        assert np.array_equal(np.asarray(x), np.asarray(y))

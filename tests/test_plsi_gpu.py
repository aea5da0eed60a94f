"""pLSI on the GPU: one EM iteration through the host ABI against the float32 oracle (tests/plsi_ref.py), chunking,
the device-resident path, the padding columns, the device initialisation, and buffalo.PLSI end to end on a
synthetic matrix with planted clusters."""
import os

import numpy as np
import pytest

from tests.helpers import rel_err
from tests.plsi_ref import OraclePLSI, oracle_iteration, plsi_iteration, random_factors

pytestmark = pytest.mark.gpu

TOL = 1e-4


def gpu_iteration(P, Q, indptr, keys, vals, alpha1=1.0, alpha2=1.0, bounds=None):
    """One iteration through the holder ABI: set_model / reset / partial_update per chunk / normalize / swap."""
    from buffalo_b200 import backend
    g = backend.CuPLSI()
    assert g.init(dict(d=P.shape[1]))
    P1, Q1 = P.copy(), Q.copy()
    g.set_model(P1, Q1)
    g.reset()
    bounds = bounds or [0, P.shape[0]]
    loss = 0.0
    for a, b in zip(bounds[:-1], bounds[1:]):
        beg = 0 if a == 0 else int(indptr[a - 1])
        end = int(indptr[b - 1]) if b > 0 else 0
        k = np.ascontiguousarray(keys[beg:end]) if end > beg else np.zeros(1, np.int32)
        v = np.ascontiguousarray(vals[beg:end]) if end > beg else np.zeros(1, np.float32)
        loss += g.partial_update(a, b, indptr, k, v)
    g.normalize(alpha1, alpha2)
    g.swap()
    return P1, Q1, loss


@pytest.fixture(scope="module")
def edge_csr():
    """3000 users x 60000 items: empty user rows, 1-nnz rows, one row of 50000 nnz, and 100 items nobody touched."""
    rng = np.random.default_rng(17)
    U, I = 3000, 60000
    lens = rng.integers(0, 40, U)
    lens[rng.choice(U, 200, replace=False)] = 0
    lens[[7, 8, 9]] = 1
    lens[11] = 50000
    keys = np.concatenate([np.sort(rng.choice(I - 100, size=int(n), replace=False)) for n in lens]).astype(np.int32)
    indptr = np.cumsum(lens).astype(np.int64)
    ints = rng.integers(1, 6, len(keys)).astype(np.float32)
    logn = rng.lognormal(0.0, 1.5, len(keys)).astype(np.float32)
    return dict(U=U, I=I, indptr=indptr, keys=keys, vals={"ints": ints, "lognormal": logn})


@pytest.mark.parametrize("vals", ["ints", "lognormal"])
@pytest.mark.parametrize("d", [1, 3, 20, 64, 100, 128, 256, 512])
def test_one_iteration_matches_oracle(cuda_lib, edge_csr, d, vals):
    c = edge_csr
    P, Q = random_factors(c["U"], d, d, axis=1), random_factors(c["I"], d, d + 1, axis=0)
    v = c["vals"][vals]
    Pg, Qg, lg = gpu_iteration(P, Q, c["indptr"], c["keys"], v)
    Po, Qo, lo = oracle_iteration(P, Q, c["indptr"], c["keys"], v)
    assert rel_err(Pg, Po) < TOL and rel_err(Qg, Qo) < TOL, (rel_err(Pg, Po), rel_err(Qg, Qo))
    assert abs(lg - lo) <= TOL * abs(lo), (lg, lo)
    empty = np.flatnonzero(np.diff(np.concatenate([[0], c["indptr"]])) == 0)
    np.testing.assert_allclose(Pg[empty], 1.0 / d, rtol=1e-6)           # alpha1 / d, normalised: uniform
    assert np.isfinite(Pg).all() and np.isfinite(Qg).all()


def test_empty_row_without_alpha1_is_nan(cuda_lib, edge_csr):
    c = edge_csr
    d = 20
    P, Q = random_factors(c["U"], d, 1, axis=1), random_factors(c["I"], d, 2, axis=0)
    Pg, Qg, _ = gpu_iteration(P, Q, c["indptr"], c["keys"], c["vals"]["ints"], alpha1=0.0, alpha2=0.0)
    Po, Qo, _ = oracle_iteration(P, Q, c["indptr"], c["keys"], c["vals"]["ints"], alpha1=0.0, alpha2=0.0)
    assert np.array_equal(np.isnan(Pg), np.isnan(Po)) and np.isnan(Pg).any()
    live = np.isfinite(Po).all(axis=1)
    assert rel_err(Pg[live], Po[live]) < TOL and rel_err(Qg, Qo) < TOL


def test_chunks_equal_one_call(cuda_lib, edge_csr):
    c = edge_csr
    d = 64
    P, Q = random_factors(c["U"], d, 3, axis=1), random_factors(c["I"], d, 4, axis=0)
    args = (P, Q, c["indptr"], c["keys"], c["vals"]["lognormal"])
    Pw, Qw, lw = gpu_iteration(*args)
    Pc, Qc, lc = gpu_iteration(*args, bounds=[0, 5, 11, 12, 1000, 1001, 2999, c["U"]])
    assert rel_err(Pc, Pw) < 1e-6 and rel_err(Qc, Qw) < 1e-6 and abs(lc - lw) <= 1e-6 * abs(lw)


def _device_run(P, Q, indptr, keys, vals, iters, vdim, alpha1=1.0, alpha2=1.0, pad_value=0.0):
    import torch
    from buffalo_b200 import backend
    d = P.shape[1]
    g = backend.CuPLSI()
    assert g.init(dict(d=d))
    assert g.get_vdim() == vdim
    dev = torch.device("cuda", 0)
    tP = torch.full((P.shape[0], vdim), pad_value, dtype=torch.float32, device=dev)
    tQ = torch.full((Q.shape[0], vdim), pad_value, dtype=torch.float32, device=dev)
    tP[:, :d], tQ[:, :d] = torch.from_numpy(P).to(dev), torch.from_numpy(Q).to(dev)
    g.bind_factors(tP, tQ)
    g.bind_csr(torch.from_numpy(indptr).to(dev), torch.from_numpy(keys).to(dev), torch.from_numpy(vals).to(dev))
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    losses = []
    for _ in range(iters):
        loss.zero_()
        g.update_device(0, P.shape[0], loss)
        g.normalize_device(alpha1, alpha2)
        g.swap_device()
        losses.append(float(loss.item()))
    return tP.cpu().numpy(), tQ.cpu().numpy(), losses


def test_resident_equals_chunked_and_oracle_trajectory(cuda_lib, edge_csr):
    c = edge_csr
    d = 20
    v = c["vals"]["ints"]
    P, Q = random_factors(c["U"], d, 5, axis=1), random_factors(c["I"], d, 6, axis=0)
    Pr, Qr, lr = _device_run(P, Q, c["indptr"], c["keys"], v, 5, 20)
    Pc, Qc, Po, Qo = P, Q, P, Q
    for i in range(5):
        Pc, Qc, lc = gpu_iteration(Pc, Qc, c["indptr"], c["keys"], v, bounds=[0, 1000, 2000, c["U"]])
        Po, Qo, lo = oracle_iteration(Po, Qo, c["indptr"], c["keys"], v)
        assert abs(lr[i] - lc) <= 1e-5 * abs(lc), (i, lr[i], lc)
        assert abs(lr[i] - lo) <= TOL * abs(lo), (i, lr[i], lo)
    assert rel_err(Pr, Pc) < 1e-5 and rel_err(Qr, Qc) < 1e-5, (rel_err(Pr, Pc), rel_err(Qr, Qc))
    # after five iterations the float32 oracle has drifted by its own rounding too: judge the device against the
    # fp64 mirror, no further from it than 1.5x the oracle's distance (or within TOL)
    Pm, Qm = P, Q
    for _ in range(5):
        Pm, Qm, _ = plsi_iteration(Pm, Qm, c["indptr"], c["keys"], v)
    for X, Xo, Xm in ((Pr, Po, Pm), (Qr, Qo, Qm)):
        assert rel_err(X, Xm) <= max(TOL, 1.5 * rel_err(Xo, Xm)), (rel_err(X, Xm), rel_err(Xo, Xm))


def test_padding_columns_stay_zero_and_do_not_leak(cuda_lib, edge_csr):
    """d = 3 rows have one padding column on the device.  Even when it starts non-zero it is masked out of latent and
    its sum (the 1e-10 floor would otherwise add to the norm), and it leaves the iteration as zero."""
    c = edge_csr
    d = 3
    v = c["vals"]["lognormal"]
    P, Q = random_factors(c["U"], d, 7, axis=1), random_factors(c["I"], d, 8, axis=0)
    Ph, Qh, lh = gpu_iteration(P, Q, c["indptr"], c["keys"], v)
    for pad in (0.0, 0.5):
        Pd, Qd, ld = _device_run(P, Q, c["indptr"], c["keys"], v, 1, 4, pad_value=pad)
        assert not Pd[:, d:].any() and not Qd[:, d:].any()
        assert rel_err(Pd[:, :d], Ph) < 1e-6 and rel_err(Qd[:, :d], Qh) < 1e-6 and abs(ld[0] - lh) <= 1e-6 * abs(lh)


@pytest.mark.parametrize("d", [1, 20, 130])
def test_initialize_model(cuda_lib, d):
    from buffalo_b200 import backend

    def draw(seed):
        g = backend.CuPLSI()
        assert g.init(dict(d=d, random_seed=seed))
        P, Q = np.zeros((777, d), np.float32), np.zeros((1234, d), np.float32)
        g.initialize_model(P, Q)
        return P, Q
    P, Q = draw(3)
    assert (P >= 0).all() and (Q >= 0).all()
    np.testing.assert_allclose(P.sum(axis=1), 1.0, atol=1e-5)
    np.testing.assert_allclose(Q.sum(axis=0), 1.0, atol=1e-5)
    P2, Q2 = draw(3)
    assert np.array_equal(P, P2) and np.array_equal(Q, Q2)
    if d > 1:                         # at d = 1 every normalised P row is exactly 1
        P3, Q3 = draw(4)
        assert not np.array_equal(P, P3) and not np.array_equal(Q, Q3)


@pytest.mark.parametrize("d", [0, 513])
def test_out_of_range_d_is_rejected(cuda_lib, d):
    from buffalo_b200 import backend
    g = backend.CuPLSI()
    assert g.init(dict(d=d)) is False
    assert "d must be in [1, 512]" in g.last_error


# ---- buffalo.PLSI end to end -------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def clustered(tmp_path_factory):
    """943 x 1682 (ml-100k-shaped), ~100k interactions: every user and item belongs to one of 10 clusters, and 85% of
    a user's items come from the user's own cluster.  Written as MatrixMarket + uid / iid files."""
    rng = np.random.default_rng(7)
    U, I, K = 943, 1682, 10
    uc, ic = rng.integers(0, K, U), rng.integers(0, K, I)
    pop = rng.zipf(1.6, I).astype(np.float64)
    pop = np.minimum(pop, 200.0)
    rows, cols = [], []
    for u in range(U):
        n = int(np.clip(rng.lognormal(np.log(90), 0.6), 10, 600))
        own = np.flatnonzero(ic == uc[u])
        k_own = min(int(n * 0.85), len(own))
        p = pop[own] / pop[own].sum()
        pick = set(rng.choice(own, size=k_own, replace=False, p=p).tolist())
        pick |= set(rng.integers(0, I, n - k_own).tolist())
        rows += [u] * len(pick)
        cols += sorted(pick)
    vals = rng.integers(1, 6, len(rows))
    d = tmp_path_factory.mktemp("plsi")
    main = os.path.join(d, "main")
    with open(main, "w") as f:
        f.write("%%MatrixMarket matrix coordinate integer general\n%d %d %d\n" % (U, I, len(rows)))
        for r, c, v in zip(rows, cols, vals):
            f.write("%d %d %d\n" % (r + 1, c + 1, v))
    with open(os.path.join(d, "uid"), "w") as f:
        f.write("\n".join("user_%d" % i for i in range(U)))
    with open(os.path.join(d, "iid"), "w") as f:
        f.write("\n".join("item_%d" % i for i in range(I)))
    return dict(main=main, uid=os.path.join(d, "uid"), iid=os.path.join(d, "iid"), dir=str(d), U=U, I=I)


def data_option(ml, name, batch_mb=None):
    from buffalo.data import MatrixMarketOptions
    o = MatrixMarketOptions().get_default_option()
    o.input.main, o.input.uid, o.input.iid = ml["main"], ml["uid"], ml["iid"]
    o.data.path = os.path.join(ml["dir"], name + ".h5py")
    o.data.validation.p, o.data.validation.max_samples = 0.1, 10000
    if batch_mb is not None:
        o.data.batch_mb = batch_mb
    return o


def make_plsi(ml, name, **kw):
    from buffalo import PLSI, PLSIOption, aux
    opt = PLSIOption().get_default_option()
    opt.update(random_seed=7, validation=aux.Option({"topk": 10}))
    opt.update(kw)
    np.random.seed(5)                 # same validation split for every model built from this fixture
    return PLSI(opt, data_opt=data_option(ml, name, batch_mb=kw.get("_batch_mb")))


def test_plsi_train_quality_queries_and_save(cuda_lib, clustered, tmp_path):
    from buffalo import PLSI
    from buffalo.misc import log
    log.set_log_level(log.WARN)
    m = make_plsi(clustered, "q", num_iters=10, d=20)
    m.initialize()
    assert m.P.shape == (943, 20) and m.Q.shape == (1682, 20) and m.P.dtype == np.float32
    np.testing.assert_allclose(m.P.sum(axis=1), 1.0, atol=1e-5)
    calls = []
    ret = m.train(training_callback=lambda i, met: calls.append((i, sorted(met))))
    assert [i for i, _ in calls] == list(range(10)) and "val_ndcg" in calls[0][1]
    res = m.get_validation_results()
    assert res["ndcg"] > 0.03 and res["map"] > 0.02, res                      # tests/algo/test_plsi.py:39-42
    assert ret["train_loss"] > 0 and abs(ret["val_ndcg"] - res["ndcg"]) < 1e-9
    np.testing.assert_allclose(m.P.sum(axis=1), 1.0, atol=1e-4)
    np.testing.assert_allclose(m.Q.sum(axis=0), 1.0, atol=1e-4)
    # raw dot products (plsi.py:121-122): the query item need not rank first, and the 11 fetched rows are then all
    # kept (buffalo/algo/base.py most_similar drops only the query itself)
    sims = m.most_similar("item_49", 10)
    assert 10 <= len(sims) <= 11 and all(isinstance(k, str) and k != "item_49" for k, _ in sims)
    recs = m.topk_recommendation(["user_0", "user_5"], topk=5)
    assert set(recs) == {"user_0", "user_5"} and len(recs["user_0"]) == 5
    path = str(tmp_path / "plsi.bin")
    m.save(path)
    other = PLSI.new(path)
    assert np.array_equal(other.P, m.P) and np.array_equal(other.Q, m.Q) and other.opt.d == 20
    assert other.most_similar("item_49", 5) == m.most_similar("item_49", 5)


def test_plsi_resident_equals_chunked(cuda_lib, clustered):
    outs = []
    for resident, batch_mb in ((True, 1024), (False, 1)):        # batch_mb = 1: several chunks per iteration
        m = make_plsi(clustered, "rc%d" % int(resident), num_iters=5, d=32, _b200_resident=resident,
                      _batch_mb=batch_mb, validation={})
        m.initialize()
        P0 = m.P.copy()
        ret = m.train()
        outs.append((P0, m.P.copy(), m.Q.copy(), ret["train_loss"]))
    (P0a, Pa, Qa, la), (P0b, Pb, Qb, lb) = outs
    assert np.array_equal(P0a, P0b)                                # the device draw depends on random_seed only
    assert rel_err(Pa, Pb) < 1e-5 and rel_err(Qa, Qb) < 1e-5, (rel_err(Pa, Pb), rel_err(Qa, Qb))
    assert abs(la - lb) <= 1e-5 * abs(lb)


@pytest.mark.parametrize("resident", [True, False])
def test_plsi_inherit_carries_rows_into_training(cuda_lib, clustered, tmp_path, resident):
    from buffalo import aux
    prev = make_plsi(clustered, "inh_prev", num_iters=3, d=16, validation={})
    prev.initialize()
    prev.train()
    path = str(tmp_path / "prev.bin")
    prev.save(path)
    inherit = aux.Option({"model_path": path, "inherit_user": True, "inherit_item": True})
    m = make_plsi(clustered, "inh_%d" % int(resident), num_iters=1, d=16, random_seed=99, inherit_opt=inherit,
                  _b200_resident=resident, validation={})
    m.initialize()
    assert np.array_equal(m.P, prev.P) and np.array_equal(m.Q, prev.Q)
    P0, Q0 = m.P.copy(), m.Q.copy()
    ret = m.train()
    grp = m.data.get_group("rowwise")
    indptr = np.asarray(grp["indptr"][:], dtype=np.int64)
    n = int(indptr[-1])
    keys = np.asarray(grp["key"][:n], dtype=np.int32)
    vals = np.asarray(grp["val"][:n], dtype=np.float32)
    Po, Qo, lo = oracle_iteration(P0, Q0, indptr, keys, vals, m.opt.alpha1, m.opt.alpha2)
    assert rel_err(m.P, Po) < TOL and rel_err(m.Q, Qo) < TOL, (rel_err(m.P, Po), rel_err(m.Q, Qo))
    assert abs(ret["train_loss"] - lo / float(np.sum(vals, dtype=np.float64))) <= TOL * abs(ret["train_loss"])


def test_oracle_holder_protocol_matches_backend(cuda_lib):
    """The holder call sequence of buffalo/algo/plsi.py:_iterate on the backend and on the oracle, three iterations."""
    from buffalo_b200 import backend
    from tests.helpers import make_csr
    U, I, d = 500, 400, 12
    indptr, keys, vals, _ = make_csr(U, I, 8000, seed=21, empty_rows=30)
    g, o = backend.CuPLSI(), OraclePLSI()
    assert g.init(dict(d=d))
    o.init(dict(d=d))
    Pg, Qg = random_factors(U, d, 1, axis=1), random_factors(I, d, 2, axis=0)
    Po, Qo = Pg.copy(), Qg.copy()
    g.set_model(Pg, Qg)
    o.initialize_model(Po, Qo)
    for _ in range(3):
        g.reset()
        o.reset()
        lg = g.partial_update(0, U, indptr, keys, vals)
        lo = o.partial_update(0, U, indptr, keys, vals)
        g.normalize(1.0, 1.0)
        o.normalize(1.0, 1.0)
        g.swap()
        o.swap()
        assert abs(lg - lo) <= TOL * abs(lo)
    assert rel_err(Pg, Po) < TOL and rel_err(Qg, Qo) < TOL
    g.release()

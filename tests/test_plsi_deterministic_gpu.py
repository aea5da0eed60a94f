"""Deterministic pLSI on the GPU: the item pass over the colwise CSR (with a hot item cut into several segments), the
row pass without atomics and the fixed-order loss, through the host ABI, the device-resident ABI and buffalo.PLSI."""
import numpy as np
import pytest

from tests.helpers import make_csr, rel_err, transpose_csr
from tests.plsi_ref import oracle_iteration, random_factors
from tests.test_plsi_gpu import clustered, make_plsi  # noqa: F401  (the planted-cluster fixture and its trainer)

pytestmark = pytest.mark.gpu

TOL = 1e-4
SEGMENT = 4096


@pytest.fixture(scope="module")
def det_csr():
    """16000 users x 60000 items: empty user rows, 1-nnz rows, one row of 50000 nnz, 100 items nobody touched, and a
    hot item held by 13000 rows: more than three segments of 4096 entries."""
    rng = np.random.default_rng(23)
    U, I = 16000, 60000
    hot = I - 101
    lens = rng.integers(0, 40, U)
    lens[rng.choice(U, 300, replace=False)] = 0
    lens[[7, 8, 9]] = 1
    lens[11] = 50000
    live = np.flatnonzero(lens > 1)
    hot_rows = set(rng.choice(live, 13000, replace=False).tolist())
    rows = []
    for x, n in enumerate(lens):
        r = rng.choice(hot, size=int(n), replace=False).tolist() if n else []
        if x in hot_rows:
            r.append(hot)
        rows.append(np.sort(np.asarray(r, dtype=np.int64)))
    keys = np.concatenate(rows).astype(np.int32)
    indptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
    ints = rng.integers(1, 6, len(keys)).astype(np.float32)
    logn = rng.lognormal(0.0, 1.5, len(keys)).astype(np.float32)
    vals = {"ints": ints, "lognormal": logn}
    col = {k: transpose_csr(indptr, keys, v, U, I) for k, v in vals.items()}
    clens = np.diff(col["ints"][0], prepend=0)
    assert clens[hot] > 3 * SEGMENT and (clens[-100:] == 0).all()
    return dict(U=U, I=I, indptr=indptr, keys=keys, vals=vals, col=col)


def chunk(indptr, keys, vals, a, b):
    beg = 0 if a == 0 else int(indptr[a - 1])
    end = int(indptr[b - 1]) if b > 0 else 0
    k = np.ascontiguousarray(keys[beg:end]) if end > beg else np.zeros(1, np.int32)
    v = np.ascontiguousarray(vals[beg:end]) if end > beg else np.zeros(1, np.float32)
    return k, v


def holder_run(P, Q, indptr, keys, vals, col, iters=1, rbounds=None, cbounds=None, deterministic=True,
               alpha1=1.0, alpha2=1.0):
    """iters iterations through the holder ABI: reset / partial_update_items per colwise chunk (deterministic mode) /
    partial_update per rowwise chunk / normalize / swap.  Returns (P, Q, per-iteration losses)."""
    from buffalo_b200 import backend
    cind, ckeys, cvals = col
    g = backend.CuPLSI()
    assert g.init(dict(d=P.shape[1], deterministic=deterministic))
    P1, Q1 = P.copy(), Q.copy()
    g.set_model(P1, Q1)
    rbounds = rbounds or [0, P.shape[0]]
    cbounds = cbounds or [0, Q.shape[0]]
    losses = []
    for _ in range(iters):
        g.reset()
        if deterministic:
            for a, b in zip(cbounds[:-1], cbounds[1:]):
                g.partial_update_items(a, b, cind, *chunk(cind, ckeys, cvals, a, b))
        loss = 0.0
        for a, b in zip(rbounds[:-1], rbounds[1:]):
            loss += g.partial_update(a, b, indptr, *chunk(indptr, keys, vals, a, b))
        g.normalize(alpha1, alpha2)
        g.swap()
        losses.append(loss)
    return P1, Q1, losses


def device_run(P, Q, indptr, keys, vals, col, iters=1, rranges=None, iranges=None):
    """iters deterministic iterations through the device-resident ABI; returns (P, Q, losses)."""
    import torch
    from buffalo_b200 import backend
    d = P.shape[1]
    g = backend.CuPLSI()
    assert g.init(dict(d=d, deterministic=True))
    vdim = g.get_vdim()
    dev = torch.device("cuda", 0)
    tP = torch.zeros((P.shape[0], vdim), dtype=torch.float32, device=dev)
    tQ = torch.zeros((Q.shape[0], vdim), dtype=torch.float32, device=dev)
    tP[:, :d], tQ[:, :d] = torch.from_numpy(P).to(dev), torch.from_numpy(Q).to(dev)
    g.bind_factors(tP, tQ)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)    # noqa: E731
    g.bind_csr(t(indptr), t(keys), t(vals))
    g.bind_colwise_csr(*(t(a) for a in col))
    rranges = rranges or [(0, P.shape[0])]
    iranges = iranges or [(0, Q.shape[0])]
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    losses = []
    for _ in range(iters):
        loss.zero_()
        for a, b in iranges:
            g.update_items_device(a, b)
        for a, b in rranges:
            g.update_device(a, b, loss)
        g.normalize_device(1.0, 1.0)
        g.swap_device()
        losses.append(float(loss.item()))
    return tP[:, :d].cpu().numpy(), tQ[:, :d].cpu().numpy(), losses


# ---- (a) one iteration against the float32 oracle ------------------------------------------------------------------
@pytest.mark.parametrize("vals", ["ints", "lognormal"])
@pytest.mark.parametrize("d", [1, 3, 20, 64, 100, 128, 256, 512])
def test_one_iteration_matches_oracle(cuda_lib, det_csr, d, vals):
    c = det_csr
    P, Q = random_factors(c["U"], d, d, axis=1), random_factors(c["I"], d, d + 1, axis=0)
    v = c["vals"][vals]
    Pg, Qg, (lg,) = holder_run(P, Q, c["indptr"], c["keys"], v, c["col"][vals])
    Po, Qo, lo = oracle_iteration(P, Q, c["indptr"], c["keys"], v)
    assert rel_err(Pg, Po) < TOL and rel_err(Qg, Qo) < TOL, (rel_err(Pg, Po), rel_err(Qg, Qo))
    assert abs(lg - lo) <= TOL * abs(lo), (lg, lo)
    assert np.isfinite(Pg).all() and np.isfinite(Qg).all()


# ---- (b) + (c) reproducible, and the same in both feeding modes and under any chunking ---------------------------
def test_runs_repeat_bitwise_and_modes_agree(cuda_lib, det_csr):
    c = det_csr
    d = 20
    v = c["vals"]["lognormal"]
    P, Q = random_factors(c["U"], d, 5, axis=1), random_factors(c["I"], d, 6, axis=0)
    args = (P, Q, c["indptr"], c["keys"], v, c["col"]["lognormal"])
    res1, res2 = device_run(*args, iters=5), device_run(*args, iters=5)
    ch1 = holder_run(*args, iters=5, rbounds=[0, 1000, 2000, c["U"]], cbounds=[0, 30000, c["I"]])
    ch2 = holder_run(*args, iters=5, rbounds=[0, 1000, 2000, c["U"]], cbounds=[0, 30000, c["I"]])
    for a, b in ((res1, res2), (ch1, ch2)):
        assert np.array_equal(a[0], b[0]) and np.array_equal(a[1], b[1]) and np.array_equal(a[2], b[2])
    assert np.array_equal(res1[0], ch1[0]) and np.array_equal(res1[1], ch1[1])
    for lr, lc in zip(res1[2], ch1[2]):
        assert abs(lr - lc) <= 1e-12 * abs(lc), (lr, lc)
    # other chunk bounds on either side, a hot-item chunk of its own, and split device ranges
    hot = c["I"] - 101
    ch3 = holder_run(*args, iters=5, rbounds=[0, 5, 11, 12, 7000, 7001, c["U"]],
                     cbounds=[0, 1, hot, hot + 1, 59950, c["I"]])
    res3 = device_run(*args, iters=5, rranges=[(0, 12), (12, 9000), (9000, c["U"])],
                      iranges=[(0, hot), (hot, hot + 1), (hot + 1, c["I"])])
    for X in (ch3, res3):
        assert np.array_equal(X[0], ch1[0]) and np.array_equal(X[1], ch1[1])
        for lx, lc in zip(X[2], ch1[2]):
            assert abs(lx - lc) <= 1e-12 * abs(lc), (lx, lc)


# ---- (d) close to the default mode on random data ------------------------------------------------------------------
@pytest.mark.parametrize("d", [8, 100])
def test_close_to_default_mode(cuda_lib, d):
    U, I = 3000, 2000
    indptr, keys, vals, _ = make_csr(U, I, 90000, seed=41, empty_rows=50)
    col = transpose_csr(indptr, keys, vals, U, I)
    P, Q = random_factors(U, d, 7, axis=1), random_factors(I, d, 8, axis=0)
    Pd, Qd, (ld,) = holder_run(P, Q, indptr, keys, vals, col)
    Pa, Qa, (la,) = holder_run(P, Q, indptr, keys, vals, col, deterministic=False)
    assert rel_err(Pd, Pa) < 1e-5 and rel_err(Qd, Qa) < 1e-5, (rel_err(Pd, Pa), rel_err(Qd, Qa))
    assert abs(ld - la) <= 1e-12 * abs(la)


# ---- (e) only the order of the item sums differs ------------------------------------------------------------------
@pytest.mark.parametrize("d", [1, 20, 100, 128, 256, 512])
def test_bitwise_default_when_items_occur_once(cuda_lib, d):
    """Every item occurs in at most one row, so each new item row is one product in both modes: the modes must agree
    bit for bit, P included (its rounding is the same product-then-sum)."""
    rng = np.random.default_rng(d)
    U, I = 2500, 40000
    lens = rng.integers(0, 25, U)
    lens[[3, 4]] = 0, 1
    perm = rng.permutation(I)[:int(lens.sum())]
    indptr = np.cumsum(lens).astype(np.int64)
    keys = np.concatenate([np.sort(perm[b - n:b]) for b, n in zip(indptr, lens)]).astype(np.int32)
    vals = rng.lognormal(0.0, 1.0, len(keys)).astype(np.float32)
    col = transpose_csr(indptr, keys, vals, U, I)
    P, Q = random_factors(U, d, 9, axis=1), random_factors(I, d, 10, axis=0)
    Pd, Qd, (ld,) = holder_run(P, Q, indptr, keys, vals, col)
    Pa, Qa, (la,) = holder_run(P, Q, indptr, keys, vals, col, deterministic=False)
    assert np.array_equal(Pd, Pa) and np.array_equal(Qd, Qa)
    assert abs(ld - la) <= 1e-12 * abs(la)


# ---- (g) call order and shapes --------------------------------------------------------------------------------------
def test_item_pass_after_row_pass_is_a_state_error(cuda_lib):
    import torch
    from buffalo_b200 import backend
    from buffalo_b200._cabi import BackendError
    U, I, d = 300, 200, 12
    indptr, keys, vals, _ = make_csr(U, I, 3000, seed=5)
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
    P, Q = random_factors(U, d, 1, axis=1), random_factors(I, d, 2, axis=0)
    g = backend.CuPLSI()
    assert g.init(dict(d=d, deterministic=True))
    g.set_model(P.copy(), Q.copy())
    g.reset()
    g.partial_update_items(0, I, cind, ckeys, cvals)
    g.partial_update(0, U, indptr, keys, vals)
    with pytest.raises(BackendError, match="status 3"):
        g.partial_update_items(0, I, cind, ckeys, cvals)
    g.reset()                                         # a new iteration may run the item pass again
    g.partial_update_items(0, I, cind, ckeys, cvals)
    # without the option there is no item pass
    a = backend.CuPLSI()
    assert a.init(dict(d=d))
    a.set_model(P.copy(), Q.copy())
    a.reset()
    with pytest.raises(BackendError, match="status 3"):
        a.partial_update_items(0, I, cind, ckeys, cvals)
    # device path: after update_device, until swap_device
    dev = torch.device("cuda", 0)
    t = lambda x: torch.from_numpy(np.ascontiguousarray(x)).to(dev)    # noqa: E731
    h = backend.CuPLSI()
    assert h.init(dict(d=d, deterministic=True))
    vdim = h.get_vdim()
    tP, tQ = torch.zeros((U, vdim), device=dev), torch.zeros((I, vdim), device=dev)
    tP[:, :d], tQ[:, :d] = t(P), t(Q)
    h.bind_factors(tP, tQ)
    h.bind_csr(t(indptr), t(keys), t(vals))
    with pytest.raises(BackendError, match="status 3"):
        h.update_items_device(0, I)                   # no colwise CSR bound yet
    with pytest.raises(BackendError, match="status 4"):
        h.bind_colwise_csr(t(cind[:-1]), t(ckeys), t(cvals))
    h.bind_colwise_csr(t(cind), t(ckeys), t(cvals))
    h.update_items_device(0, I)
    h.update_device(0, U)
    with pytest.raises(BackendError, match="status 3"):
        h.update_items_device(0, I)
    h.normalize_device(1.0, 1.0)
    h.swap_device()
    h.update_items_device(0, I)
    torch.cuda.synchronize()


def test_segment_length_constant(cuda_lib):
    from buffalo_b200 import backend
    assert backend.CuPLSI().item_segment_len() == SEGMENT


# ---- (f) buffalo.PLSI(..., deterministic=True) --------------------------------------------------------------------
def test_plsi_deterministic_training(cuda_lib, clustered, tmp_path):
    from buffalo import PLSI
    from buffalo.misc import log
    log.set_log_level(log.WARN)
    runs = []
    for name, kw in (("det_a", {}), ("det_b", {}), ("det_c", dict(_b200_resident=False, _batch_mb=1))):
        m = make_plsi(clustered, name, num_iters=10, d=20, deterministic=True, **kw)
        m.initialize()
        ret = m.train()
        runs.append((m, ret))
    (ma, ra), (mb, rb), (mc, rc) = runs
    assert np.array_equal(ma.P, mb.P) and np.array_equal(ma.Q, mb.Q) and ra["train_loss"] == rb["train_loss"]
    assert np.array_equal(ma.P, mc.P) and np.array_equal(ma.Q, mc.Q)
    assert abs(ra["train_loss"] - rc["train_loss"]) <= 1e-12 * abs(ra["train_loss"])
    res = ma.get_validation_results()
    assert res["ndcg"] > 0.03 and res["map"] > 0.02, res
    np.testing.assert_allclose(ma.P.sum(axis=1), 1.0, atol=1e-4)
    np.testing.assert_allclose(ma.Q.sum(axis=0), 1.0, atol=1e-4)
    path = str(tmp_path / "plsi_det.bin")
    ma.save(path)
    other = PLSI.new(path)
    assert np.array_equal(other.P, ma.P) and np.array_equal(other.Q, ma.Q) and other.opt.deterministic is True

"""Deterministic BPRMF / WARP (option `deterministic`): the gradient sums of an epoch are taken in a fixed order, so the
same inputs give the same bits on every run and under every chunking of the rows.

Per configuration and epoch, five deterministic runs -- ShardedSGD(world=1), add_jobs_device on the three uneven
ranges of ranged_csr and on one range, the host add_jobs on the ranges and in one chunk -- must agree bitwise in the
gradient accumulators (after reduce_items_device), the factors, the probe loss and the WARP loss statistic.  Against
references they are held to the bars of test_sgd_resident_gpu.py: gradient 1e-5 against the fp64 mirror, factors 1e-4
against the C oracle, probe loss 1e-5, the default (atomics) mode 1e-5 after the first epoch and the oracle bar after the
later ones, with its ill-conditioned-element rule."""
import numpy as np
import pytest

from tests.helpers import csr_from_lengths, init_factors
from tests.test_sgd_gpu import _hr_at_10, _planted, sgd_opt
from tests.test_sgd_resident_gpu import (DeviceRun, check_grad, host_run, ill_conditioned, key_slice, masked_err,
                                         probe_triples, ranged_csr, scalar_err)

pytestmark = pytest.mark.gpu

ORACLE_TOL = 1e-4
PATH_TOL = 1e-5


def _same(label, runs):
    """every run's arrays bitwise equal to the first run's"""
    base = runs[0][1]
    for name, arrs in runs[1:]:
        for k, (x, y) in enumerate(zip(base, arrs)):
            assert np.array_equal(np.atleast_1d(x).view(np.uint8), np.atleast_1d(y).view(np.uint8)), (label, name, k)


def det_epochs(kind, opt, indptr, keys, ranges, I, seed, epochs=3, cum=None):
    import oracle
    from oracle import np_mirror
    warp = kind == "warp"
    d = opt["d"]
    U, nnz = len(indptr), len(keys)
    dopt = dict(opt, deterministic=True)
    scale = d ** -0.25
    P = init_factors(U, d, d, seed + 1, scale=scale, signed=True)
    Q = init_factors(I, d, d, seed + 2, scale=scale, signed=True)
    Qb = np.zeros((I, 1), np.float32) if warp else init_factors(I, 1, 1, seed + 3, scale=0.3, signed=True)
    sharded = DeviceRun(kind, dopt, P, Q, Qb, indptr, keys, cum)
    ranged = DeviceRun(kind, dopt, P, Q, Qb, indptr, keys, cum)
    whole = DeviceRun(kind, dopt, P, Q, Qb, indptr, keys, cum)
    default = DeviceRun(kind, opt, P, Q, Qb, indptr, keys, cum)
    h, (Ph, Qh, Qbh) = host_run(kind, dopt, P, Q, Qb, nnz, cum)
    h1, (Ph1, Qh1, Qbh1) = host_run(kind, dopt, P, Q, Qb, nnz, cum)
    o = oracle.OracleSGD(warp=warp, use_lut=False)
    o.init(opt)
    Po, Qo, Qbo = P.copy(), Q.copy(), Qb.copy()
    o.initialize_model(Po, Qo, Qbo, nnz)
    if cum is not None:
        o.set_cumulative_table(cum, len(cum))
    probe = probe_triples(indptr, keys, I, 400, seed)
    ot, on = np.zeros(nnz, np.int32), np.zeros(nnz, np.int32)
    diverged = default_diverged = False
    pcn = opt["per_coordinate_normalize"]
    mP, mQ, mB = np.zeros((U, d), bool), np.zeros((I, d), bool), np.zeros((I, 1), bool)
    for e in range(epochs):
        lab = "%s d=%d epoch %d" % (kind, d, e)
        b = ranged
        P0, Q0, Qb0, gP0, gQ0, gQb0, cP0, cQ0 = b.host(b.P, b.Q, b.Qb, b.gP, b.gQ, b.gQb, b.cP, b.cQ)
        stats0 = [r.g.read_stats() for r in (ranged, whole)]
        if warp:
            b.trials.fill_(-2)
        else:
            import torch
            tri = [torch.zeros(nnz * opt["num_negative_samples"], dtype=torch.int32, device="cuda") for _ in range(3)]
            b.g.sample_device(0, U, *tri)
            us, ps, ns = b.host(*tri)
        if warp:
            default.trials.fill_(-2)
        sharded.drv.epoch()
        default.drv.epoch()
        for lo, hi in ranges:
            ranged.g.add_jobs_device(lo, hi)
            beg, end = key_slice(indptr, keys, lo, hi)
            k = np.ascontiguousarray(keys[beg:end])
            h.add_jobs(lo, hi, indptr, k)
            if warp:
                o.add_jobs(lo, hi, indptr, k, trials_out=ot[beg:end], negs_out=on[beg:end])
            else:
                o.add_jobs(lo, hi, indptr, k)
        whole.g.add_jobs_device(0, U)
        h1.add_jobs(0, U, indptr, keys)
        ranged.g.reduce_items_device()
        whole.g.reduce_items_device()
        grads = [r.host(r.gP, r.gQ, r.gQb, r.cP, r.cQ) for r in (ranged, whole)]
        _same(lab + " gradients", [("ranges", grads[0]), ("one range", grads[1])])
        stats1 = [r.g.read_stats() for r in (ranged, whole)]
        assert stats1[0][0] - stats0[0][0] == stats1[1][0] - stats0[1][0], (lab, stats0, stats1)
        gP1, gQ1, gQb1, cP1, cQ1 = grads[0]
        Pd, Qd = P0[:, :d], Q0[:, :d]
        if warp:
            gt, gn = b.host(b.trials, b.negs)
            wgP, wgQ, wcP, wcQ, wloss, wupd = np_mirror.warp_accumulate(
                Pd, Qd, indptr, keys, gt, gn, opt["reg_u"], opt["reg_i"], opt["reg_j"], opt["threshold"],
                opt["score_func"])
            if not pcn:
                wcP, wcQ = 0 * wcP, 0 * wcQ
            assert scalar_err(stats1[0][0] - stats0[0][0], wloss) < 1e-4, (lab, stats1, stats0, wloss)
            assert stats1[0][1] - stats0[0][1] == wupd, lab
            mism = (gt != ot) | (gn != on)
            assert mism.mean() < 2e-3, (lab, mism.mean())
            diverged = diverged or bool(mism.any())
            # the default mode's rank sampling compares fp32 scores too: a decision within rounding of the margin
            dt, dn = default.host(default.trials, default.negs)
            default_diverged = default_diverged or bool(((dt != gt) | (dn != gn)).any())
        else:
            wgP, wgQ, wgQb, wcP, wcQ = np_mirror.bpr_accumulate(
                Pd, Qd, Qb0, us, ps, ns, use_bias=opt["use_bias"], update_i=opt["update_i"], update_j=opt["update_j"],
                per_coordinate_normalize=pcn, num_negative_samples=opt["num_negative_samples"])
            check_grad(lab + " gQb", gQb1, gQb0, wgQb[:, 0])
        check_grad(lab + " gP", gP1[:, :d], gP0[:, :d], wgP)
        check_grad(lab + " gQ", gQ1[:, :d], gQ0[:, :d], wgQ)
        assert np.array_equal(cP1 - cP0, wcP) and np.array_equal(cQ1 - cQ0, wcQ), (lab, "sample counters")
        mP |= ill_conditioned(gP1[:, :d], cP1, Pd, opt["reg_u"], pcn)
        mQ |= ill_conditioned(gQ1[:, :d], cQ1, Qd, opt["reg_i"], pcn)
        if not warp:
            mB |= ill_conditioned(gQb1, cQ1, Qb0, opt["reg_b"], pcn)
        assert mP.sum() + mQ.sum() + mB.sum() <= 5, (lab, mP.sum(), mQ.sum(), mB.sum())
        for r in (ranged, whole):
            r.g.update_parameters_device()
        h.update_parameters()
        h1.update_parameters()
        o.update_parameters()
        runs = [("sharded", sharded.host(sharded.P, sharded.Q, sharded.Qb)),
                ("ranges", ranged.host(ranged.P, ranged.Q, ranged.Qb)),
                ("one range", whole.host(whole.P, whole.Q, whole.Qb)),
                ("host ranges", (Ph, Qh, Qbh)), ("host one chunk", (Ph1, Qh1, Qbh1))]
        _same(lab + " factors", runs)
        losses = [(n, [np.float64(x.compute_loss(*probe))]) for n, x in
                  (("sharded", sharded.g), ("ranges", ranged.g), ("one range", whole.g), ("host", h), ("host1", h1))]
        _same(lab + " probe loss", losses)
        Pb, Qb_, Qbb = runs[1][1]
        Pdf, Qdf, Qbdf = default.host(default.P, default.Q, default.Qb)
        if not diverged:
            errs = masked_err(Pb[:, :d], Po, mP), masked_err(Qb_[:, :d], Qo, mQ), masked_err(Qbb, Qbo, mB)
            assert max(errs) < ORACLE_TOL, (lab, "vs oracle", errs)
        if not diverged and not default_diverged:
            errs = (masked_err(Pdf[:, :d], Pb[:, :d], mP), masked_err(Qdf[:, :d], Qb_[:, :d], mQ),
                    masked_err(Qbdf, Qbb, mB))
            # after the first step the two modes' rounding differences go through the later Adagrad / Adam steps, whose
            # g / sqrt(v) magnifies them where v is small: from then on the oracle bar
            strict = e == 0 and not (mP.any() or mQ.any() or mB.any())
            assert max(errs) < (PATH_TOL if strict else ORACLE_TOL), (lab, "default", errs)
        lg = losses[0][1][0]
        if warp:
            lm = np_mirror.warp_loss(Pb[:, :d], Qb_[:, :d], *probe, threshold=opt["threshold"], score=opt["score_func"])
            assert abs(lg - lm) <= 2.0 / len(probe[0]) + 1e-12, (lab, lg, lm)
        else:
            lm = np_mirror.bpr_loss(Pb[:, :d], Qb_[:, :d], Qbb, *probe, use_bias=opt["use_bias"])
            assert scalar_err(lg, lm) < 1e-5 and scalar_err(lg, default.g.compute_loss(*probe)) < 1e-5, (lab, lg, lm)
    return runs


CONFIGS = {
    "warp-dot-adagrad": ("warp", dict(optimizer="adagrad", score_func="dot")),
    "warp-l2-adam-pcn": ("warp", dict(optimizer="adam", score_func="l2", per_coordinate_normalize=True)),
    "bpr-adagrad-bias-neg2-pop": ("bpr", dict(optimizer="adagrad", num_negative_samples=2, sampling_power=1.0)),
    "bpr-adam-pcn": ("bpr", dict(optimizer="adam", per_coordinate_normalize=True)),
    "bpr-no-update-j": ("bpr", dict(optimizer="adagrad", update_j=False)),
}


def _opt(kind, d, kw):
    kw = dict(kw)
    kw.setdefault("num_negative_samples", 1)
    return sgd_opt(d=d, num_iters=3, max_trials=30, reg_u=0.01, reg_i=0.02, reg_j=0.03, use_bias=(kind == "bpr"), **kw)


def _cum(keys, I, kw):
    p = int(kw.get("sampling_power", 0))
    return np.cumsum(np.bincount(keys, minlength=I).astype(np.int64) ** p).astype(np.int64) if p else None


# every configuration at d = 3 and 30 (NV = 1, vdim != d); the wider rows (NV = 2 and 4, d = 129 with one active lane in
# its second column group) at the width / optimizer pairs test_sgd_resident_gpu.py holds to the oracle bar
CASES = [(n, d) for n in CONFIGS for d in (3, 30)] + [
    ("warp-dot-adagrad", 129), ("warp-dot-adagrad", 256), ("warp-dot-adagrad", 512), ("warp-l2-adam-pcn", 129),
    ("bpr-adagrad-bias-neg2-pop", 256), ("bpr-adagrad-bias-neg2-pop", 512), ("bpr-adam-pcn", 129),
    ("bpr-no-update-j", 256)]


@pytest.mark.parametrize("name,d", CASES)
def test_repeatable_across_drivers(cuda_lib, name, d):
    kind, kw = CONFIGS[name]
    U, I = 300, 400
    indptr, keys, ranges = ranged_csr(U, I, d, 10)
    opt = _opt(kind, d, kw)
    first = det_epochs(kind, opt, indptr, keys, ranges, I, seed=d, cum=_cum(keys, I, kw))
    second = det_epochs(kind, opt, indptr, keys, ranges, I, seed=d, cum=_cum(keys, I, kw))
    _same("%s d=%d rerun" % (name, d), [first[1], second[1]])


@pytest.mark.parametrize("kind", ["bpr", "warp"])
def test_long_rows_and_hot_items_span_segments(cuda_lib, kind):
    """A user with more than three segments of samples and an item that is a positive (and, for BPR, a popularity-drawn
    negative) more than two segments' worth of times: the combine path, still bitwise repeatable and at parity."""
    from buffalo_b200 import backend
    seg = backend.CuSGD.segment_len()
    rng = np.random.default_rng(3)
    U, I = 3 * seg, 3 * seg + 500
    lengths = rng.integers(1, 4, U)
    lengths[5] = 3 * seg + 100
    indptr, keys, _ = csr_from_lengths(lengths, I, rng)
    beg = np.concatenate([[0], indptr[:-1]])
    for u in range(U):     # item 0 becomes a positive of every row
        if 0 not in keys[beg[u]:indptr[u]]:
            keys[beg[u]] = 0
        keys[beg[u]:indptr[u]] = np.sort(keys[beg[u]:indptr[u]])
    a = U // 3
    ranges = [(0, a), (a, a + 1), (a + 1, U)]
    kw = dict(optimizer="adagrad", sampling_power=1.0) if kind == "bpr" else dict(optimizer="adagrad")
    opt = _opt(kind, 30, kw)
    assert np.sum(keys == 0) > 2 * seg
    first = det_epochs(kind, opt, indptr, keys, ranges, I, seed=11, epochs=2, cum=_cum(keys, I, kw))
    second = det_epochs(kind, opt, indptr, keys, ranges, I, seed=11, epochs=2, cum=_cum(keys, I, kw))
    _same("segments rerun", [first[1], second[1]])


def test_bitwise_equal_to_default_when_rows_get_one_term(cuda_lib):
    """BPR with one positive per user and draws that collide neither with each other nor with the positives: every
    gradient row receives one term, so the fixed order and the atomics give the same bits."""
    import torch
    U, I, d = 120, 400000, 30
    rng = np.random.default_rng(0)
    keys = rng.permutation(I)[:U].astype(np.int32)
    indptr = np.arange(1, U + 1, dtype=np.int64)
    for seed in range(1, 50):
        opt = _opt("bpr", d, dict(optimizer="adagrad", random_seed=seed))
        P = init_factors(U, d, d, 1, scale=d ** -0.25, signed=True)
        Q = init_factors(I, d, d, 2, scale=d ** -0.25, signed=True)
        Qb = init_factors(I, 1, 1, 3, scale=0.3, signed=True)
        det = DeviceRun("bpr", dict(opt, deterministic=True), P, Q, Qb, indptr, keys, None)
        tri = [torch.zeros(U, dtype=torch.int32, device="cuda") for _ in range(3)]
        det.g.sample_device(0, U, *tri)
        ns = det.host(tri[2])[0]
        if len(set(ns.tolist()) | set(keys.tolist())) == 2 * U:
            break
    else:
        pytest.fail("no collision-free seed")
    ref = DeviceRun("bpr", opt, P, Q, Qb, indptr, keys, None)
    for r in (det, ref):
        r.g.add_jobs_device(0, U)
    det.g.reduce_items_device()
    _same("one term", [("det", det.host(det.gP, det.gQ, det.gQb)), ("default", ref.host(ref.gP, ref.gQ, ref.gQb))])
    for r in (det, ref):
        r.g.update_parameters_device()
    _same("one term step", [("det", det.host(det.P, det.Q, det.Qb)), ("default", ref.host(ref.P, ref.Q, ref.Qb))])


def test_explicit_triples_refused(cuda_lib):
    import torch
    from buffalo_b200 import _cabi, backend
    g = backend.CuSGD("bpr")
    assert g.init(sgd_opt(d=8, optimizer="adagrad", deterministic=True))
    dev = torch.device("cuda:0")
    g.bind_factors(torch.zeros(4, 8, device=dev), torch.zeros(6, 8, device=dev), torch.zeros(6, device=dev), 4)
    t = torch.zeros(2, dtype=torch.int32, device=dev)
    with pytest.raises(_cabi.BackendError):
        g.apply_triples_device(t, t, t, 0.1)
    plain = backend.CuSGD("bpr")
    assert plain.init(sgd_opt(d=8, optimizer="adagrad"))
    plain.bind_factors(torch.zeros(4, 8, device=dev), torch.zeros(6, 8, device=dev), torch.zeros(6, device=dev), 4)
    with pytest.raises(_cabi.BackendError):
        plain.reduce_items_device()


def _train(cls_name, tmp_path, batch_mb, m):
    import buffalo
    from buffalo.data import MatrixMarketOptions
    dopt = MatrixMarketOptions().get_default_option()
    dopt.input.main = m
    dopt.data.path = str(tmp_path / ("mm_%s_%d.h5py" % (cls_name, batch_mb)))
    dopt.data.validation.p = 0.1
    dopt.data.validation.max_samples = 200
    dopt.data.batch_mb = batch_mb
    from buffalo_b200.misc import aux
    opt = getattr(buffalo, cls_name + "Option")().get_default_option()
    opt.update(d=20, num_iters=3, random_seed=7, optimizer="adagrad", lr=0.05, deterministic=True,
               validation=aux.Option({"topk": 10}), evaluation_period=1)
    # the database's validation split draws from the global NumPy state: the same state gives the same split
    np.random.seed(7)
    algo = getattr(buffalo, cls_name)(opt, data_opt=dopt)
    algo.initialize()
    ret = algo.train()
    return algo.P.copy(), algo.Q.copy(), algo.Qb.copy(), ret


@pytest.mark.parametrize("cls_name", ["BPRMF", "WARP"])
def test_public_api_repeatable(cuda_lib, tmp_path, cls_name):
    """Two fresh trainings with random_seed = 7 give the same bits; a third with another batch_mb (other chunk
    bounds) too."""
    import scipy.sparse
    rng = np.random.default_rng(1)
    U, I = 3000, 800
    indptr, keys, _ = csr_from_lengths(rng.integers(0, 30, U), I, rng)
    m = scipy.sparse.csr_matrix((np.ones(len(keys), np.float32), keys, np.concatenate([[0], indptr])), shape=(U, I))
    a = _train(cls_name, tmp_path, 1024, m)
    b = _train(cls_name, tmp_path, 1024, m)
    c = _train(cls_name, tmp_path, 1, m)
    assert "val_ndcg" in a[3] and "train_loss" in a[3], a[3]
    for name, x in (("rerun", b), ("batch_mb", c)):
        _same(cls_name + " " + name, [("first", a[:3]), (name, x[:3])])
        assert a[3] == x[3], (name, a[3], x[3])


def test_hr10_in_the_oracle_band(cuda_lib):
    """WARP deterministic on the planted matrix over 5 seeds: HR@10 within the band test_sgd_gpu.py allows against the
    oracle (3 combined standard errors, floor 0.02)."""
    import oracle
    from tests.test_sgd_gpu import make_pair
    U, I, indptr, keys, held_item = _planted()
    users = np.nonzero(held_item >= 0)[0]
    users = np.random.default_rng(0).choice(users, size=1500, replace=False)
    d, epochs = 32, 6
    hr_g, hr_o = [], []
    for seed in (1, 2, 3, 4, 5):
        opt = sgd_opt(d=d, optimizer="adagrad", lr=0.1, random_seed=seed, num_iters=epochs, reg_u=0.01, reg_i=0.01,
                      reg_j=0.01, reg_b=0.01, use_bias=False, max_trials=100)
        P = init_factors(U, d, d, seed, scale=0.05, signed=True)
        Q = init_factors(I, d, d, seed + 10, scale=0.05, signed=True)
        Qb = np.zeros((I, 1), np.float32)
        g, _, (Pg, Qg, _), _ = make_pair("warp", dict(opt, deterministic=True), P, Q, Qb, indptr, keys)
        o = oracle.OracleSGD(warp=True, use_lut=False)
        o.init(dict(opt, num_workers=8))
        Po, Qo, Qbo = P.copy(), Q.copy(), Qb.copy()
        o.initialize_model(Po, Qo, Qbo, len(keys))
        for _ in range(epochs):
            g.add_jobs(0, U, indptr, keys)
            o.add_jobs(0, U, indptr, keys)
            g.update_parameters()
            o.update_parameters()
        g.wait_until_done()
        hr_g.append(_hr_at_10(Pg, Qg, None, indptr, keys, held_item, users))
        hr_o.append(_hr_at_10(Po, Qo, None, indptr, keys, held_item, users))
    mg, mo = float(np.mean(hr_g)), float(np.mean(hr_o))
    se = float(np.sqrt(np.var(hr_o, ddof=1) / 5 + np.var(hr_g, ddof=1) / 5))
    assert mg > 20 * 10.0 / I and abs(mg - mo) <= max(3 * se, 0.02), (hr_g, hr_o)

"""The device-resident BPRMF / WARP path (bind_factors / bind_csr / add_jobs_device / update_parameters_device, the path
`bench.py --algo bpr|warp` times) and the SGD kernels at every row width they are instantiated for, against the fp64
NumPy mirror (oracle/np_mirror.py) and the C oracle.  Worst errors measured on an H100 (700 W) in brackets.

Per epoch and per configuration:
* the accumulate kernels against fp64: the gradient buffers are not cleared by the optimizer step (algo.cc:382-465), so
  the difference across one epoch's accumulate is compared with np_mirror.bpr_accumulate (on the epoch's triples from
  sample_device, a pure function of seed, epoch and positive index) or np_mirror.warp_accumulate (on the kernel's own
  rank-sampling trace).  Bound 1e-5 of the larger of the gradient and the buffer it was added to [7e-7].  Sample
  counters exactly; WARP's running loss sum 1e-4 relative [2e-8], its update count exactly;
* the whole epoch against the C oracle: factors 1e-4 relative max-norm, the bar of test_sgd_gpu.py [2e-5], lr schedule
  to 1e-12, epoch counter, probe losses 1e-5 against the oracle and the mirror [4e-7];
* three GPU drivers -- ShardedSGD(world=1) as in the benchmark, add_jobs_device on three row ranges, the host-pointer
  add_jobs on the same ranges -- agree to 1e-5, and to the oracle bar once an element was excused (its neighbours then
  differ too); they differ only in the order of float atomics [7e-6].
An element whose optimizer input cancels to rounding level (ill_conditioned) is excused from the element-wise
comparisons; at most 5 per run [1, in the d = 384 Adam case].

Widths d = 3 .. 512 cover NV = 1, 2 and 4 of the float4 kernels (NV = ceil(vdim / 128)), vdim != d, and d = 129 whose
second 128-column group has only lane 0 active.  The GPU holds vdim-padded rows, the oracle and the mirror [:, :d]."""
import ctypes as C

import numpy as np
import pytest

from tests.helpers import csr_from_lengths, init_factors, rel_err
from tests.test_sgd_gpu import sgd_opt

pytestmark = pytest.mark.gpu

WIDTHS = (3, 30, 129, 200, 256, 257, 384, 512)
GRAD_TOL = 1e-5      # accumulate vs fp64, relative to max(|gradient|, |buffer before|)
ORACLE_TOL = 1e-4    # factors after the optimizer step vs the C oracle
PATH_TOL = 1e-5      # the three GPU drivers against each other


def ranged_csr(U, I, seed, mean):
    """Rowwise CSR and the three job ranges of an epoch.  Row 0, the last row and ~10 % of the others are empty; the
    middle range holds no positives at all and the last range starts at an empty row > 0."""
    rng = np.random.default_rng(seed)
    lengths = rng.integers(1, 2 * mean, U)
    lengths[rng.choice(U, U // 10, replace=False)] = 0
    a, b = U // 3, U // 3 + 7
    lengths[[0, U - 1]] = 0
    lengths[a:b + 2] = 0
    indptr, keys, _ = csr_from_lengths(lengths, I, rng)
    return indptr, keys, [(0, a), (a, b), (b, U)]


def key_slice(indptr, keys, lo, hi):
    beg = 0 if lo == 0 else int(indptr[lo - 1])
    return beg, int(indptr[hi - 1])


def padded(F, vdim):
    out = np.zeros((F.shape[0], vdim), np.float32)
    out[:, :F.shape[1]] = F
    return out


class DeviceRun(object):
    """One device-resident run set up as benchmarks/sgd_bench.py does: torch factors, bind_factors, bind_csr,
    launch_workers, and the gradient / counter views that ShardedSGD all-reduces for the accumulating optimizers."""

    def __init__(self, kind, opt, P, Q, Qb, indptr, keys, cum):
        import torch
        from buffalo_b200 import backend
        from buffalo_b200.parallel.dist import ShardedSGD
        dev = torch.device("cuda:0")
        U, I = P.shape[0], Q.shape[0]
        self.g = g = backend.CuSGD(kind)
        assert g.init(opt)
        vdim = g.get_vdim()
        self.P, self.Q = torch.from_numpy(padded(P, vdim)).to(dev), torch.from_numpy(padded(Q, vdim)).to(dev)
        self.Qb = torch.from_numpy(Qb.copy()).to(dev)
        shard = ShardedSGD(None, None, self.P, self.Q, self.Qb, indptr)
        g.bind_factors(self.P, self.Q, self.Qb, shard.local_positives(indptr))
        self.indptr, self.keys = torch.from_numpy(indptr).to(dev), torch.from_numpy(keys).to(dev)
        g.bind_csr(self.indptr, self.keys)
        if cum is not None:
            g.set_cumulative_table(cum, len(cum))
        g.launch_workers()
        self.gP, self.gQ = g.grad_tensor(0, (U, vdim)), g.grad_tensor(1, (I, vdim))
        self.gQb = g.grad_tensor(2, (I,))
        self.cP, self.cQ = g.count_tensor(0, U), g.count_tensor(1, I)
        grads = None
        if opt["optimizer"] != "sgd" or kind == "warp":
            grads = [self.gP, self.gQ] + ([self.gQb] if kind == "bpr" else []) + [self.cP, self.cQ]
        if kind == "warp":
            self.trials = torch.zeros(len(keys), dtype=torch.int32, device=dev)
            self.negs = torch.zeros(len(keys), dtype=torch.int32, device=dev)
            g.set_trace(self.trials, self.negs)
        self.drv = ShardedSGD(g.add_jobs_device, g.update_parameters_device, self.P, self.Q, self.Qb, indptr,
                              grads=grads)
        self.drv.begin()

    def host(self, *tensors):
        import torch
        torch.cuda.synchronize()
        return [t.cpu().numpy().copy() for t in tensors]


def host_run(kind, opt, P, Q, Qb, nnz, cum):
    from buffalo_b200 import backend
    g = backend.CuSGD(kind)
    assert g.init(opt)
    vdim = g.get_vdim()
    F = (padded(P, vdim), padded(Q, vdim), Qb.copy())
    g.initialize_model(*F, nnz)
    if cum is not None:
        g.set_cumulative_table(cum, len(cum))
    g.launch_workers()
    return g, F


def check_grad(label, after, before, want):
    """after - before (fp32 buffers) against the fp64 gradient `want`"""
    got = after.astype(np.float64) - before.astype(np.float64)
    scale = max(np.abs(want).max(), np.abs(before).max(), 1e-30)
    err = np.abs(got - want).max() / scale
    assert err < GRAD_TOL, (label, err, np.unravel_index(np.argmax(np.abs(got - want)), got.shape))


def ill_conditioned(grad, cnt, theta, reg, pcn):
    """Elements whose optimizer input g = grad / count - 2 reg theta (algo.cc:399-403) cancels to within 1e-5 of its
    terms.  Summed in another fp32 order such a g can move by a large fraction of itself, and the first Adam / Adagrad
    step g / (|g| + 1e-10) (beta2 = beta1, algo.cc:396) with it when |g| is near 1e-10: no fp32 restatement can
    decide them."""
    gr = grad.astype(np.float64).reshape(len(theta), -1)
    if pcn:
        gr = gr / np.maximum(cnt, 1)[:, None]
    t = 2.0 * reg * theta.astype(np.float64).reshape(gr.shape)
    return np.abs(gr - t) < 1e-5 * (np.abs(gr) + np.abs(t))


def masked_err(X, X0, mask):
    """rel_err over the elements outside `mask`"""
    diff = np.abs(np.asarray(X, np.float64) - np.asarray(X0, np.float64)).reshape(mask.shape)
    return float(np.where(mask, 0.0, diff).max() / max(np.abs(X0).max(), 1e-30))


def scalar_err(got, want):
    return abs(got - want) / max(1.0, abs(want))


def probe_triples(indptr, keys, I, n, seed):
    rng = np.random.default_rng(seed)
    beg = np.concatenate([[0], indptr[:-1]])
    us = rng.choice(np.nonzero(indptr > beg)[0], n).astype(np.int32)
    ps = np.array([keys[rng.integers(beg[u], indptr[u])] for u in us], np.int32)
    return us, ps, rng.integers(0, I, n).astype(np.int32)


def run_epochs(kind, opt, U, I, mean, seed, epochs=3, cum_power=0):
    """Runs the device-resident driver twice (ShardedSGD and direct ranges), the host-pointer path and the oracle in
    lockstep and checks every epoch; see the module docstring."""
    import oracle
    import torch
    from oracle import np_mirror
    d = opt["d"]
    warp = kind == "warp"
    indptr, keys, ranges = ranged_csr(U, I, seed, mean)
    nnz = len(keys)
    scale = d ** -0.25        # scores of order 1: both branches of the logit clamp / several WARP trials occur
    P = init_factors(U, d, d, seed + 1, scale=scale, signed=True)
    Q = init_factors(I, d, d, seed + 2, scale=scale, signed=True)
    Qb = np.zeros((I, 1), np.float32) if warp else init_factors(I, 1, 1, seed + 3, scale=0.3, signed=True)
    cum = None
    if cum_power:
        cum = np.cumsum(np.bincount(keys, minlength=I).astype(np.int64) ** cum_power).astype(np.int64)
    a = DeviceRun(kind, opt, P, Q, Qb, indptr, keys, cum)
    b = DeviceRun(kind, opt, P, Q, Qb, indptr, keys, cum)
    h, (Ph, Qh, Qbh) = host_run(kind, opt, P, Q, Qb, nnz, cum)
    o = oracle.OracleSGD(warp=warp, use_lut=False)
    o.init(opt)
    Po, Qo, Qbo = P.copy(), Q.copy(), Qb.copy()
    o.initialize_model(Po, Qo, Qbo, nnz)
    if cum is not None:
        o.set_cumulative_table(cum, len(cum))
    probe = probe_triples(indptr, keys, I, 400, seed)
    dev = torch.device("cuda:0")
    ot, on = np.zeros(nnz, np.int32), np.zeros(nnz, np.int32)
    diverged = False     # a WARP rank-sampling decision within fp32 rounding of the margin went the other way
    pcn = opt["per_coordinate_normalize"]
    # elements excused from the element-wise comparisons once their optimizer input was ill-conditioned (see
    # ill_conditioned); they must stay a tiny fraction
    mP, mQ, mB = np.zeros((U, d), bool), np.zeros((I, d), bool), np.zeros((I, 1), bool)
    for e in range(epochs):
        lab = "%s d=%d epoch %d" % (kind, d, e)
        P0, Q0, Qb0, gP0, gQ0, gQb0, cP0, cQ0 = b.host(b.P, b.Q, b.Qb, b.gP, b.gQ, b.gQb, b.cP, b.cQ)
        if warp:
            b.trials.fill_(-2)
            stats0 = b.g.read_stats()
        else:
            n = nnz * o.o.num_negative_samples
            tri = [torch.zeros(n, dtype=torch.int32, device=dev) for _ in range(3)]
            b.g.sample_device(0, U, *tri)
            us, ps, ns = b.host(*tri)
            ou, op, on_ = o.sample(0, U, indptr, keys)
            assert np.array_equal(us, ou) and np.array_equal(ps, op) and np.array_equal(ns, on_), lab
        a.drv.epoch()
        lr_start = None
        for lo, hi in ranges:
            b.g.add_jobs_device(lo, hi)
            beg, end = key_slice(indptr, keys, lo, hi)
            k = np.ascontiguousarray(keys[beg:end])
            h.add_jobs(lo, hi, indptr, k)
            if warp:
                o.add_jobs(lo, hi, indptr, k, trials_out=ot[beg:end], negs_out=on[beg:end])
            else:
                o.add_jobs(lo, hi, indptr, k)
            lr_start = o.lr if lr_start is None else lr_start    # ShardedSGD(world=1) makes one job per epoch
        gP1, gQ1, gQb1, cP1, cQ1 = b.host(b.gP, b.gQ, b.gQb, b.cP, b.cQ)
        Pd, Qd = P0[:, :d], Q0[:, :d]
        if warp:
            gt, gn = b.host(b.trials, b.negs)
            assert (gt >= 0).all(), (lab, "positives never visited", np.flatnonzero(gt < 0)[:10])
            m = np_mirror.warp_accumulate(Pd, Qd, indptr, keys, gt, gn, opt["reg_u"], opt["reg_i"], opt["reg_j"],
                                          opt["threshold"], opt["score_func"])
            wgP, wgQ, wcP, wcQ, wloss, wupd = m
            if not opt["per_coordinate_normalize"]:
                wcP, wcQ = 0 * wcP, 0 * wcQ
            stats1 = b.g.read_stats()
            assert scalar_err(stats1[0] - stats0[0], wloss) < 1e-4, (lab, stats1, stats0, wloss)
            assert stats1[1] - stats0[1] == wupd, (lab, stats1, stats0, wupd)
            mism = (gt != ot) | (gn != on)
            assert mism.mean() < 2e-3, (lab, mism.mean())
            diverged = diverged or bool(mism.any())
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
        assert mP.sum() + mQ.sum() + mB.sum() <= 5, (lab, "ill-conditioned elements", mP.sum(), mQ.sum(), mB.sum())
        b.g.update_parameters_device()
        h.update_parameters()
        o.update_parameters()
        Pa, Qa, Qba, Pb, Qb_, Qbb, gP2, gQ2 = b.host(a.P, a.Q, a.Qb, b.P, b.Q, b.Qb, b.gP, b.gQ)
        for name, F in (("P", Pa), ("Q", Qa), ("P", Pb), ("Q", Qb_), ("gP", gP2), ("gQ", gQ2), ("P host", Ph),
                        ("Q host", Qh)):
            assert not F[:, d:].any(), (lab, name, "padding columns must stay zero")
        if not diverged:
            errs = masked_err(Pb[:, :d], Po, mP), masked_err(Qb_[:, :d], Qo, mQ), masked_err(Qbb, Qbo, mB)
            assert max(errs) < ORACLE_TOL, (lab, "vs oracle", errs)
            for name, (Px, Qx, Qbx) in (("sharded", (Pa, Qa, Qba)), ("host", (Ph, Qh, Qbh))):
                errs = (masked_err(Px[:, :d], Pb[:, :d], mP), masked_err(Qx[:, :d], Qb_[:, :d], mQ),
                        masked_err(Qbx, Qbb, mB))
                # once an excused element differs, its neighbours in the next epochs differ too, within the oracle bar
                assert max(errs) < (ORACLE_TOL if mP.any() or mQ.any() or mB.any() else PATH_TOL), (lab, name, errs)
        for g, lr in ((a.g, lr_start), (b.g, o.lr), (h, o.lr)):
            assert abs(g.current_lr() - lr) < 1e-12 and g.epoch() == o.epoch == e + 1, (lab, g.current_lr(), lr)
        lg, lo_ = b.g.compute_loss(*probe), o.compute_loss(*probe)
        if warp:
            lm = np_mirror.warp_loss(Pb[:, :d], Qb_[:, :d], *probe, threshold=opt["threshold"], score=opt["score_func"])
            # a violation test within fp32 rounding of the margin may flip: at most two of the probe triples
            assert abs(lg - lm) <= 2.0 / len(probe[0]) + 1e-12, (lab, lg, lm)
            if not diverged:
                assert abs(lg - lo_) <= 2.0 / len(probe[0]) + 1e-12, (lab, lg, lo_)
        else:
            lm = np_mirror.bpr_loss(Pb[:, :d], Qb_[:, :d], Qbb, *probe, use_bias=opt["use_bias"])
            assert scalar_err(lg, lm) < 1e-5 and scalar_err(lg, lo_) < 1e-5, (lab, lg, lm, lo_)
    if warp:
        assert np.linalg.norm(Pb[:, :d], axis=1).max() <= 1.0 + 1e-5     # warp.cc:196-200
    return diverged


@pytest.mark.parametrize("kind,kw", [
    ("bpr", dict(d=128, optimizer="adagrad")),
    ("bpr", dict(d=128, optimizer="adam", per_coordinate_normalize=True)),
    ("bpr", dict(d=64, optimizer="adagrad", sampling_power=1.0)),
    ("warp", dict(d=64, optimizer="adagrad", score_func="dot")),
    ("warp", dict(d=64, optimizer="adam", score_func="l2", per_coordinate_normalize=True)),
], ids=["bpr-adagrad", "bpr-adam-pcn", "bpr-popularity", "warp-adagrad-dot", "warp-adam-l2"])
def test_device_resident_epochs(cuda_lib, kind, kw):
    opt = sgd_opt(num_iters=3, num_negative_samples=2 if kind == "bpr" else 1, max_trials=30, reg_u=0.01, reg_i=0.02,
                  reg_j=0.03, use_bias=(kind == "bpr"), **kw)
    run_epochs(kind, opt, U=600, I=500, mean=12, seed=kw["d"] + len(kw), cum_power=int(kw.get("sampling_power", 0)))


@pytest.mark.parametrize("kind", ["bpr", "warp"])
@pytest.mark.parametrize("d", WIDTHS)
def test_sgd_widths(cuda_lib, kind, d):
    # adam + per-coordinate counters at two widths, the l2 score at two, adagrad / dot elsewhere
    kw = dict(optimizer="adam", per_coordinate_normalize=True) if d in (129, 384) else dict(optimizer="adagrad")
    if kind == "warp" and d in (30, 257):
        kw["score_func"] = "l2"
    opt = sgd_opt(d=d, num_iters=3, num_negative_samples=2 if kind == "bpr" else 1, max_trials=30, reg_u=0.01,
                  reg_i=0.02, reg_j=0.03, use_bias=(kind == "bpr"), **kw)
    run_epochs(kind, opt, U=150, I=400, mean=10, seed=d)


@pytest.mark.parametrize("d", WIDTHS)
def test_bpr_sgd_triples_collision_free_widths(cuda_lib, d):
    """apply_triples_device (plain SGD, pre-update form) on triples that share no row: exact up to fp32 rounding
    against orc_bpr_update_preupdate (1e-5 relative, as at d = 128 in test_sgd_gpu.py) [9e-8]."""
    import oracle
    import torch
    from buffalo_b200 import backend
    U, I, n = 600, 1300, 500
    opt = sgd_opt(d=d, optimizer="sgd")
    P = init_factors(U, d, d, 1, scale=d ** -0.25, signed=True)
    Q = init_factors(I, d, d, 2, scale=d ** -0.25, signed=True)
    Qb = init_factors(I, 1, 1, 3, scale=0.1, signed=True)
    rng = np.random.default_rng(d)
    us = rng.permutation(U)[:n].astype(np.int32)
    items = rng.permutation(I)[:2 * n].astype(np.int32)
    ps, ns = items[:n].copy(), items[n:].copy()
    g = backend.CuSGD("bpr")
    assert g.init(opt)
    vdim = g.get_vdim()
    dev = torch.device("cuda:0")
    tP, tQ = torch.from_numpy(padded(P, vdim)).to(dev), torch.from_numpy(padded(Q, vdim)).to(dev)
    tQb = torch.from_numpy(Qb.copy()).to(dev)
    g.bind_factors(tP, tQ, tQb, n)
    g.apply_triples_device(*(torch.from_numpy(x).to(dev) for x in (us, ps, ns)), 0.05)
    torch.cuda.synchronize()
    o = oracle.sgd_opt_struct(opt)
    Po, Qo, Qbo = P.copy(), Q.copy(), Qb.copy()
    oracle.lib().orc_bpr_update_preupdate(C.byref(o), oracle._f32(Po), oracle._f32(Qo), oracle._f32(Qbo),
                                          oracle._i32(us), oracle._i32(ps), oracle._i32(ns), C.c_int64(n),
                                          C.c_float(0.05))
    Pg, Qg, Qbg = tP.cpu().numpy(), tQ.cpu().numpy(), tQb.cpu().numpy()
    assert not Pg[:, d:].any() and not Qg[:, d:].any(), "padding columns must stay zero"
    assert rel_err(Pg[:, :d], Po) < 1e-5 and rel_err(Qg[:, :d], Qo) < 1e-5 and rel_err(Qbg, Qbo) < 1e-5
    # every touched row moved, in every column (a kernel that skips a column group leaves it at its start value)
    assert (Pg[us, :d] != P[us]).mean() > 0.99 and (Qg[ps, :d] != Q[ps]).mean() > 0.99


def test_bpr_sgd_device_path_converges_like_oracle(cuda_lib):
    """Plain-SGD BPR through ShardedSGD(world=1) is Hogwild (lock-free concurrent updates, bpr.cc:157-171), so it is
    held to the band of test_sgd_gpu.py::test_bpr_sgd_converges_like_oracle instead of element-wise equality: the same
    lr schedule, monotone learning, and after 8 epochs the oracle's loss level within 25 %."""
    import oracle
    from tests.test_sgd_gpu import _planted
    U, I, indptr, keys, _ = _planted(U=20000, I=3000, seed=5)
    d, epochs = 32, 8
    rng = np.random.default_rng(6)
    beg = np.concatenate([[0], indptr[:-1]])
    probe_u = rng.choice(np.nonzero(indptr > beg)[0], 2000).astype(np.int32)
    probe_p = np.array([keys[rng.integers(beg[u], indptr[u])] for u in probe_u], np.int32)
    probe_n = rng.integers(0, I, 2000).astype(np.int32)
    opt = sgd_opt(d=d, optimizer="sgd", lr=0.1, random_seed=1, num_iters=epochs, reg_u=0.01, reg_i=0.01, reg_j=0.01,
                  reg_b=0.01)
    P, Q = init_factors(U, d, d, 1, scale=0.05), init_factors(I, d, d, 11, scale=0.05)
    Qb = np.zeros((I, 1), np.float32)
    run = DeviceRun("bpr", opt, P, Q, Qb, indptr, keys, None)
    assert run.drv.mode == "sgd"
    o = oracle.OracleSGD(warp=False, use_lut=True)
    o.init(opt)
    Po, Qo, Qbo = P.copy(), Q.copy(), Qb.copy()
    o.initialize_model(Po, Qo, Qbo, len(keys))
    hist = [(run.g.compute_loss(probe_u, probe_p, probe_n), o.compute_loss(probe_u, probe_p, probe_n))]
    for _ in range(epochs):
        run.drv.epoch()
        o.add_jobs(0, U, indptr, keys)
        o.update_parameters()
        hist.append((run.g.compute_loss(probe_u, probe_p, probe_n), o.compute_loss(probe_u, probe_p, probe_n)))
        assert abs(run.g.current_lr() - o.lr) < 1e-12
    lgs = [x[0] for x in hist]
    assert all(y <= x * 1.02 for x, y in zip(lgs, lgs[1:])), hist
    assert lgs[-1] < 0.5 * lgs[0] and hist[-1][1] < 0.5 * hist[0][1], hist
    assert abs(hist[-1][0] - hist[-1][1]) < 0.25 * hist[-1][1], hist
    Pg, = run.host(run.P)
    assert np.isfinite(Pg).all()


@pytest.mark.parametrize("cls_name,d", [("BPRMF", 10), ("BPRMF", 130), ("WARP", 10), ("WARP", 130)])
def test_sgd_public_api_widths(cuda_lib, tmp_path, cls_name, d):
    """buffalo.BPRMF / buffalo.WARP end to end at widths that are not multiples of 4: the model is trained vdim-padded,
    handed back at width d, and a model set at width d is re-padded by the next train() (sgd_common.py _prepare_train).
    Both trainings start from the same factors (the epoch counter and the draws restart with initialize_model) and must
    match the C oracle's epochs on the same CSR (adagrad: chunking does not change the step; 1e-4 relative).  The start
    is of order d^-1/4 rather than the 1/d^2 of init_factors, whose first Adagrad step (g / |g|) the fp32 restatements
    cannot decide in the elements where g cancels."""
    import scipy.sparse
    import buffalo
    import oracle
    from buffalo.data import MatrixMarketOptions
    rng = np.random.default_rng(d)
    U, I = 300, 250
    indptr, keys, _ = csr_from_lengths(rng.integers(0, 25, U), I, rng)
    m = scipy.sparse.csr_matrix((np.ones(len(keys), np.float32), keys, np.concatenate([[0], indptr])), shape=(U, I))
    dopt = MatrixMarketOptions().get_default_option()
    dopt.input.main = m
    dopt.data.path = str(tmp_path / "mm.h5py")
    dopt.data.validation.p = 0.0
    opt = getattr(buffalo, cls_name + "Option")().get_default_option()
    opt.update(d=d, num_iters=2, random_seed=3, optimizer="adagrad", lr=0.05)
    algo = getattr(buffalo, cls_name)(opt, data_opt=dopt)
    algo.initialize()
    vdim = algo.obj.get_vdim()
    assert algo.P.shape == (U, vdim) and vdim == (d + 3) // 4 * 4
    P0 = init_factors(U, d, d, 1, scale=d ** -0.25, signed=True)
    Q0 = init_factors(I, d, d, 2, scale=d ** -0.25, signed=True)
    Qb0 = init_factors(I, 1, 1, 3, scale=0.3, signed=True) if cls_name == "BPRMF" else np.zeros((I, 1), np.float32)
    grp = algo.data.get_group("rowwise")
    g_ind, g_keys = np.asarray(grp["indptr"][:], np.int64), np.ascontiguousarray(grp["key"][:], np.int32)
    warp = cls_name == "WARP"
    o = oracle.OracleSGD(warp=warp, use_lut=False)
    o.init(dict(algo.opt))
    Po, Qo, Qbo = P0.copy(), Q0.copy(), Qb0.copy()
    o.initialize_model(Po, Qo, Qbo, len(g_keys))
    mP, mQ, mB = np.zeros(Po.shape, bool), np.zeros(Qo.shape, bool), np.zeros(Qbo.shape, bool)
    for _ in range(2):
        o.add_jobs(0, U, g_ind, g_keys)
        mP |= ill_conditioned(o.gP, o.cP, Po, o.o.reg_u, False)
        mQ |= ill_conditioned(o.gQ, o.cQ, Qo, o.o.reg_i, False)
        if not warp:
            mB |= ill_conditioned(o.gQb, o.cQ, Qbo, o.o.reg_b, False)
        o.update_parameters()
    assert mP.sum() + mQ.sum() + mB.sum() <= 5, (mP.sum(), mQ.sum(), mB.sum())
    for rnd in range(2):
        if rnd == 0:    # the layout initialize() leaves
            algo.P, algo.Q, algo.Qb = padded(P0, vdim), padded(Q0, vdim), Qb0.copy()
        else:           # factors set by the user at width d
            algo.P, algo.Q, algo.Qb = P0.copy(), Q0.copy(), Qb0.copy()
        algo.train()
        assert algo.P.shape == (U, d) and algo.Q.shape == (I, d), (rnd, algo.P.shape)
        assert np.isfinite(algo.P).all() and np.isfinite(algo.Q).all()
        if warp:
            # rank sampling flips where a score sits within fp32 rounding of the margin: allow a few rows
            bad = (np.abs(algo.P - Po) > 1e-4 * np.abs(Po).max()) & ~mP
            assert bad.any(axis=1).mean() < 0.02, (rnd, bad.sum())
            assert np.linalg.norm(algo.P, axis=1).max() <= 1.0 + 1e-5
        else:
            errs = masked_err(algo.P, Po, mP), masked_err(algo.Q, Qo, mQ), masked_err(algo.Qb, Qbo, mB)
            assert max(errs) < 1e-4, (rnd, errs)


def test_bind_factors_rejects_wrong_width_and_bias(cuda_lib):
    """The kernels stride rows by vdim: bind_factors refuses anything else before a kernel can run."""
    import torch
    from buffalo_b200 import backend
    g = backend.CuSGD("bpr")
    assert g.init(sgd_opt(d=30, optimizer="adagrad"))
    assert g.get_vdim() == 32
    dev = torch.device("cuda:0")
    P, Q, Qb = torch.zeros(10, 32, device=dev), torch.zeros(20, 32, device=dev), torch.zeros(20, 1, device=dev)
    for bad in (dict(P=torch.zeros(10, 30, device=dev)), dict(Q=torch.zeros(20, 30, device=dev)),
                dict(Q=torch.zeros(20 * 32, device=dev)), dict(Qb=torch.zeros(19, 1, device=dev)),
                dict(Qb=torch.zeros(21, device=dev))):
        args = dict(dict(P=P, Q=Q, Qb=Qb), **bad)
        with pytest.raises(ValueError):
            g.bind_factors(args["P"], args["Q"], args["Qb"], 100)
    g.bind_factors(P, Q, Qb, 100)
    g.bind_factors(P, Q, torch.zeros(20, device=dev), 100)     # a flat bias of Q.shape[0] floats is fine

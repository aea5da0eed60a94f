"""ALS parity on the GPU: the CUDA path, driven through the C ABI exactly as the reference's Python
driver drives `self.obj` (buffalo/algo/als.py:115-142), against the CPU oracle on the same seeded
inputs and against the committed golden fixtures.

Tolerance: factors within 1e-3 relative max-norm (BASELINE.json north_star), stated per test; both
sides compute in fp32 with different summation orders.  Loss pieces within 1e-4 relative.
"""
import json
import os

import numpy as np
import pytest

from tests.helpers import (FACTOR_TOL, check_loss, check_rows, csr_from_lengths, full_opt, gpu_half, init_factors,
                           make_csr, oracle_half, rel_err, transpose_csr)

pytestmark = pytest.mark.gpu
GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


@pytest.mark.parametrize("case", json.load(open(os.path.join(GOLDEN, "golden_als.json")))["cases"],
                         ids=lambda c: c["file"][:-4])
def test_golden_fixture(cuda_lib, case):
    z = np.load(os.path.join(GOLDEN, case["file"]))
    X, n, dn = gpu_half(case["opt"], z["P"], z["Q"], z["indptr"], z["keys"], z["vals"], case["axis"])
    assert rel_err(X, z["X"]) < FACTOR_TOL
    check_loss(n, dn, float(z["nume"]), float(z["deno"]))


@pytest.mark.parametrize("d,optimizer,kw", [
    (32, "manual_cg", {}),                       # BASELINE configs[0] shape family (d=32, default optimizer)
    (32, "manual_cg", {"adaptive_reg": True, "num_cg_max_iters": 5}),
    (10, "manual_cg", {}), (40, "manual_cg", {}), (80, "manual_cg", {}),   # benchmark D sweep (test_performance.py:9)
    (5, "llt", {}), (20, "ldlt", {}), (64, "llt", {"adaptive_reg": True}), (96, "ldlt", {}),
    (100, "ialspp", {"block_size": 7}), (64, "ialspp", {"block_size": 16}), (48, "ialspp", {"block_size": 64}),
    (128, "manual_cg", {}), (160, "manual_cg", {}), (256, "manual_cg", {}), (128, "llt", {"block_size": 64}),
])
def test_parity_vs_oracle(cuda_lib, d, optimizer, kw):
    U, I, nnz = 3000, 2000, 90000
    indptr, keys, vals, _ = make_csr(U, I, nnz, seed=d * 7 + len(optimizer), empty_rows=20)
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
    opt = full_opt(d=d, optimizer=optimizer, **kw)
    # a state as met after a few ALS iterations: signed factors of moderate size
    P = init_factors(U, d, d, 1, scale=0.1, signed=True)
    Q = init_factors(I, d, d, 2, scale=0.1, signed=True)
    X, n, dn = gpu_half(opt, P, Q, indptr, keys, vals, 0)
    X0, n0, dn0 = oracle_half(opt, P, Q, indptr, keys, vals, 0)
    assert rel_err(X, X0) < FACTOR_TOL
    check_loss(n, dn, n0, dn0)
    X, n, dn = gpu_half(opt, P, Q, cind, ckeys, cvals, 1)
    X0, n0, dn0 = oracle_half(opt, P, Q, cind, ckeys, cvals, 1)
    assert rel_err(X, X0) < FACTOR_TOL
    check_loss(n, dn, n0, dn0)


def test_c1_config_training_trajectory(cuda_lib):
    """BASELINE configs[0]: ALS d=32 on 10k x 5k, 200k nnz, default options, from the reference's own
    initialisation abs(N(0, 1/d^2)) (als.py:85-86), three full iterations.
    (1) every half-epoch started from the oracle's state matches the oracle to 1e-3 (the parity bar);
    (2) the GPU's own trajectory (never re-synchronised) stays within 5e-3 of the oracle's and reports the
        same RMSE (als.py:171) -- 3-step CG does not contract rounding differences, so they add up."""
    U, I, nnz, d = 10000, 5000, 200000, 32
    indptr, keys, vals, _ = make_csr(U, I, nnz, seed=1234)
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
    opt = full_opt(d=d)
    Pg = init_factors(U, d, d, 7)
    Qg = init_factors(I, d, d, 8)
    Po, Qo = Pg.copy(), Qg.copy()
    for it in range(3):
        Ps, _, _ = gpu_half(opt, Po, Qo, indptr, keys, vals, 0)         # (1) from the oracle's state
        Pg, n1, d1 = gpu_half(opt, Pg, Qg, indptr, keys, vals, 0)       # (2) own trajectory
        Po, m1, e1 = oracle_half(opt, Po, Qo, indptr, keys, vals, 0)
        assert rel_err(Ps, Po) < FACTOR_TOL, it
        Qs, _, _ = gpu_half(opt, Po, Qo, cind, ckeys, cvals, 1)
        Qg, n2, d2 = gpu_half(opt, Pg, Qg, cind, ckeys, cvals, 1)
        Qo, m2, e2 = oracle_half(opt, Po, Qo, cind, ckeys, cvals, 1)
        assert rel_err(Qs, Qo) < FACTOR_TOL, it
        assert rel_err(Pg, Po) < 5e-3 and rel_err(Qg, Qo) < 5e-3, it
        rmse_g = ((n1 + n2) / (d1 + d2 + 1e-10)) ** 0.5     # als.py:171
        rmse_o = ((m1 + m2) / (e1 + e2 + 1e-10)) ** 0.5
        assert abs(rmse_g - rmse_o) < 1e-4 * rmse_o


@pytest.mark.parametrize("d", [128, 64, 32, 96, 160, 192, 224, 256])
def test_tuned_kernel_all_row_length_classes(cuda_lib, d):
    """Rows are binned by length (<=32, 64, 128, 256, 512, 1536, 12288, longer).  Default (_b200_kernel_mode=0):
    at d=128 the rows of 65..1536 nnz go through the fused tensor-core kernel (als_tc.cuh), the longer ones through its
    split-row mode (2048-entry chunks + explicit solve); at d=256 the rows beyond 1536 nnz take the split-row mode;
    everything else runs on the tuned SIMT kernels (d = 160..256 read the Gram matrix through L1/L2).
    _b200_kernel_mode=2 = SIMT kernels only (rows beyond 12288 on the generic kernel), 1 = generic kernels.
    One input that hits every class, checked row by row against the oracle and against the generic kernel."""
    rng = np.random.default_rng(d)
    lengths = np.concatenate([rng.integers(1, 33, 300), rng.integers(33, 65, 200), rng.integers(65, 129, 150),
                              rng.integers(129, 257, 80), rng.integers(257, 513, 40), rng.integers(513, 1025, 20),
                              rng.integers(1025, 1537, 12), rng.integers(1537, 12289, 5),
                              [12289, 13000, 1536, 1537, 1024, 1025, 512, 513, 32, 33, 0, 0, 1]])
    rng.shuffle(lengths)
    U, I = len(lengths), 14000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    opt = full_opt(d=d, optimizer="ialspp", block_size=32)
    P = init_factors(U, d, d, 1, scale=0.05, signed=True)
    Q = init_factors(I, d, d, 2, scale=0.05, signed=True)
    for axis_opt in (dict(), dict(adaptive_reg=True)):
        o = dict(opt, **axis_opt)
        X0, n0, dn0 = oracle_half(o, P, Q, indptr, keys, vals, 0)
        Xf, nf, dnf = gpu_half(o, P, Q, indptr, keys, vals, 0)
        Xg, ng, dng = gpu_half(dict(o, _b200_kernel_mode=1), P, Q, indptr, keys, vals, 0)
        Xs, ns, dns = gpu_half(dict(o, _b200_kernel_mode=2), P, Q, indptr, keys, vals, 0)   # SIMT kernels only
        assert rel_err(Xf, X0) < FACTOR_TOL and rel_err(Xg, X0) < FACTOR_TOL and rel_err(Xs, X0) < FACTOR_TOL
        assert rel_err(Xf, Xg) < FACTOR_TOL
        # no single row is off either (the Frobenius norm would hide one bad row-length class)
        row_err = check_rows({"default": Xf, "simt": Xs}, X0, P, Q, indptr, keys, vals, o, 0, label="d=%d" % d)
        assert row_err["default"].max() < 5e-3, (int(row_err["default"].argmax()), float(row_err["default"].max()))
        check_loss(nf, dnf, n0, dn0)
        check_loss(ns, dns, n0, dn0)
        Xr, nr, dnr = gpu_half(dict(o, _b200_kernel_mode=4), P, Q, indptr, keys, vals, 0)   # 513..1536 re-gathered
        assert rel_err(Xr, X0) < FACTOR_TOL
        check_loss(nr, dnr, n0, dn0)
    # negative confidence values are legal input for every kernel variant
    vneg = vals.copy()
    vneg[::7] *= -0.25
    X0, n0, dn0 = oracle_half(opt, P, Q, indptr, keys, vneg, 0)
    for mode in (0, 2):
        Xf, nf, dnf = gpu_half(dict(opt, _b200_kernel_mode=mode), P, Q, indptr, keys, vneg, 0)
        assert np.isfinite(Xf).all() and rel_err(Xf, X0) < FACTOR_TOL, mode
    # item side (loss has the extra x G x and observed terms): reuse the same CSR as a colwise matrix
    Pi = init_factors(I, d, d, 3, scale=0.05, signed=True)      # "users" are now the opposite side
    Qi = init_factors(U, d, d, 4, scale=0.05, signed=True)      # rows being updated (axis 1)
    X0, n0, dn0 = oracle_half(opt, Pi, Qi, indptr, keys, vals, 1)
    Xf, nf, dnf = gpu_half(opt, Pi, Qi, indptr, keys, vals, 1)
    assert rel_err(Xf, X0) < FACTOR_TOL
    check_loss(nf, dnf, n0, dn0)


@pytest.mark.parametrize("d", [128, 256])
def test_long_rows_split_tensor_core_path(cuda_lib, d):
    """Rows far beyond the SIMT kernels' cap (2e4, 2e5 and 1e6 nnz; Zipf head items of BASELINE configs[4]) are cut into
    2048-entry chunks over the SMs, their explicit matrices summed by the tensor-core (wgmma) kernel and solved by
    als_explicit_solve_kernel.  Bar (check_rows): 1e-3 against the fp32 oracle per row; where the oracle's own
    sequential fp32 sums over 1e6 terms drift further than that from the fp64 mirror, the GPU must be at least as close
    to the mirror."""
    rng = np.random.default_rng(d + 1)
    lengths = np.array([20000, 200000, 1000000, 700, 12289, 40, 16385, 8193], dtype=np.int64)
    U, I = len(lengths), 1_200_000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    opt = full_opt(d=d, optimizer="ialspp", block_size=32)
    P = init_factors(U, d, d, 1, scale=0.05, signed=True)
    Q = init_factors(I, d, d, 2, scale=0.05, signed=True)
    for axis in (0, 1):
        # axis 1 exercises the loss pieces (x G x, observed terms) of the split path: same CSR read as a colwise matrix
        Pa, Qa = (P, Q) if axis == 0 else (Q, P)
        X0, n0, dn0 = oracle_half(opt, Pa, Qa, indptr, keys, vals, axis)
        Xf, nf, dnf = gpu_half(opt, Pa, Qa, indptr, keys, vals, axis)
        Xup, Yop = (Pa, Qa) if axis == 0 else (Qa, Pa)
        check_rows({"default": Xf}, X0, Xup, Yop, indptr, keys, vals, opt, axis, label="axis %d" % axis)
        assert abs(nf - n0) <= 2e-4 * max(1.0, abs(n0)), (nf, n0)
        assert abs(dnf - dn0) <= 1e-4 * max(1.0, abs(dn0)), (dnf, dn0)


def test_d128_reference_init_three_iterations(cuda_lib):
    """The benched state: d=128 from the reference's own abs(N(0, 1/d^2)) initialisation (als.py:85-86), three full
    iterations.  There the Gram matrix is numerically rank-one and the fp32 oracle itself sits 1e-2..1e-1 away from
    the fp64 mirror on the first passes (DESIGN.md 2), so the bar is: per half-epoch, started from the oracle's state,
    the GPU is no further from the oracle than the oracle is from the fp64 mirror (or within 1e-3), and the RMSE of the
    GPU's own trajectory matches the oracle's."""
    from oracle import np_mirror
    U, I, nnz, d = 1500, 900, 60000, 128
    indptr, keys, vals, _ = make_csr(U, I, nnz, seed=4321)
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
    opt = full_opt(d=d)
    Pg = init_factors(U, d, d, 7)
    Qg = init_factors(I, d, d, 8)
    Po, Qo = Pg.copy(), Qg.copy()
    for it in range(3):
        Ps, _, _ = gpu_half(opt, Po, Qo, indptr, keys, vals, 0)
        Pm, _, _ = np_mirror.als_half_epoch(Po, Qo, indptr, keys, vals, opt, 0)
        Pg, n1, d1 = gpu_half(opt, Pg, Qg, indptr, keys, vals, 0)
        Po, m1, e1 = oracle_half(opt, Po, Qo, indptr, keys, vals, 0)
        assert rel_err(Ps, Po) <= max(FACTOR_TOL, 1.5 * rel_err(Po, Pm)), (it, rel_err(Ps, Po), rel_err(Po, Pm))
        Qs, _, _ = gpu_half(opt, Po, Qo, cind, ckeys, cvals, 1)
        Qm, _, _ = np_mirror.als_half_epoch(Qo, Po, cind, ckeys, cvals, opt, 1)
        Qg, n2, d2 = gpu_half(opt, Pg, Qg, cind, ckeys, cvals, 1)
        Qo, m2, e2 = oracle_half(opt, Po, Qo, cind, ckeys, cvals, 1)
        assert rel_err(Qs, Qo) <= max(FACTOR_TOL, 1.5 * rel_err(Qo, Qm)), (it, rel_err(Qs, Qo), rel_err(Qo, Qm))
        rmse_g = ((n1 + n2) / (d1 + d2 + 1e-10)) ** 0.5     # als.py:171
        rmse_o = ((m1 + m2) / (e1 + e2 + 1e-10)) ** 0.5
        assert abs(rmse_g - rmse_o) <= 2e-3 * rmse_o, (it, rmse_g, rmse_o)


def test_chunked_equals_whole_and_placeholder(cuda_lib):
    # BufferedDataMatrix feeds row-aligned chunks (buffered_data.py:85-118); results must not depend on chunking.
    # ~160 entries per item, so that the item rows (axis 1) run on the fused tensor-core kernel
    U, I, nnz, d = 2000, 1500, 240000, 128
    indptr, keys, vals, _ = make_csr(U, I, nnz, seed=99, empty_rows=30)
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
    opt = full_opt(d=d)
    P = init_factors(U, d, d, 1, scale=0.1, signed=True)
    Q = init_factors(I, d, d, 2, scale=0.1, signed=True)
    X1, n1, d1 = gpu_half(opt, P, Q, cind, ckeys, cvals, 1, chunks=1)
    X5, n5, d5 = gpu_half(opt, P, Q, cind, ckeys, cvals, 1, chunks=5, placeholder=(indptr, cind))
    assert rel_err(X5, X1) < 1e-5
    check_loss(n5, d5, n1, d1)


def test_empty_rows_untouched_and_empty_chunk(cuda_lib):
    U, I, d = 500, 300, 16
    indptr, keys, vals, rows = make_csr(U, I, 4000, seed=3, empty_rows=60)
    P = init_factors(U, d, d, 1, scale=0.1)
    Q = init_factors(I, d, d, 2, scale=0.1)
    empty = np.setdiff1d(np.arange(U), rows)
    for optimizer in ("llt", "manual_cg", "ialspp"):
        X, _, _ = gpu_half(full_opt(d=d, optimizer=optimizer), P, Q, indptr, keys, vals, 0)
        assert np.array_equal(X[empty], P[empty])      # als.cc:159-162
    from buffalo_b200 import backend
    obj = backend.CuALS()
    obj.init(full_opt(d=d))
    Pp, Qp = P.copy(), Q.copy()
    obj.initialize_model(Pp, Qp)
    obj.precompute(0)
    assert obj.partial_update(7, 7, indptr, keys, vals, 0) == (0.0, 0.0)   # als.cc:115-118


def test_device_path_equals_host_path(cuda_lib):
    import torch
    from buffalo_b200 import backend
    U, I, nnz, d = 4000, 2500, 150000, 128
    indptr, keys, vals, _ = make_csr(U, I, nnz, seed=5, empty_rows=11)
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
    opt = full_opt(d=d)
    P = init_factors(U, d, d, 1, scale=0.1, signed=True)
    Q = init_factors(I, d, d, 2, scale=0.1, signed=True)
    Xh, nh, dh = gpu_half(opt, P, Q, indptr, keys, vals, 0)
    Yh, mh, eh = gpu_half(opt, Xh, Q, cind, ckeys, cvals, 1)
    obj = backend.CuALS()
    obj.init(opt)
    dev = torch.device("cuda:0")
    tP, tQ = torch.from_numpy(P).to(dev), torch.from_numpy(Q).to(dev)
    obj.bind_factors(tP, tQ)
    obj.bind_csr(0, torch.from_numpy(indptr).to(dev), torch.from_numpy(keys).to(dev), torch.from_numpy(vals).to(dev))
    obj.bind_csr(1, torch.from_numpy(cind).to(dev), torch.from_numpy(ckeys).to(dev), torch.from_numpy(cvals).to(dev))
    loss = torch.zeros(2, dtype=torch.float64, device=dev)
    obj.precompute_device(0)
    obj.update_device(0, 0, U, loss)
    l0 = loss.cpu().numpy().copy()
    loss.zero_()
    obj.precompute_device(1)
    obj.update_device(1, 0, I // 2, loss)       # two row ranges = one pass
    obj.update_device(1, I // 2, I, loss)
    torch.cuda.synchronize()
    assert rel_err(tP.cpu().numpy(), Xh) < 1e-5
    assert rel_err(tQ.cpu().numpy(), Yh) < 1e-5
    check_loss(l0[0], l0[1], nh, dh)
    l1 = loss.cpu().numpy()
    check_loss(l1[0], l1[1], mh, eh)


def test_gram_precompute(cuda_lib):
    import torch
    from buffalo_b200 import backend
    for d, rows in [(32, 5000), (100, 3333), (128, 20000), (256, 1000)]:
        obj = backend.CuALS()
        obj.init(full_opt(d=d))
        rng = np.random.default_rng(d)
        Q = rng.normal(size=(rows, obj.get_vdim())).astype(np.float32)
        Q[:, d:] = 0
        tP = torch.zeros(8, obj.get_vdim(), device="cuda")
        tQ = torch.from_numpy(Q).cuda()
        obj.bind_factors(tP, tQ)
        obj.precompute_device(0)
        torch.cuda.synchronize()
        G = obj.gram_tensor().cpu().numpy()
        G0 = Q[:, :d].astype(np.float64).T @ Q[:, :d].astype(np.float64)
        assert rel_err(G, G0) < 1e-5


def test_unsupported_optimizer_and_state_errors(cuda_lib):
    from buffalo_b200 import _cabi, backend
    obj = backend.CuALS()
    assert obj.init(full_opt(optimizer="eigen_cg")) is False        # rejected like an invalid option file
    assert "eigen_cg" in obj.last_error
    obj = backend.CuALS()
    with pytest.raises(_cabi.BackendError):
        obj.precompute(0)                                            # before init/initialize_model


def test_mid_size_sampled_rows_property(cuda_lib):
    """Size-independent check at a size the oracle cannot sweep in seconds: solve 1M x 200k, 40M nnz on the
    device, then re-solve a random sample of rows with the oracle (full opposite factors, sampled CSR rows)."""
    import torch
    from buffalo_b200 import backend
    import oracle
    dev = torch.device("cuda:0")
    U, I, nnz, d = 1_000_000, 200_000, 40_000_000, 128
    g = torch.Generator(device=dev)
    g.manual_seed(2024)
    rows = torch.randint(0, U, (nnz,), device=dev, generator=g, dtype=torch.int64)
    cols = torch.randint(0, I, (nnz,), device=dev, generator=g, dtype=torch.int64)
    key = torch.sort(rows * I + cols).values
    rows, cols = key // I, (key % I).to(torch.int32)
    indptr = torch.cumsum(torch.bincount(rows, minlength=U), 0)
    vals = torch.ones(nnz, device=dev, dtype=torch.float32)
    P = (torch.randn(U, d, device=dev, generator=g) * 0.05).contiguous()
    Q = (torch.randn(I, d, device=dev, generator=g) * 0.05).contiguous()
    P0 = P.clone()
    opt = full_opt(d=d, compute_loss_on_training=False)
    obj = backend.CuALS()
    obj.init(opt)
    obj.bind_factors(P, Q)
    obj.bind_csr(0, indptr, cols, vals)
    obj.precompute_device(0)
    obj.update_device(0, 0, U)
    torch.cuda.synchronize()
    assert torch.isfinite(P).all()
    sample = torch.randint(0, U, (300,), generator=torch.Generator().manual_seed(1)).numpy()
    hind = indptr.cpu().numpy()
    beg = np.concatenate([[0], hind[:-1]])
    sub_keys = np.concatenate([cols[beg[u]:hind[u]].cpu().numpy() for u in sample]).astype(np.int32)
    sub_ind = np.cumsum([hind[u] - beg[u] for u in sample]).astype(np.int64)
    subP = P0[torch.from_numpy(sample)].cpu().numpy().copy()
    Qh = Q.cpu().numpy()
    o = oracle.OracleALS()
    o.init(opt)
    o.initialize_model(subP, Qh)
    o.precompute(0)
    o.partial_update(0, len(sample), sub_ind, sub_keys, np.ones(len(sub_keys), np.float32), 0)
    got = P[torch.from_numpy(sample)].cpu().numpy()
    assert rel_err(got, subP) < FACTOR_TOL

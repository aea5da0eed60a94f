"""Kernel widths above d = 128: the generic iALS++ row solve at NC = 8 and 16 (d in (128, 512] off the tuned path),
Gram slab grids of 2x2 .. 4x4, the sharded Gram of ShardedALS emulated on one GPU, and the top-k scoring loop past one
16-byte pass per lane and at the 4096-item slice edges, each against a float64 reference of the same operation.

Tolerances (worst errors measured on an H100, 700 W, in brackets):
* ALS factors: FACTOR_TOL = 1e-3 relative max-norm against the fp32 oracle, and row by row through check_rows, which
  re-solves a row with the fp64 mirror where the oracle's own fp32 sums are not decisive [2e-6]; loss pieces 1e-4
  relative [2e-8];
* Gram matrices: 1e-5 relative max-norm against fp64 F^T F [3e-7];
* sharded Gram: the sum of the range partials 1e-5 against fp64 [1e-7]; the factors solved from it 1e-4 against the
  unsharded solve, the bound of the multi-GPU test (different fp32 summation order of G) [2e-6];
* top-k: the criteria of test_topk_gpu.py (scores of the picked items within 1e-4 of the fp64 k best, non-increasing,
  > 99 % of the indices equal, no duplicates); exact ties in index order."""
import numpy as np
import pytest

from tests.helpers import (FACTOR_TOL, check_loss, check_rows, csr_from_lengths, full_opt, gpu_half, init_factors,
                           make_csr, oracle_half, rel_err, transpose_csr)
from tests.test_topk_gpu import ref_topk

pytestmark = pytest.mark.gpu


def edge_csr(d, num_rows, num_cols, seed):
    """Rows of every kind the row solve meets: empty, one entry, short, and longer than d."""
    rng = np.random.default_rng(seed)
    lengths = np.concatenate([np.zeros(15, np.int64), np.ones(25, np.int64), rng.integers(2, 64, num_rows - 60),
                              rng.integers(d + 1, d + 200, 20)])
    rng.shuffle(lengths)
    return csr_from_lengths(lengths, num_cols, rng)


@pytest.mark.parametrize("d,kw", [
    (130, {}), (200, {}), (200, {"adaptive_reg": True}), (288, {}), (384, {}), (512, {}),
    (256, {"block_size": 64}),          # d = 256 off the tuned path: generic kernel, NC = 8
], ids=["d130", "d200", "d200-adaptive", "d288", "d384", "d512", "d256-bs64"])
def test_als_generic_wide_parity(cuda_lib, d, kw):
    """Both axes of one ALS iteration on the host-pointer path against the C oracle (test_parity_vs_oracle pattern).
    d >= 128 forces iALS++; none of these shapes is on the tuned path (d % 32, d > 256 or block_size != 32), so every
    row runs als_ialspp_warp_kernel<8> (d <= 256) or <16>."""
    U, I = 700, 900
    indptr, keys, vals = edge_csr(d, U, I, seed=d + len(kw))
    opt = full_opt(d=d, optimizer="ialspp", **kw)
    P = init_factors(U, d, d, 1, scale=0.1, signed=True)
    Q = init_factors(I, d, d, 2, scale=0.1, signed=True)
    for axis in (0, 1):
        # axis 1 (loss with the x G x and observed terms) reads the same CSR as a colwise matrix
        Pa, Qa = (P, Q) if axis == 0 else (Q, P)
        X, n, dn = gpu_half(opt, Pa, Qa, indptr, keys, vals, axis)
        X0, n0, dn0 = oracle_half(opt, Pa, Qa, indptr, keys, vals, axis)
        Xup, Yop = (Pa, Qa) if axis == 0 else (Qa, Pa)
        assert rel_err(X, X0) < FACTOR_TOL, (d, axis, rel_err(X, X0))
        check_rows({"gpu": X}, X0, Xup, Yop, indptr, keys, vals, opt, axis, label="d=%d axis %d" % (d, axis))
        check_loss(n, dn, n0, dn0)
        empty = np.flatnonzero(indptr == np.concatenate([[0], indptr[:-1]]))
        assert np.array_equal(X[empty], Xup[empty, :d]), (d, axis, "empty rows must stay untouched")


@pytest.mark.parametrize("d", [129, 200, 257, 384, 512])
def test_gram_wide(cuda_lib, d):
    """Gram matrix on slab grids of 2x2, 3x3 and 4x4, from one row (one partial tile) to enough rows that every CTA
    accumulates several tiles and several CTAs write partials."""
    import torch
    from buffalo_b200 import backend
    obj = backend.CuALS()
    assert obj.init(full_opt(d=d))
    vdim = obj.get_vdim()
    rng = np.random.default_rng(d)
    for rows in (1, 31, 33, 5000):
        Q = np.zeros((rows, vdim), np.float32)
        Q[:, :d] = rng.normal(size=(rows, d))
        tP, tQ = torch.zeros(8, vdim, device="cuda"), torch.from_numpy(Q).cuda()
        obj.bind_factors(tP, tQ)
        obj.precompute_device(0)
        torch.cuda.synchronize()
        G = obj.gram_tensor().cpu().numpy()
        G0 = Q[:, :d].astype(np.float64).T @ Q[:, :d].astype(np.float64)
        assert rel_err(G, G0) < 1e-5, (d, rows, rel_err(G, G0))


@pytest.mark.parametrize("d", [32, 128, 256, 384])
def test_sharded_gram_equals_unsharded(cuda_lib, d):
    """ShardedALS on one GPU: the Gram partials of three ranges of the opposite factor (empty, 45 rows, the rest) are
    summed the way the all-reduce sums them, written back through gram_tensor(), and every range of the updated factor
    is solved with update_device.  At d = 128 the tensor-core kernel takes its operand scale from the whole replica."""
    import torch
    from buffalo_b200 import backend
    U, I = 2000, 1500
    indptr, keys, vals, _ = make_csr(U, I, 100000, seed=d, empty_rows=13)
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
    opt = full_opt(d=d)
    P = init_factors(U, d, d, 1, scale=0.1, signed=True)
    Q = init_factors(I, d, d, 2, scale=0.1, signed=True)
    dev = torch.device("cuda:0")
    t = lambda a: torch.from_numpy(a).to(dev)  # noqa: E731
    runs = []
    for sharded in (False, True):
        obj = backend.CuALS()
        assert obj.init(opt)
        tP, tQ = t(P.copy()), t(Q.copy())
        obj.bind_factors(tP, tQ)
        obj.bind_csr(0, t(indptr), t(keys), t(vals))
        obj.bind_csr(1, t(cind), t(ckeys), t(cvals))
        for axis in (0, 1):
            rows, opp = (U, I) if axis == 0 else (I, U)
            if not sharded:
                obj.precompute_device(axis)
                obj.update_device(axis, 0, rows)
                continue
            Y = (tQ if axis == 0 else tP).cpu().numpy().astype(np.float64)
            G = torch.zeros(d, d, dtype=torch.float32, device=dev)
            for lo, hi in ((0, 0), (0, 45), (45, opp)):
                obj.precompute_rows_device(axis, lo, hi)
                part = obj.gram_tensor().clone()
                if hi == lo:
                    assert not part.any(), (d, axis, "an empty range contributes a zero partial")
                G += part
            G0 = Y.T @ Y
            assert rel_err(G.cpu().numpy(), G0) < 1e-5, (d, axis, rel_err(G.cpu().numpy(), G0))
            obj.gram_tensor().copy_(G)
            for lo, hi in ((0, 0), (0, 45), (45, rows)):
                obj.update_device(axis, lo, hi)
        torch.cuda.synchronize()
        runs.append((tP.cpu().numpy(), tQ.cpu().numpy()))
    (P1, Q1), (P2, Q2) = runs
    assert rel_err(P2, P1) < 1e-4 and rel_err(Q2, Q1) < 1e-4, (d, rel_err(P2, P1), rel_err(Q2, Q1))
    assert rel_err(P1, P) > 1e-2, "the solve must have moved the factors"


def _k_values(n_items):
    last = (n_items - 1) % 4096 + 1          # items in the last 4096-item slice
    return sorted({1, min(last + 1, n_items, 4096), min(n_items, 4096), 4096})


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("n_items", [4095, 4096, 4097, 8193])
@pytest.mark.parametrize("d", [129, 256, 512])
def test_topk_wide_and_slice_edges(cuda_lib, d, n_items, bias):
    """d = 256 and 512 take two and four 16-byte passes per lane of the scoring loop, d = 129 the scalar loop; item
    counts on both sides of the 4096-item slice; k = 1, k just above the last slice's size, k = I and k = 4096; seven
    queries (a partial group of four)."""
    from buffalo_b200 import backend
    nq = 7
    rng = np.random.default_rng(d * 10 + n_items + bias)
    P = rng.normal(size=(nq, d)).astype(np.float32)
    Q = rng.normal(size=(n_items, d)).astype(np.float32)
    Qb = rng.normal(size=(n_items, 1)).astype(np.float32) if bias else None
    s = P.astype(np.float64) @ Q.astype(np.float64).T + (0 if Qb is None else Qb.reshape(1, -1))
    for k in _k_values(n_items):
        got = backend.topk_host(P, Q, Qb, k)
        kk = min(k, n_items)
        assert got.shape == (nq, kk), (d, n_items, k)
        ridx, rval = ref_topk(P, Q, Qb, kk)
        gval = np.take_along_axis(s, got.astype(np.int64), axis=1)
        assert np.allclose(gval, rval, rtol=0, atol=1e-4 * max(1.0, np.abs(rval).max())), (d, n_items, k)
        assert (np.diff(gval, axis=1) <= 1e-4).all(), (d, n_items, k)
        assert (got == ridx).mean() > 0.99, (d, n_items, k, (got == ridx).mean())
        for r in range(nq):
            assert len(set(got[r].tolist())) == kk, (d, n_items, k, r)


@pytest.mark.parametrize("d", [129, 256])
def test_topk_ties_across_slice_boundaries(cuda_lib, d):
    """Identical item rows (bit-identical scores) on both sides of the slice boundaries 4096 and 8192 are the best
    items of every query: they come back in ascending index order, also when k cuts through the tie."""
    import torch
    from buffalo_b200 import backend
    nq, n_items = 6, 8193
    rng = np.random.default_rng(d)
    P = np.abs(rng.normal(size=(nq, d))).astype(np.float32) + 0.1
    Q = (rng.normal(size=(n_items, d)) * 0.01).astype(np.float32)
    tied = np.array([10, 4095, 4096, 4097, 8191, 8192])
    Q[tied] = 1.0
    Qb = (rng.normal(size=n_items) * 0.01).astype(np.float32)
    Qb[tied] = 0.5
    for k in (1, 3, 5, 6, 9):
        idx, _ = backend.topk_device(*(torch.from_numpy(x).cuda() for x in (P, Q, Qb)), k)
        idx = idx.cpu().numpy()
        want = ref_topk(P, Q, Qb, k)[0]        # stable sort: equal scores in ascending index order
        assert np.array_equal(want[:, :min(k, len(tied))], np.tile(tied[:k], (nq, 1)))
        assert np.array_equal(idx, want), (d, k, idx, want)

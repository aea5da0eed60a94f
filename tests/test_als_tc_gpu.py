"""The d = 128 tensor-core row solve (als_tc.cuh) at production depth.

Each fused CTA is persistent and walks a stream of rows; the hand-offs between rows go through rings of NXS = NBV = 8
slots (x buffers, bad-row flags, b / sum q / sum w vectors) and the accumulator barriers flip parity every row, so a
slot is first reused, on a flipped phase, by the 9th row of a CTA's stream.  The launch gives each CTA
ceil(rows / min(rows, #SMs)) rows: the deep tests size their inputs from the SM count so that every CTA walks at least
64 rows (8 laps of every ring).  Split rows (> 1536 nnz), the routing knob _b200_tc_min_class, the host-pointer
path's sub-chunk pipeline (_b200_sub_chunk_nnz), run-to-run reproducibility and the operand scale's dynamic range are
covered here as well.

Bar: check_rows (tests/helpers.py) -- every row within 1e-3 of the fp32 oracle relative to its norm, or, where the
oracle is not decisive, no further from the fp64 mirror than 1.5x the oracle is; loss pieces within 1e-4 relative.
"""
import numpy as np
import pytest

from tests.helpers import (check_loss, check_rows, csr_from_lengths, full_opt, gpu_half, init_factors, oracle_half,
                           rel_err)

pytestmark = pytest.mark.gpu
D = 128
ROWS_PER_CTA = 66     # > 64: every per-row ring of a fused CTA goes round at least 8 times


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tc_opt(**kw):
    return full_opt(d=D, optimizer="ialspp", block_size=32, **kw)


def deep_lengths(rng, nsm):
    """ROWS_PER_CTA rows per SM, all on the fused kernel: 7/8 of them of 65..320 nnz (every residue mod 16, 32, 64 and
    128 -- a k-step, a tile, a two-tile hand-off group, a planner super-chunk -- many times), the rest up to 1536."""
    n = ROWS_PER_CTA * nsm
    nlong = n // 8
    lengths = np.concatenate([rng.integers(65, 321, n - nlong), rng.integers(321, 1537, nlong)])
    rng.shuffle(lengths)
    return lengths


def half_both(opt, Xup, Yop, indptr, keys, vals, axis, **gpu_kw):
    """(GPU, oracle) results of one half-epoch that updates Xup (rows of the CSR) against the opposite factor Yop."""
    Pa, Qa = (Xup, Yop) if axis == 0 else (Yop, Xup)
    return gpu_half(opt, Pa, Qa, indptr, keys, vals, axis, **gpu_kw), oracle_half(opt, Pa, Qa, indptr, keys, vals, axis)


@pytest.mark.parametrize("vals_kind", ["ints", "lognormal"])
def test_deep_fused_stream(cuda_lib, vals_kind):
    """~66 rows per CTA on the fused kernel, both axes (axis 1 with the loss = the LOSS1 instantiation), integer and
    heavy-tailed fractional values.  The SIMT kernels (_b200_kernel_mode=2) are held to the same row-wise bar on the
    same input, so the two paths agree wherever the oracle is decisive."""
    rng = np.random.default_rng(11 if vals_kind == "ints" else 12)
    lengths = deep_lengths(rng, num_sms())
    U, I = len(lengths), 4000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng,
                                          vals="ints" if vals_kind == "ints" else (lambda r, n: r.lognormal(0.0, 1.0, n)))
    X = init_factors(U, D, D, 1, scale=0.05, signed=True)
    Y = init_factors(I, D, D, 2, scale=0.05, signed=True)
    for axis in (0, 1):
        opt = tc_opt()
        (Xf, nf, dnf), (X0, n0, dn0) = half_both(opt, X, Y, indptr, keys, vals, axis)
        Pa, Qa = (X, Y) if axis == 0 else (Y, X)
        Xs, ns, dns = gpu_half(dict(opt, _b200_kernel_mode=2), Pa, Qa, indptr, keys, vals, axis)
        check_rows({"fused": Xf, "simt": Xs}, X0, X, Y, indptr, keys, vals, opt, axis,
                   label="%s axis %d" % (vals_kind, axis))
        check_loss(nf, dnf, n0, dn0)
        check_loss(ns, dns, n0, dn0)


def negative_layouts(lengths, vals, rng):
    """Negative weights (-0.25 v, so that M stays positive definite) in every tile layout the planner distinguishes,
    row by row in turn: only in the first tile, only the last entry, one whole 32-entry tile, a single entry inside an
    otherwise positive 128-entry super-chunk, alternating; plus rows with zero values and untouched rows."""
    v = vals.copy()
    beg = np.concatenate([[0], np.cumsum(lengths)[:-1]])
    for r, (b, n) in enumerate(zip(beg, lengths)):
        kind = r % 7
        if kind == 0:       # first tile only (a few entries of it)
            idx = b + rng.choice(min(n, 32), size=min(n, 32) // 3 + 1, replace=False)
        elif kind == 1:     # the last entry only
            idx = np.array([b + n - 1])
        elif kind == 2:     # one whole tile
            t = rng.integers(0, n // 32)
            idx = b + 32 * t + np.arange(32)
        elif kind == 3:     # one entry inside a 128-entry super-chunk that is otherwise positive
            sc = rng.integers(0, max(1, n // 128))
            idx = np.array([b + min(n - 1, 128 * sc + rng.integers(1, 127))])
        elif kind == 4:     # alternating
            idx = b + np.arange(1, n, 2)
        elif kind == 5:     # zero values in the middle of a positive row
            v[b + rng.choice(n, size=n // 4, replace=False)] = 0.0
            continue
        else:
            continue
        v[idx] *= -0.25
    return v


def test_negative_weight_tile_layouts(cuda_lib):
    """Entries with negative weight travel in their own tiles and are subtracted by the negate-A wgmma; every layout of
    negative entries inside a row, in a deep stream, on both axes."""
    rng = np.random.default_rng(21)
    lengths = deep_lengths(rng, num_sms())
    U, I = len(lengths), 8000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    vals = negative_layouts(lengths, vals, rng)
    assert (vals < 0).any() and (vals == 0).any()
    X = init_factors(U, D, D, 3, scale=0.05, signed=True)
    Y = init_factors(I, D, D, 4, scale=0.05, signed=True)
    for axis in (0, 1):
        opt = tc_opt()
        (Xf, nf, dnf), (X0, n0, dn0) = half_both(opt, X, Y, indptr, keys, vals, axis)
        check_rows({"fused": Xf}, X0, X, Y, indptr, keys, vals, opt, axis, label="axis %d" % axis)
        check_loss(nf, dnf, n0, dn0)


@pytest.mark.parametrize("tc_min_class", [2, 1, 0])
def test_length_edges_and_routing_knob(cuda_lib, tc_min_class):
    """Three rows of every length 65..320 and of the class / chunk edges 383..385, 511..513, 1023..1025, 1535, 1536 in
    one launch; with _b200_tc_min_class 0 or 1 the rows of 1..64 nnz (one-entry tiles, single k-steps) go to the
    tensor-core kernel as well."""
    rng = np.random.default_rng(31 + tc_min_class)
    lens = list(range(65, 321)) + [383, 384, 385, 511, 512, 513, 1023, 1024, 1025, 1535, 1536]
    if tc_min_class < 2:
        lens += list(range(1, 65))
    lengths = np.repeat(np.array(lens, dtype=np.int64), 3)
    rng.shuffle(lengths)
    U, I = len(lengths), 4000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    X = init_factors(U, D, D, 5, scale=0.05, signed=True)
    Y = init_factors(I, D, D, 6, scale=0.05, signed=True)
    for axis in (0, 1):
        opt = tc_opt(_b200_tc_min_class=tc_min_class)
        (Xf, nf, dnf), (X0, n0, dn0) = half_both(opt, X, Y, indptr, keys, vals, axis)
        check_rows({"fused": Xf}, X0, X, Y, indptr, keys, vals, opt, axis, label="axis %d" % axis)
        check_loss(nf, dnf, n0, dn0)


def split_lengths(rng, nrows=2000):
    """nrows split rows (> 1536 nnz): 1537..6000, the chunk edges 2048 k - 1, 2048 k, 2048 k + 1 (last chunks of one
    entry) and one row beyond 12288 nnz."""
    edges = [2048 * k + o for k in (1, 2) for o in (-1, 0, 1)] + [14337]
    lengths = np.concatenate([rng.integers(1537, 6001, nrows - len(edges)), edges])
    rng.shuffle(lengths)
    return lengths


@pytest.mark.parametrize("d", [128, 256])
def test_split_row_fan_out(cuda_lib, d):
    """Thousands of split rows in flight: ~2 chunk items per row, tens per CTA, one 2048-entry scratch slot per row
    (64 KB at d = 128, 256 KB at d = 256), at d = 256 in three passes; both axes."""
    rng = np.random.default_rng(41 + d)
    lengths = split_lengths(rng)
    U, I = len(lengths), 20000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    X = init_factors(U, d, d, 7, scale=0.05, signed=True)
    Y = init_factors(I, d, d, 8, scale=0.05, signed=True)
    for axis in (0, 1):
        opt = full_opt(d=d, optimizer="ialspp", block_size=32)
        (Xf, nf, dnf), (X0, n0, dn0) = half_both(opt, X, Y, indptr, keys, vals, axis)
        check_rows({"split": Xf}, X0, X, Y, indptr, keys, vals, opt, axis, label="d=%d axis %d" % (d, axis))
        check_loss(nf, dnf, n0, dn0)


def device_half(opt, X, Y, indptr, keys, vals):
    """axis-0 half-epoch over the whole CSR through the resident-CSR device path (bind_* / update_device)"""
    import torch
    from buffalo_b200 import backend
    obj = backend.CuALS()
    assert obj.init(opt)
    vdim = obj.get_vdim()
    tX = torch.zeros(X.shape[0], vdim, device="cuda")
    tY = torch.zeros(Y.shape[0], vdim, device="cuda")
    tX[:, :X.shape[1]] = torch.from_numpy(X).cuda()
    tY[:, :Y.shape[1]] = torch.from_numpy(Y).cuda()
    obj.bind_factors(tX, tY)
    obj.bind_csr(0, torch.from_numpy(indptr).cuda(), torch.from_numpy(keys).cuda(), torch.from_numpy(vals).cuda())
    loss = torch.zeros(2, dtype=torch.float64, device="cuda")
    obj.precompute_device(0)
    obj.update_device(0, 0, X.shape[0], loss)
    torch.cuda.synchronize()
    l = loss.cpu().numpy()
    return tX.cpu().numpy(), float(l[0]), float(l[1])


@pytest.mark.parametrize("d", [128, 126])
def test_sub_chunk_pipeline(cuda_lib, d):
    """partial_update cuts a call into row-aligned sub-chunks and pipelines them over three streams (H2D of k + 1 | solve
    of k | D2H of k - 1) with double-buffered staging.  A small _b200_sub_chunk_nnz gives >= 8 sub-chunks, one row
    longer than a sub-chunk among them; the result must equal the device path's on the same data (same kernels, one
    launch set) and pass the oracle's bar.  d = 126 runs the generic kernels with two padding columns (vdim 128),
    which must stay zero."""
    rng = np.random.default_rng(51)
    sub = 40000
    lengths = np.concatenate([rng.integers(1, 400, 2400), [sub + 5000]])
    rng.shuffle(lengths)
    U, I = len(lengths), 60000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    assert indptr[-1] >= 8 * sub
    X = init_factors(U, d, d, 9, scale=0.05, signed=True)
    Y = init_factors(I, d, d, 10, scale=0.05, signed=True)
    opt = full_opt(d=d, optimizer="ialspp", block_size=32)
    Xh, nh, dnh = gpu_half(dict(opt, _b200_sub_chunk_nnz=sub), X, Y, indptr, keys, vals, 0)   # pads, checks padding
    Xd, nd, dnd = device_half(opt, X, Y, indptr, keys, vals)
    assert not Xd[:, d:].any()
    assert rel_err(Xh, Xd[:, :d]) < 1e-5
    check_loss(nh, dnh, nd, dnd, tol=1e-6)
    X0, n0, dn0 = oracle_half(opt, X, Y, indptr, keys, vals, 0)
    check_rows({"sub-chunked": Xh}, X0, X, Y, indptr, keys, vals, opt, 0)
    check_loss(nh, dnh, n0, dn0)


def test_sub_chunk_pipeline_default_size(cuda_lib):
    """One partial_update call of ~36 M entries at d = 128: three sub-chunks of the default 16 Mi entries."""
    rng = np.random.default_rng(52)
    U, I = 120_000, 100_000
    lengths = rng.integers(65, 536, U)
    nnz = int(lengths.sum())
    assert nnz > 2 * (16 << 20)
    indptr = np.cumsum(lengths).astype(np.int64)
    keys = rng.integers(0, I, nnz, dtype=np.int32)     # repeated keys in a row are separate observations to every solver
    vals = rng.integers(1, 4, nnz).astype(np.float32)
    X = init_factors(U, D, D, 11, scale=0.05, signed=True)
    Y = init_factors(I, D, D, 12, scale=0.05, signed=True)
    opt = tc_opt()
    (Xf, nf, dnf), (X0, n0, dn0) = half_both(opt, X, Y, indptr, keys, vals, 0)
    check_rows({"default": Xf}, X0, X, Y, indptr, keys, vals, opt, 0)
    check_loss(nf, dnf, n0, dn0)


class DeviceRun:
    """One handle on resident device data; run() restores the updated factor and solves the axis again.  The handle
    keeps its binned row lists (FastCache): a repeat reuses the row placement, a fresh handle bins again, and since rows
    reach their class lists through an atomic cursor, that changes which CTA solves a row next to which neighbours."""

    def __init__(self, opt, X, Y, indptr, keys, vals, axis):
        import torch
        from buffalo_b200 import backend
        self.obj = backend.CuALS()
        assert self.obj.init(opt)
        self.axis = axis
        self.X0 = torch.from_numpy(X).cuda()
        self.tX = self.X0.clone()
        tY = torch.from_numpy(Y).cuda()
        tP, tQ = (self.tX, tY) if axis == 0 else (tY, self.tX)
        self.obj.bind_factors(tP, tQ)
        self.obj.bind_csr(axis, torch.from_numpy(indptr).cuda(), torch.from_numpy(keys).cuda(),
                          torch.from_numpy(vals).cuda())

    def run(self):
        import torch
        self.tX.copy_(self.X0)
        loss = torch.zeros(2, dtype=torch.float64, device="cuda")
        self.obj.precompute_device(self.axis)
        self.obj.update_device(self.axis, 0, self.tX.shape[0], loss)
        torch.cuda.synchronize()
        return self.tX.cpu().numpy(), loss.cpu().numpy()


def test_reproducible_across_row_placements(cuda_lib):
    """The deep fused problem on two fresh handles, then once more on the second.  Every row's arithmetic is fixed and
    only its CTA and neighbours change, so the fused and the SIMT factors must be bitwise identical: a difference points to
    state leaking from one row into the next.  Loss values are fp64 atomics (order-dependent): 1e-12 relative.
    The split path adds chunk matrices with fp32 atomicAdd in arrival order and is not bitwise reproducible; its
    run-to-run spread is bounded by 1e-5 relative per row (measured 1.4e-7 on an H100 80GB HBM3 SXM, 700 W)."""
    rng = np.random.default_rng(61)
    lengths = deep_lengths(rng, num_sms())
    U, I = len(lengths), 4000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    X = init_factors(U, D, D, 13, scale=0.05, signed=True)
    Y = init_factors(I, D, D, 14, scale=0.05, signed=True)
    for axis in (0, 1):
        for mode in (0, 2):
            opt = tc_opt(_b200_kernel_mode=mode)
            a = DeviceRun(opt, X, Y, indptr, keys, vals, axis).run()
            hb = DeviceRun(opt, X, Y, indptr, keys, vals, axis)
            b, c = hb.run(), hb.run()
            for other in (b, c):
                diff = np.flatnonzero((a[0] != other[0]).any(axis=1))
                assert not len(diff), (axis, mode, len(diff), [(int(r), int(lengths[r])) for r in diff[:8]])
                assert np.allclose(a[1], other[1], rtol=1e-12, atol=0), (axis, mode, a[1], other[1])
    # split rows: bounded run-to-run spread
    lengths = split_lengths(np.random.default_rng(62), nrows=400)
    U, I = len(lengths), 20000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    X = init_factors(U, D, D, 15, scale=0.05, signed=True)
    Y = init_factors(I, D, D, 16, scale=0.05, signed=True)
    runs = [DeviceRun(tc_opt(), X, Y, indptr, keys, vals, 0).run()[0] for _ in range(3)]
    spread = max(float((np.linalg.norm(r - runs[0], axis=1) / np.linalg.norm(runs[0], axis=1)).max()) for r in runs[1:])
    print("split-row run-to-run spread: %.3g" % spread)
    assert spread < 1e-5, spread


def range_case(case, rng, nsm):
    """(opt, indptr, keys, vals, X, Y) of one operand-range case.  Opposite-factor row 0, and in the lognormal-norm case
    the 1% largest rows, are never observed: they set max|Y| (the launch's operand scale) and enter the Gram matrix only.
    (A row that itself observes the largest rows of such a factor is fp32-ill-conditioned: there the oracle, the generic,
    the SIMT and the tensor-core kernels all land 1e-4..4e-2 away from the fp64 solution, in no particular order --
    DESIGN.md 4.1.)"""
    lengths = deep_lengths(rng, nsm)
    U, I = len(lengths), 4000
    vals_kind = "lognormal" if case == "lognormal_values" else "ints"
    X = init_factors(U, D, D, 17, scale=0.05, signed=True)
    Y = init_factors(I, D, D, 18, scale=0.05, signed=True)
    opt = tc_opt()
    observable = np.arange(1, I)
    if case == "factor_norms_lognormal":
        norms = rng.lognormal(0.0, 1.5, I).astype(np.float32)
        Y[:, :D] *= norms[:, None]
        observable = observable[norms[1:] <= np.quantile(norms, 0.99)]
    elif case.startswith("alpha_"):
        opt["alpha"] = float(case[len("alpha_"):])
    elif case == "reference_init":
        X = init_factors(U, D, D, 19)
        Y = init_factors(I, D, D, 20)
    indptr, keys, vals = csr_from_lengths(lengths, len(observable), rng, vals=vals_kind)
    keys = observable[keys].astype(np.int32)
    if case == "one_huge_unobserved_row":
        Y[0, :D] *= 1e4
    return opt, indptr, keys, vals, X, Y


RANGE_CASES = ["lognormal_values", "factor_norms_lognormal", "one_huge_unobserved_row", "alpha_0", "alpha_0.5", "alpha_40",
               "reference_init"]


@pytest.mark.parametrize("case", RANGE_CASES)
def test_operand_range(cuda_lib, case):
    """One launch-wide power-of-two operand scale comes from the largest |Y| and |w| anywhere in the launch
    (tc_scale_kernel); a deep launch per case where that scale is far from most rows' operands, or the problem is badly
    conditioned (the reference's own abs(N(0, 1/d^2)) initialisation), judged by the row-wise bar."""
    rng = np.random.default_rng(71 + RANGE_CASES.index(case))
    opt, indptr, keys, vals, X, Y = range_case(case, rng, num_sms())
    (Xf, nf, dnf), (X0, n0, dn0) = half_both(opt, X, Y, indptr, keys, vals, 0)
    check_rows({"fused": Xf}, X0, X, Y, indptr, keys, vals, opt, 0, label=case)
    check_loss(nf, dnf, n0, dn0)

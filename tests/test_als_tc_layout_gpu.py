"""The shared-memory layout of the fused d = 128 tensor-core row solve (als_tc.cuh).

A group of two gathered tiles and its fp16 operand slabs share one stage of a three-stage ring (gathered, converted in
place, read by wgmma), and every CTA loads 2^2e (G + reg I) into shared memory once, as a block-packed lower
triangle that starts the accumulator of each of its rows.  These tests drive the ring through many laps and row ends
at every phase, and change reg between the two axes, against the fp32 oracle at the bar of tests/helpers.py
check_rows.
"""
import numpy as np
import pytest

from tests.helpers import (check_rows, csr_from_lengths, full_opt, gpu_half, init_factors, oracle_half,
                           transpose_csr)

pytestmark = pytest.mark.gpu
D = 128


def num_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def tc_opt(**kw):
    return full_opt(d=D, optimizer="ialspp", block_size=32, **kw)


def test_long_row_stream_per_cta(cuda_lib):
    """More than 10 000 rows of 65..300 nnz per CTA in one fused launch (the launch has one CTA per SM and deals the
    rows out round-robin), so each CTA starts thousands of rows back to back from the shared-memory copy of G and its
    stage ring wraps thousands of times.  The CSR (~240M nnz) is built on the device; the oracle re-solves a random
    sample of rows from the same state (a row's solve depends only on its own entries and on G)."""
    import torch
    from buffalo_b200 import backend

    dev = torch.device("cuda", 0)
    g = torch.Generator(device=dev)
    g.manual_seed(2031)
    U, I = 10_050 * num_sms(), 50_000
    lengths = torch.randint(65, 301, (U,), device=dev, generator=g)
    indptr = torch.cumsum(lengths, 0)
    nnz = int(indptr[-1].item())
    begin = indptr - lengths
    start = torch.randint(0, I - 300, (U,), device=dev, generator=g)   # a row's keys: a sorted run of distinct items
    keys = (torch.repeat_interleave(start - begin, lengths) + torch.arange(nnz, device=dev)).to(torch.int32)
    vals = torch.randint(1, 4, (nnz,), device=dev, generator=g).to(torch.float32)
    X = (torch.randn(U, D, device=dev, generator=g) * 0.05).contiguous()
    Y = (torch.randn(I, D, device=dev, generator=g) * 0.05).contiguous()

    sample = torch.sort(torch.randperm(U, device=dev, generator=g)[:1500]).values
    X_before = X[sample].cpu().numpy()
    opt = tc_opt()
    obj = backend.CuALS()
    assert obj.init(opt)
    assert obj.get_vdim() == D
    obj.bind_factors(X, Y)
    obj.bind_csr(0, indptr, keys, vals)
    loss = torch.zeros(2, dtype=torch.float64, device=dev)
    obj.precompute_device(0)
    obj.update_device(0, 0, U, loss)
    torch.cuda.synchronize()

    sl = lengths[sample]
    sub_begin = torch.cumsum(sl, 0) - sl
    idx = torch.repeat_interleave(begin[sample] - sub_begin, sl) + torch.arange(int(sl.sum().item()), device=dev)
    sub_indptr = torch.cumsum(sl, 0).cpu().numpy().astype(np.int64)
    sub_keys, sub_vals = keys[idx].cpu().numpy(), vals[idx].cpu().numpy()
    Yh = Y.cpu().numpy()
    X0, _, _ = oracle_half(opt, X_before, Yh, sub_indptr, sub_keys, sub_vals, 0)
    check_rows({"fused": X[sample].cpu().numpy()}, X0, X_before, Yh, sub_indptr, sub_keys, sub_vals, opt, 0,
               label="%d rows per CTA" % (U // num_sms()))


def test_short_and_long_rows_alternate(cuda_lib):
    """The CSR alternates 65-nnz rows with 1536- and 1505-nnz rows, ~8 of each kind per CTA.  The launch's row list is
    binned by length, so a CTA takes its short rows first: 3 tiles each, so their row ends fall on either tile of a
    two-tile group, in every stage.  Its long rows (48 and 47 tiles, in random order) then end at shifting stages and
    tiles as well, so stages are reused across row ends at every phase of the ring."""
    rng = np.random.default_rng(41)
    n = 8 * num_sms()
    long_rows = rng.choice([1536, 1505], size=n)
    lengths = np.stack([np.full(n, 65), long_rows], axis=1).reshape(-1)
    U, I = len(lengths), 4000
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    X = init_factors(U, D, D, 1, scale=0.05, signed=True)
    Y = init_factors(I, D, D, 2, scale=0.05, signed=True)
    opt = tc_opt()
    Xf, _, _ = gpu_half(opt, X, Y, indptr, keys, vals, 0)
    X0, _, _ = oracle_half(opt, X, Y, indptr, keys, vals, 0)
    check_rows({"fused": Xf}, X0, X, Y, indptr, keys, vals, opt, 0, label="65 / 1536 / 1505 nnz")


def test_reg_differs_between_axes(cuda_lib):
    """One handle trains a user pass and then an item pass with reg_u != reg_i (and the loss on): each launch must start
    its rows from its own G + reg I, which a stale shared-memory copy or the other axis' reg would miss by far more than
    the bar."""
    import oracle
    from buffalo_b200 import backend

    rng = np.random.default_rng(43)
    U, I = 4 * num_sms(), 1500
    lengths = rng.integers(65, 321, U)
    indptr, keys, vals = csr_from_lengths(lengths, I, rng)
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
    P = init_factors(U, D, D, 1, scale=0.05, signed=True)
    Q = init_factors(I, D, D, 2, scale=0.05, signed=True)
    opt = tc_opt(reg_u=0.05, reg_i=3.0)
    g = backend.CuALS()
    assert g.init(opt)
    o = oracle.OracleALS()
    o.init(opt)
    Pg, Qg, Po, Qo = P.copy(), Q.copy(), P.copy(), Q.copy()
    g.initialize_model(Pg, Qg)
    o.initialize_model(Po, Qo)
    for axis, (ind, k, v, rows) in enumerate([(indptr, keys, vals, U), (cind, ckeys, cvals, I)]):
        Xb = (Pg if axis == 0 else Qg).copy()
        Yb = Qg if axis == 0 else Pg
        g.precompute(axis)
        o.precompute(axis)
        g.partial_update(0, rows, ind, k, v, axis)
        o.partial_update(0, rows, ind, k, v, axis)
        check_rows({"gpu": Pg if axis == 0 else Qg}, Po if axis == 0 else Qo, Xb, Yb, ind, k, v, opt, axis,
                   label="axis %d" % axis)

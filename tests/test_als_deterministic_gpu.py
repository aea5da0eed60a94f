"""Deterministic ALS (option `deterministic`) on the GPU: with the same factors, CSR, options and feed, P, Q and the
training loss are bitwise equal from run to run -- split rows are summed chunk by chunk in a fixed order and the loss by
a fixed tree over per-row terms -- and the result is still the ALS the oracle computes.

One CSR shape serves every kernel test: empty rows, rows of one entry, every row-length class of the tuned kernels,
several split rows of 1537..12288 entries, one of 9000 (more than three 2048-entry chunks) and one of 40000 (more than
16 chunks); values all-ones, or lognormal with a share of negative weights.
"""
import os

import numpy as np
import pytest

from tests.helpers import check_loss, check_rows, full_opt, gpu_half, init_factors, oracle_half, row_rel_err

pytestmark = pytest.mark.gpu

N = 42000            # rows of either axis, and the key range: the longest row has 40000 entries
SPECIAL = [0, 0, 1, 1, 2, 31, 32, 33, 64, 65, 100, 128, 129, 200, 256, 257, 400, 512, 513, 900, 1536,      # classes 0..5
           1537, 2047, 2048, 2049, 3000, 4096, 4097, 6000, 9000, 12288,                                 # class 6, split
           12289, 40000]                                                                                 # class 7


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32 if a.dtype == np.float32 else np.uint64)


def same_bits(a, b):
    return a.shape == b.shape and np.array_equal(bits(a), bits(b))


def make_side(seed, kind, long_rows=True):
    """(indptr, keys, vals) of N rows: the SPECIAL lengths three times over (twice without the 40000 row) among short
    rows of 0..40 entries.  Keys are drawn with replacement: a repeated key is a separate observation to every solver."""
    rng = np.random.default_rng(seed)
    special = [n for n in SPECIAL if long_rows or n <= 1536]
    lengths = rng.integers(0, 41, N)
    where = rng.choice(N, size=3 * len(special), replace=False)
    lengths[where] = np.tile(special, 3)
    if long_rows:
        lengths[where[-1]] = lengths[where[-1 - len(special)]] = 5000      # 40000 once is enough
    nnz = int(lengths.sum())
    keys = rng.integers(0, N, nnz).astype(np.int32)
    if kind == "ones":
        vals = np.ones(nnz, np.float32)
    else:
        vals = rng.lognormal(0.0, 1.0, nnz).astype(np.float32)
        vals[rng.random(nnz) < 0.05] *= -0.25          # M stays positive definite
    return np.cumsum(lengths).astype(np.int64), keys, vals


def start_factors(d):
    return (init_factors(N, d, d, 101, scale=0.05, signed=True), init_factors(N, d, d, 102, scale=0.05, signed=True))


def resident_run(opt, P0, Q0, sides, iters=3):
    """`iters` ALS iterations through the device-resident ABI on a fresh handle -> (P, Q, losses[iters, 2])."""
    import torch
    from buffalo_b200 import backend
    obj = backend.CuALS()
    assert obj.init(opt), getattr(obj, "last_error", "")
    tP, tQ = torch.from_numpy(P0).cuda(), torch.from_numpy(Q0).cuda()
    obj.bind_factors(tP, tQ)
    for axis, (indptr, keys, vals) in enumerate(sides):
        obj.bind_csr(axis, torch.from_numpy(indptr).cuda(), torch.from_numpy(keys).cuda(), torch.from_numpy(vals).cuda())
    losses = []
    for _ in range(iters):
        loss = torch.zeros(2, dtype=torch.float64, device="cuda")
        for axis in (0, 1):
            obj.precompute_device(axis)
            obj.update_device(axis, 0, N, loss)
        losses.append(loss.cpu().numpy())
    torch.cuda.synchronize()
    return tP.cpu().numpy(), tQ.cpu().numpy(), np.stack(losses)


def assert_same_run(a, b, what):
    for name, x, y in zip(("P", "Q", "loss"), a, b):
        assert same_bits(x, y), "%s: %s differs in %d elements" % (what, name, int((bits(x) != bits(y)).sum()))
    assert np.isfinite(a[0]).all() and np.isfinite(a[1]).all() and np.isfinite(a[2]).all() and (a[2][:, 1] > 0).all()


def det_opt(d, **kw):
    kw.setdefault("optimizer", "ialspp")
    return full_opt(d=d, deterministic=True, **kw)


# ---- 1. run to run ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,kind", [(128, "ones"), (128, "lognormal"), (256, "lognormal")])
def test_run_to_run_bitwise(cuda_lib, d, kind):
    """d = 128: fused tensor-core rows, split rows and the SIMT classes 0, 1; d = 256: split rows and SIMT classes."""
    sides = (make_side(1, kind), make_side(2, kind))
    P0, Q0 = start_factors(d)
    a = resident_run(det_opt(d), P0, Q0, sides)
    b = resident_run(det_opt(d), P0, Q0, sides)
    assert_same_run(a, b, "d=%d %s" % (d, kind))


# ---- 2. batching changes nothing -------------------------------------------------------------------------------------
@pytest.mark.parametrize("d", [128, 256])
def test_scratch_batches_do_not_change_a_bit(cuda_lib, d):
    """A 0.1 MB budget is below two chunk slots (64.5 KB each at d = 128): every batch holds exactly one long row."""
    sides = (make_side(1, "lognormal"), make_side(2, "lognormal"))
    P0, Q0 = start_factors(d)
    one = resident_run(det_opt(d), P0, Q0, sides, iters=2)
    many = resident_run(det_opt(d, _b200_det_scratch_mb=0.1), P0, Q0, sides, iters=2)
    some = resident_run(det_opt(d, _b200_det_scratch_mb=3), P0, Q0, sides, iters=2)
    assert_same_run(one, many, "one row per batch")
    assert_same_run(one, some, "3 MB batches")


# ---- 3. the loss on every routing ------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,kw", [(128, dict(_b200_kernel_mode=0)), (128, dict(_b200_kernel_mode=1)),
                                  (128, dict(_b200_kernel_mode=2)), (20, dict(optimizer="manual_cg")),
                                  (20, dict(optimizer="llt")), (64, dict(optimizer="ialspp"))],
                         ids=["tc", "generic", "simt", "manual_cg", "llt", "ialspp64"])
def test_every_routing_bitwise(cuda_lib, d, kw):
    sides = (make_side(1, "lognormal"), make_side(2, "lognormal"))
    P0, Q0 = start_factors(d)
    a = resident_run(det_opt(d, **kw), P0, Q0, sides, iters=2)
    b = resident_run(det_opt(d, **kw), P0, Q0, sides, iters=2)
    assert_same_run(a, b, str(kw))


# ---- 4. still ALS ----------------------------------------------------------------------------------------------------
def device_half(opt, P0, Q0, side, axis):
    import torch
    from buffalo_b200 import backend
    obj = backend.CuALS()
    assert obj.init(opt)
    tP, tQ = torch.from_numpy(P0).cuda(), torch.from_numpy(Q0).cuda()
    obj.bind_factors(tP, tQ)
    obj.bind_csr(axis, *[torch.from_numpy(x).cuda() for x in side])
    loss = torch.zeros(2, dtype=torch.float64, device="cuda")
    obj.precompute_device(axis)
    obj.update_device(axis, 0, N, loss)
    torch.cuda.synchronize()
    l = loss.cpu().numpy()
    return (tP if axis == 0 else tQ).cpu().numpy(), float(l[0]), float(l[1])


@pytest.mark.parametrize("axis", [0, 1])
def test_matches_oracle_and_default_mode(cuda_lib, axis):
    d = 128
    side = make_side(3 + axis, "lognormal")
    P0, Q0 = start_factors(d)
    opt = full_opt(d=d, optimizer="ialspp")
    Xd, nd, dd = device_half(dict(opt, deterministic=True), P0, Q0, side, axis)
    Xa, na, da = device_half(opt, P0, Q0, side, axis)
    X0, n0, d0 = oracle_half(opt, P0, Q0, *side, axis)
    Xb, Y = (P0, Q0) if axis == 0 else (Q0, P0)
    check_rows({"deterministic": Xd, "default": Xa}, X0, Xb, Y, *side, opt, axis, label="axis %d" % axis)
    check_loss(nd, dd, n0, d0)
    check_loss(nd, dd, na, da)
    assert row_rel_err(Xd, Xa).max() < 1e-3


# ---- 5. host-pointer path --------------------------------------------------------------------------------------------
def test_host_pointer_path_same_feed(cuda_lib):
    d = 128
    side = make_side(5, "lognormal")
    P0, Q0 = start_factors(d)
    opt = det_opt(d, _b200_sub_chunk_nnz=60000)
    a = gpu_half(opt, P0, Q0, *side, 0, chunks=3)
    b = gpu_half(opt, P0, Q0, *side, 0, chunks=3)
    assert same_bits(a[0], b[0]) and a[1] == b[1] and a[2] == b[2]


@pytest.mark.parametrize("axis", [0, 1])
def test_host_pointer_path_equals_resident_with_uniform_values(cuda_lib, axis):
    """All-ones values: every launch sees the same max|v|, so the operand scale, and with it every bit of the factors,
    is the same however the rows are cut into sub-chunks.  The loss is a host sum of sub-chunk sums: 1e-12."""
    d = 128
    side = make_side(6, "ones")
    P0, Q0 = start_factors(d)
    Xr, nr, dr = device_half(det_opt(d), P0, Q0, side, axis)
    for sub, chunks in ((50000, 1), (300000, 4)):
        Xh, nh, dh = gpu_half(det_opt(d, _b200_sub_chunk_nnz=sub), P0, Q0, *side, axis, chunks=chunks)
        assert same_bits(Xh, Xr), (sub, int((bits(Xh) != bits(Xr)).sum()))
        assert abs(nh - nr) <= 1e-12 * abs(nr) and abs(dh - dr) <= 1e-12 * abs(dr), (nh, nr, dh, dr)


# ---- 6. rows without split rows --------------------------------------------------------------------------------------
@pytest.mark.parametrize("d,kw", [(128, {}), (128, dict(_b200_kernel_mode=2)), (256, {}), (20, dict(optimizer="manual_cg"))],
                         ids=["tc", "simt", "simt256", "manual_cg"])
def test_factors_equal_default_mode_without_split_rows(cuda_lib, d, kw):
    """No row above 1536 entries: only the loss path differs between the modes, so the factors are bitwise the default
    mode's (whose rows are each solved by one CTA in a fixed order)."""
    kw.setdefault("optimizer", "ialspp")
    sides = (make_side(7, "lognormal", long_rows=False), make_side(8, "lognormal", long_rows=False))
    P0, Q0 = start_factors(d)
    det = resident_run(full_opt(d=d, deterministic=True, **kw), P0, Q0, sides, iters=2)
    dflt = resident_run(full_opt(d=d, **kw), P0, Q0, sides, iters=2)
    assert same_bits(det[0], dflt[0]) and same_bits(det[1], dflt[1])
    assert np.allclose(det[2], dflt[2], rtol=1e-10, atol=0)


# ---- 7. API ----------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def small_mm(tmp_path_factory):
    """600 x 900 MatrixMarket file with a planted rank-6 structure.  No row reaches 1537 entries, so d = 128 runs the
    fused tensor-core and SIMT classes and the loss tree here; split rows are covered by the kernel tests above."""
    rng = np.random.default_rng(9)
    U, I, k = 600, 900, 6
    S = rng.normal(size=(U, k)) @ rng.normal(size=(I, k)).T + rng.gumbel(size=(U, I)) * 0.5
    rows, cols = np.nonzero(S > np.quantile(S, 0.92))
    vals = rng.integers(1, 6, len(rows))
    d = tmp_path_factory.mktemp("als_det")
    main = os.path.join(d, "main")
    with open(main, "w") as f:
        f.write("%%MatrixMarket matrix coordinate integer general\n%d %d %d\n" % (U, I, len(rows)))
        f.write("".join("%d %d %d\n" % (r + 1, c + 1, v) for r, c, v in zip(rows, cols, vals)))
    return dict(main=main, dir=str(d))


@pytest.mark.parametrize("d", [128, 32])
def test_api_training_is_repeatable(cuda_lib, small_mm, d):
    from buffalo import ALS, ALSOption, aux
    from buffalo.data import MatrixMarketOptions
    from buffalo.misc import log
    log.set_log_level(log.WARN)
    runs = []
    for name in ("a", "b"):
        do = MatrixMarketOptions().get_default_option()
        do.input.main = small_mm["main"]
        do.data.path = os.path.join(small_mm["dir"], "%s_%d.h5py" % (name, d))
        do.data.validation.p, do.data.validation.max_samples = 0.1, 5000
        opt = ALSOption().get_default_option()
        opt.update(d=d, num_iters=4, random_seed=11, deterministic=True, validation=aux.Option({"topk": 10}))
        np.random.seed(5)            # the validation split is drawn when the database is created
        m = ALS(opt, data_opt=do)
        m.initialize()
        ret = m.train()
        runs.append((m.P.copy(), m.Q.copy(), ret, m.get_validation_results()))
    (Pa, Qa, ra, va), (Pb, Qb, rb, vb) = runs
    assert same_bits(Pa, Pb) and same_bits(Qa, Qb)
    assert ra["train_loss"] == rb["train_loss"] and ra["train_loss"] > 0
    assert va == vb and va["ndcg"] > 0

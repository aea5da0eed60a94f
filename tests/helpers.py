"""Synthetic inputs (seeded, NumPy only) and the ALS half-epoch drivers and row-wise checks shared by the tests."""
import numpy as np

FACTOR_TOL = 1e-3
ROW_CLASS_EDGES = (32, 64, 128, 256, 512, 1536, 12288)   # row-length classes of the tuned kernels (als_fast.cuh)


def make_csr(num_rows, num_cols, nnz, seed, empty_rows=0, vals="ints", sort_keys=True):
    """Random CSR in the reference layout (buffalo/data/base.py:187-192): indptr = exclusive END
    offsets (no leading zero), keys int32 sorted within a row, vals float32."""
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, num_rows, nnz)
    if empty_rows:
        dead = rng.choice(num_rows, size=empty_rows, replace=False)
        rows = rows[~np.isin(rows, dead)]
    cols = rng.integers(0, num_cols, len(rows)).astype(np.int32)
    pairs = np.unique(np.stack([rows, cols], axis=1), axis=0) if sort_keys else np.stack([rows, cols], axis=1)
    rows, cols = pairs[:, 0], pairs[:, 1].astype(np.int32)
    order = np.lexsort((cols, rows))
    rows, cols = rows[order], cols[order]
    indptr = np.cumsum(np.bincount(rows, minlength=num_rows)).astype(np.int64)
    if vals == "ints":
        v = rng.integers(1, 6, len(rows)).astype(np.float32)
    else:
        v = np.ones(len(rows), dtype=np.float32)
    return indptr, np.ascontiguousarray(cols), v, rows.astype(np.int64)


def transpose_csr(indptr, keys, vals, num_rows, num_cols):
    """colwise copy, sorted by (col, row) like fileio.hpp:330-341."""
    beg = np.concatenate([[0], indptr[:-1]])
    rows = np.repeat(np.arange(num_rows), indptr - beg)
    order = np.lexsort((rows, keys))
    cind = np.cumsum(np.bincount(keys, minlength=num_cols)).astype(np.int64)
    return cind, rows[order].astype(np.int32), np.ascontiguousarray(vals[order])


def init_factors(rows, d, vdim, seed, scale=None, signed=False):
    """abs(N(0, 1/d^2)) like buffalo/algo/als.py:85-86 (scaled up so the problem is well conditioned)."""
    rng = np.random.default_rng(seed)
    s = (1.0 / d ** 2) if scale is None else scale
    F = rng.normal(scale=s, size=(rows, d)).astype(np.float32)
    if not signed:
        F = np.abs(F)
    out = np.zeros((rows, vdim), dtype=np.float32)
    out[:, :d] = F
    return out


def rel_err(a, b):
    a = np.asarray(a, dtype=np.float64)
    b = np.asarray(b, dtype=np.float64)
    return float(np.abs(a - b).max() / max(np.abs(b).max(), 1e-30))


def csr_from_lengths(lengths, num_cols, rng, vals="ints"):
    """CSR with the given row lengths: distinct keys per row, sorted; vals "ints" (1..3), "lognormal" (sigma 2) or a
    callable (rng, n) -> values."""
    lengths = np.asarray(lengths, dtype=np.int64)
    keys = np.concatenate([np.sort(rng.choice(num_cols, size=int(n), replace=False)) for n in lengths]).astype(np.int32)
    indptr = np.cumsum(lengths).astype(np.int64)
    if vals == "ints":
        v = rng.integers(1, 4, len(keys))
    elif vals == "lognormal":
        v = rng.lognormal(0.0, 2.0, len(keys))
    else:
        v = vals(rng, len(keys))
    return indptr, keys, np.asarray(v, dtype=np.float32)


def row_class(n):
    """row-length class of a row of n entries (als_fast.cuh fast_class_of)"""
    return int(np.searchsorted(ROW_CLASS_EDGES, n))


def full_opt(**kw):
    opt = dict(d=20, optimizer="manual_cg", num_workers=8, compute_loss_on_training=True, alpha=8.0, reg_u=0.1,
               reg_i=0.1, block_size=32, adaptive_reg=False, num_cg_max_iters=3, eps=1e-10, cg_tolerance=1e-10)
    opt.update(kw)
    return opt


def gpu_half(opt, P, Q, indptr, keys, vals, axis, chunks=1, placeholder=None):
    """One half-epoch through the host-pointer C ABI (init / initialize_model / precompute / partial_update)."""
    from buffalo_b200 import backend
    obj = backend.CuALS()
    assert obj.init(opt)
    vdim = obj.get_vdim()
    d = opt["d"]
    Pp = np.zeros((P.shape[0], vdim), np.float32)
    Qp = np.zeros((Q.shape[0], vdim), np.float32)
    Pp[:, :d], Qp[:, :d] = P[:, :d], Q[:, :d]
    obj.initialize_model(Pp, Qp)
    if placeholder is not None:
        obj.set_placeholder(placeholder[0], placeholder[1], len(keys))
    obj.precompute(axis)
    rows = P.shape[0] if axis == 0 else Q.shape[0]
    bounds = np.linspace(0, rows, chunks + 1).astype(int)
    nume = deno = 0.0
    for a, b in zip(bounds[:-1], bounds[1:]):
        beg = 0 if a == 0 else int(indptr[a - 1])
        end = int(indptr[b - 1]) if b > 0 else 0
        k = np.ascontiguousarray(keys[beg:end]) if end > beg else np.zeros(1, np.int32)
        v = np.ascontiguousarray(vals[beg:end]) if end > beg else np.zeros(1, np.float32)
        n_, d_ = obj.partial_update(int(a), int(b), indptr, k, v, axis)
        nume += n_
        deno += d_
    X = Pp if axis == 0 else Qp
    assert not X[:, d:].any(), "padding columns must stay zero"
    return X[:, :d].copy(), nume, deno


def oracle_half(opt, P, Q, indptr, keys, vals, axis):
    import oracle
    o = oracle.OracleALS()
    o.init(opt)
    P1, Q1 = P.copy(), Q.copy()
    o.initialize_model(P1, Q1)
    o.precompute(axis)
    rows = P.shape[0] if axis == 0 else Q.shape[0]
    n, dn = o.partial_update(0, rows, indptr, keys, vals, axis)
    return (P1 if axis == 0 else Q1), n, dn


def check_loss(n, dn, n0, dn0, tol=1e-4):
    assert abs(n - n0) <= tol * max(1.0, abs(n0)), (n, n0)
    assert abs(dn - dn0) <= tol * max(1.0, abs(dn0)), (dn, dn0)


def row_rel_err(X, X0):
    """per-row distance of X from X0, relative to the norm of X0's row"""
    X = np.asarray(X, dtype=np.float64)
    X0 = np.asarray(X0, dtype=np.float64)
    return np.linalg.norm(X - X0, axis=1) / np.maximum(np.linalg.norm(X0, axis=1), 1e-6)


def check_rows(results, X0, X_before, Y, indptr, keys, vals, opt, axis, tol=FACTOR_TOL, label=""):
    """Row-wise bar for GPU factors `results` ({name: X}) against the fp32 oracle's X0 of the same half-epoch.

    A row passes when it lies within `tol` of the oracle relative to the oracle row's norm.  Where it does not, the
    oracle is not decisive by itself (its sequential fp32 sums drift on ill-conditioned rows), so the row is re-solved by
    the fp64 mirror (oracle/np_mirror.py) from X_before (the rows' state before the update) and the opposite factor Y:
    the GPU row must then be no further from the mirror than 1.5x the oracle's own distance (or within `tol`).  The
    mirror only runs on the rows that miss the first bar.  Returns {name: per-row error against the oracle}."""
    errs = {name: row_rel_err(X, X0) for name, X in results.items()}
    miss = np.flatnonzero(np.logical_or.reduce([e >= tol for e in errs.values()]))
    if len(miss):
        from oracle import np_mirror
        d = X0.shape[1]
        beg = np.concatenate([[0], indptr[:-1]])
        lens = indptr[miss] - beg[miss]
        sub_keys = np.concatenate([keys[beg[r]:indptr[r]] for r in miss]).astype(np.int32)
        sub_vals = np.concatenate([vals[beg[r]:indptr[r]] for r in miss]).astype(np.float32)
        Xm, _, _ = np_mirror.als_half_epoch(X_before[miss, :d], Y[:, :d], np.cumsum(lens), sub_keys, sub_vals, opt, axis)
        eo = row_rel_err(X0[miss], Xm)
        for name, X in results.items():
            eg = row_rel_err(X[miss], Xm)
            bad = np.flatnonzero(eg > np.maximum(1.5 * eo, tol))
            assert not len(bad), "%s %s: %d rows fail, e.g. %s" % (label, name, len(bad), [
                dict(row=int(miss[i]), nnz=int(lens[i]), row_class=row_class(lens[i]), err_vs_oracle=float(errs[name][miss[i]]),
                     err_vs_fp64=float(eg[i]), oracle_vs_fp64=float(eo[i])) for i in bad[:5]])
    for name, X in results.items():
        assert np.isfinite(X).all(), (label, name)
    return errs

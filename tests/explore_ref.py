"""fp64 NumPy restatement of ALS.posterior_sample (DESIGN.md 4.17, posterior_sample_kernel): per history row the
matrix A_r of the user half-epoch, its Cholesky factor from numpy.linalg.cholesky, the Box-Muller normals of the
row's Philox words (the Philox of tests/item_fold_in_ref.py, vectorised here and checked against it), y = L^-T z and
the draw mean + scale y."""
import numpy as np

from tests import explain_ref, item_fold_in_ref

POSTERIOR_TAG = 0x54530417
M32 = np.uint64(0xFFFFFFFF)


def philox_np(c0, c1, c2, c3, k0, k1):
    """Philox4x32-10 on uint64 arrays holding 32-bit words (broadcast); returns the four output words."""
    c = [np.asarray(x, dtype=np.uint64) & M32 for x in (c0, c1, c2, c3)]
    k = [np.uint64(k0) & M32, np.uint64(k1) & M32]
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k[0]) & M32, p1 & M32, ((p0 >> np.uint64(32)) ^ c[3] ^ k[1]) & M32,
             p0 & M32]
        k = [(k[0] + np.uint64(0x9E3779B9)) & M32, (k[1] + np.uint64(0xBB67AE85)) & M32]
    return c


def words(seed, key, D):
    """uint64 [len(key), D]: draw_u32(seed, POSTERIOR_TAG, key, t) for t < D, for every draw key."""
    key = np.asarray(key, dtype=np.uint64).reshape(-1, 1)
    q = np.arange((D + 3) // 4, dtype=np.uint64).reshape(1, -1)
    w = philox_np(key & M32, key >> np.uint64(32), q, POSTERIOR_TAG, seed, 0x5EED)
    return np.stack(w, axis=2).reshape(len(key), -1)[:, :D]


def words_scalar(seed, key, D):
    """words() for one key through tests/item_fold_in_ref.draw_u32 (the per-word statement)."""
    return np.array([item_fold_in_ref.draw_u32(seed, POSTERIOR_TAG, int(key), t) for t in range(D)], dtype=np.uint64)


def normals(seed, key, D):
    """fp64 [len(key), D] z: column pair k from w0 = word 2k, w1 = word 2k + 1 as u1 = (w0 + 1) 2^-32, u2 = w1 2^-32,
    sqrt(-2 ln u1) (cos, sin)(2 pi u2); an odd D drops the last sine."""
    W = words(seed, key, D + (D & 1)).astype(np.float64)
    u1, u2 = (W[:, 0::2] + 1.0) * 2.0 ** -32, W[:, 1::2] * 2.0 ** -32
    rad = np.sqrt(-2.0 * np.log(u1))
    z = np.empty((W.shape[0], W.shape[1]))
    z[:, 0::2], z[:, 1::2] = rad * np.cos(2 * np.pi * u2), rad * np.sin(2 * np.pi * u2)
    return z[:, :D]


def row_matrix(G, Q, keys, vals, alpha, reg, adaptive_reg):
    """fp64 A_r = G + alpha sum v q q' + reg kappa I (kappa = entries with adaptive_reg, so 0 for an empty row)."""
    return explain_ref.row_system(G, Q, keys, vals, alpha, reg, adaptive_reg)[0]


def sample_rows(Q, indptr, keys, vals, mean, draw_keys, seed, scale, alpha, reg, adaptive_reg, G=None):
    """(out fp64 [n, d], y fp64 [n, d], failed bool [n]) for the history CSR (END offsets): y = L^-T z per row, out =
    mean + scale y; a row whose A_r is not positive definite gives y = 0 and out = mean (failed).  G defaults to the
    fp64 Gram of Q."""
    Q = np.asarray(Q)
    n, d = len(indptr), Q.shape[1]
    G = Q.astype(np.float64).T @ Q.astype(np.float64) if G is None else np.asarray(G, dtype=np.float64)
    Z = normals(seed, draw_keys, d)
    beg = np.concatenate([[0], indptr[:-1]]).astype(np.int64)
    Y = np.zeros((n, d))
    failed = np.zeros(n, dtype=bool)
    for r in range(n):
        A = row_matrix(G, Q, keys[beg[r]:indptr[r]], vals[beg[r]:indptr[r]], alpha, reg, adaptive_reg)
        try:
            L = np.linalg.cholesky(A)
        except np.linalg.LinAlgError:
            failed[r] = True
            continue
        Y[r] = np.linalg.solve(L.T, Z[r])
    out = np.asarray(mean, dtype=np.float64) + scale * Y
    return out, Y, failed

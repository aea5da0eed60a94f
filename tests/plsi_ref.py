"""CPU references for pLSI (test infrastructure only; the product never imports this module).

``OraclePLSI`` restates plsi::CPLSI (lib/algo_impl/plsi/plsi.cc:40-130) in float32 NumPy with the method set of
CyPLSI (buffalo/algo/_plsi.pyx:13-57).  Its factors are injected through ``initialize_model`` (no random draw), and
it is deterministic: every sum runs in a fixed order.  ``plsi_iteration`` is an independent fp64 restatement, row by
row, of one EM iteration (reset, partial_update over all rows, normalize, swap).
"""
import numpy as np

LATENT_FLOOR = np.float32(1e-10)       # plsi.cc:95
BLOCK_ELEMS = 1 << 22                  # entries x d per vectorised block


def _segment_add(dst, idx, W):
    """dst[idx[j]] += W[j] with the contributions of one index summed in entry order."""
    if len(idx) == 0:
        return
    order = np.argsort(idx, kind="stable")
    si = idx[order]
    starts = np.flatnonzero(np.r_[True, si[1:] != si[:-1]])
    dst[si[starts]] += np.add.reduceat(W[order], starts, axis=0)


class OraclePLSI(object):
    """float32 restatement of CPLSI; P_ / Q_ are the caller's [rows, d] arrays, P / Q the accumulators."""

    def init(self, opt):
        self.d = int(opt["d"])
        return True

    def initialize_model(self, P, Q):
        assert P.dtype == np.float32 and Q.dtype == np.float32 and P.shape[1] == Q.shape[1] == self.d
        self.P_, self.Q_ = P, Q                       # kept by reference, overwritten by swap (plsi.cc:127-130)
        self.P = np.zeros_like(P)
        self.Q = np.zeros_like(Q)

    def reset(self):
        self.P[:] = 0
        self.Q[:] = 0

    def partial_update(self, start_x, next_x, indptr, keys, vals):
        """plsi.cc:72-106; keys / vals hold the chunk from row start_x on.  Returns the loss piece (fp64 sum)."""
        if next_x <= start_x:
            return 0.0
        shifted = 0 if start_x == 0 else int(indptr[start_x - 1])
        ends = np.asarray(indptr[start_x:next_x], dtype=np.int64)
        lens = np.diff(np.concatenate([[shifted], ends]))
        rows = np.repeat(np.arange(start_x, next_x, dtype=np.int64), lens)
        keys = np.asarray(keys[:len(rows)], dtype=np.int64)
        vals = np.asarray(vals[:len(rows)], dtype=np.float32)
        loss = 0.0
        step = max(1, BLOCK_ELEMS // self.d)
        for a in range(0, len(rows), step):
            r, c, v = rows[a:a + step], keys[a:a + step], vals[a:a + step]
            L = np.maximum(self.P_[r] * self.Q_[c], LATENT_FLOOR)
            norm = L.sum(axis=1, dtype=np.float32)
            loss -= float(np.sum(v.astype(np.float64) * np.log(norm).astype(np.float64)))
            W = (L / norm[:, None]) * v[:, None]
            _segment_add(self.P, r, W)
            _segment_add(self.Q, c, W)
        return loss

    def normalize(self, alpha1, alpha2):
        """plsi.cc:108-125, including 0 / 0 for an empty user row when alpha1 == 0."""
        a1 = np.float32(alpha1) / np.float32(self.d)
        a2 = np.float32(alpha2) / np.float32(self.Q.shape[0])
        with np.errstate(invalid="ignore", divide="ignore"):
            self.P += a1
            self.P /= self.P.sum(axis=1, keepdims=True, dtype=np.float32)
            self.Q += a2
            self.Q /= self.Q.sum(axis=0, keepdims=True, dtype=np.float32)

    def swap(self):
        self.P_[:] = self.P
        self.Q_[:] = self.Q


def oracle_iteration(P, Q, indptr, keys, vals, alpha1=1.0, alpha2=1.0):
    """One reference iteration over all rows from (P, Q); returns new copies and the loss numerator."""
    o = OraclePLSI()
    o.init(dict(d=P.shape[1]))
    P1, Q1 = np.array(P, dtype=np.float32), np.array(Q, dtype=np.float32)
    o.initialize_model(P1, Q1)
    o.reset()
    loss = o.partial_update(0, P1.shape[0], indptr, keys, vals)
    o.normalize(alpha1, alpha2)
    o.swap()
    return P1, Q1, loss


def plsi_iteration(P, Q, indptr, keys, vals, alpha1=1.0, alpha2=1.0):
    """fp64 mirror of one iteration, row by row.  Returns (P, Q, loss numerator) in float64."""
    P = np.asarray(P, dtype=np.float64)
    Q = np.asarray(Q, dtype=np.float64)
    d = P.shape[1]
    Pn, Qn = np.zeros_like(P), np.zeros_like(Q)
    loss = 0.0
    beg = 0
    for x in range(P.shape[0]):
        end = int(indptr[x])
        if end > beg:
            c = np.asarray(keys[beg:end], dtype=np.int64)
            v = np.asarray(vals[beg:end], dtype=np.float64)
            lat = np.maximum(P[x][None, :] * Q[c], 1e-10)
            norm = lat.sum(axis=1)
            loss -= float(np.dot(v, np.log(norm)))
            contrib = lat / norm[:, None] * v[:, None]
            Pn[x] += contrib.sum(axis=0)
            np.add.at(Qn, c, contrib)
        beg = end
    with np.errstate(invalid="ignore", divide="ignore"):
        Pn += alpha1 / d
        Pn /= Pn.sum(axis=1, keepdims=True)
        Qn += alpha2 / Q.shape[0]
        Qn /= Qn.sum(axis=0, keepdims=True)
    return Pn, Qn, loss


def random_factors(rows, d, seed, axis):
    """|N(0, 1/d)| normalised like plsi.cc:51-66: axis 1 -> rows sum to 1 (P), axis 0 -> columns sum to 1 (Q)."""
    rng = np.random.default_rng(seed)
    F = np.abs(rng.normal(scale=1.0 / d, size=(rows, d))) + 1e-3 / d
    F /= F.sum(axis=axis, keepdims=True)
    return F.astype(np.float32)

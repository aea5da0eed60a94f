"""fp64 NumPy reference of ALS.explain (DESIGN.md 4.11): per history row the system A x = b of the user half-epoch,
solved with np.linalg.solve, the score of every target, the per-item contributions (entries of one item summed) and the
top-m with ties to the smaller item."""
import numpy as np


def row_system(G, Q, keys, vals, alpha, reg, adaptive_reg):
    """fp64 (A, b): A = G + alpha sum v q q' + reg kappa I, b = sum (1 + alpha v) q; kappa = len(keys) if adaptive_reg."""
    q, v = Q[keys].astype(np.float64), np.asarray(vals, dtype=np.float64)
    kappa = float(len(keys)) if adaptive_reg else 1.0
    A = G + (q * (alpha * v)[:, None]).T @ q + reg * kappa * np.eye(Q.shape[1])
    return A, ((1.0 + alpha * v)[:, None] * q).sum(axis=0)


def merged_contributions(Q, A, keys, vals, alpha, target):
    """(items ascending, their summed contributions (q_i' A^-1 q_j)(1 + alpha v_j)) of one target i"""
    u = np.linalg.solve(A, Q[target].astype(np.float64))
    per_entry = (Q[keys].astype(np.float64) @ u) * (1.0 + alpha * np.asarray(vals, dtype=np.float64))
    items, inv = np.unique(keys, return_inverse=True)
    return items, np.bincount(inv.ravel(), weights=per_entry, minlength=len(items))


def ranked(items, contrib):
    """items and contributions in output order: descending contribution, ties to the smaller item"""
    order = np.lexsort((items, -contrib))
    return items[order], contrib[order]


def explain_rows(Q, indptr, keys, vals, targets, topm, alpha, reg, adaptive_reg, rows=None):
    """The reference of ALS.explain for `rows` (default all) of the history CSR (END offsets).  Returns a list with one
    dict per row: x (the fp64 solve, None for an empty row), scores [k], keys [k, topm], contrib [k, topm] and, per
    target, the full ranked (items, contributions) lists ("ranked", None for a -1 target or an empty row)."""
    Q = np.asarray(Q)
    G = Q.astype(np.float64).T @ Q.astype(np.float64)
    beg = np.concatenate([[0], indptr[:-1]])
    out = []
    for r in (range(len(indptr)) if rows is None else rows):
        k = targets.shape[1]
        res = dict(x=None, scores=np.zeros(k), keys=np.full((k, topm), -1, np.int64), contrib=np.zeros((k, topm)),
                   ranked=[None] * k)
        rk, rv = keys[beg[r]:indptr[r]], vals[beg[r]:indptr[r]]
        if len(rk):
            A, b = row_system(G, Q, rk, rv, alpha, reg, adaptive_reg)
            res["x"] = np.linalg.solve(A, b)
            for t, i in enumerate(targets[r]):
                if i < 0:
                    continue
                res["scores"][t] = Q[i].astype(np.float64) @ res["x"]
                items, c = ranked(*merged_contributions(Q, A, rk, rv, alpha, i))
                m = min(topm, len(items))
                res["keys"][t, :m], res["contrib"][t, :m] = items[:m], c[:m]
                res["ranked"][t] = (items, c)
        out.append(res)
    return out

"""fp64 NumPy restatement of the offline evaluation metrics (DESIGN.md 4.14): per row, from a ranked list and its
held-out items, hit, recall, precision, ndcg, ap, reciprocal rank and intra-list diversity at a cutoff, and the
coverage of a set of lists, written from the definitions one row at a time."""
import numpy as np
import scipy.sparse


def truth_rows(test):
    """Per row of a scipy sparse matrix: its distinct columns whose value, after duplicates are summed, is nonzero."""
    m = scipy.sparse.csr_matrix(test, dtype=np.float64, copy=True)
    m.sum_duplicates()
    return [np.sort(m.indices[m.indptr[r]:m.indptr[r + 1]][m.data[m.indptr[r]:m.indptr[r + 1]] != 0])
            for r in range(m.shape[0])]


def row_metrics(entries, truth, K, Q=None):
    """(hit, recall, precision, ndcg, ap, rr, ild or None) of the first K entries of one list (-1 pads; entries past
    the list count as padding) against the non-empty truth row."""
    e = np.full(K, -1, dtype=np.int64)
    e[:min(K, len(entries))] = np.asarray(entries[:K], dtype=np.int64)
    T = set(int(x) for x in truth)
    h = np.array([1.0 if x != -1 and int(x) in T else 0.0 for x in e])
    c = np.cumsum(h)
    gains = 1.0 / np.log2(np.arange(2, K + 2))
    m = min(len(T), K)
    ndcg = float((h * gains).sum() / np.cumsum(gains)[m - 1])
    ap = float((h * c / np.arange(1, K + 1)).sum() / m)
    hits = np.flatnonzero(h)
    rr = 1.0 / (hits[0] + 1) if len(hits) else 0.0
    ild = None
    if Q is not None:
        valid = e[e != -1]
        if len(valid) >= 2:
            X = np.asarray(Q, dtype=np.float64)[valid]
            norm = np.linalg.norm(X, axis=1)
            X = X / np.where(norm > 0, norm, 1.0)[:, None]     # a zero row stays zero: cos 0 with every row
            a, b = np.triu_indices(len(valid), 1)
            ild = float(np.mean(1.0 - (X[a] * X[b]).sum(1)))
    return float(c[-1] > 0), float(c[-1] / len(T)), float(c[-1] / K), ndcg, ap, float(rr), ild


def evaluate(ranked, test, cutoffs, Q=None):
    """evaluate_lists' result (with "rows" and "per_user") for the same arguments, from row_metrics."""
    truth = truth_rows(test)
    rows = np.array([r for r, t in enumerate(truth) if len(t)], dtype=np.int64)
    num_items = test.shape[1]
    res = {"users": len(rows), "rows": rows.astype(np.int32), "per_user": {}}
    names = ("hit", "recall", "precision", "ndcg", "map", "mrr")
    for K in sorted(set(int(k) for k in cutoffs)):
        vals = [row_metrics(ranked[r], truth[r], K, Q) for r in rows]
        for j, name in enumerate(names):
            col = np.array([v[j] for v in vals], dtype=np.float64)
            res["per_user"]["%s@%d" % (name, K)] = col
            res["%s@%d" % (name, K)] = float(col.mean()) if len(col) else float("nan")
        seen = set(int(x) for r in rows for x in ranked[r][:K] if x != -1)
        res["coverage@%d" % K] = len(seen) / num_items
        if Q is not None:
            col = np.array([np.nan if v[6] is None else v[6] for v in vals], dtype=np.float64)
            res["per_user"]["ild@%d" % K] = col
            ok = ~np.isnan(col)
            res["ild@%d" % K] = float(col[ok].mean()) if ok.any() else float("nan")
    return res

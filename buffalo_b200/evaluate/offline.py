"""Offline evaluation on held-out interactions (csrc/offline_eval.cu, DESIGN.md 4.14): hit rate, recall, precision,
NDCG, MAP and MRR at several cutoffs, catalogue coverage and intra-list diversity, for a trained model
(Evaluable.evaluate: the masked top-k of the validation path, then the metrics) or for ranked lists made elsewhere
(evaluate_lists).  Both go through one metric pass: per batch of rows the cutoff terms, the diversity terms and the
coverage marks on the device, then the fixed-order sums of bfl_eval_sum_device.  Per-row values depend on the row alone,
so neither they nor the means change with the batch split."""
import numpy as np
import scipy.sparse

from buffalo_b200 import backend
from buffalo_b200.evaluate.device import MEM_FRACTION, SortedRows, _StageTimer, to_device

MAX_CUTOFF = 4096
MEAN_METRICS = ("hit", "recall", "precision", "ndcg", "map", "mrr")   # columns 0-5 of a cutoff's slab
BATCH_ROWS = None   # at most this many rows per batch when set (the batch split never changes a result)


def check_cutoffs(cutoffs, diversity):
    """The cutoffs ascending and distinct (int32); ValueError unless they are integers in [1, 4096], and with
    diversity at most 256."""
    if isinstance(cutoffs, (int, np.integer)) and not isinstance(cutoffs, bool):
        cutoffs = (cutoffs,)
    try:
        values = list(cutoffs)
    except TypeError:
        raise ValueError("cutoffs must be a sequence of integers, got %r" % (cutoffs,))
    if not values or any(isinstance(c, bool) or not isinstance(c, (int, np.integer)) or not 1 <= c <= MAX_CUTOFF
                         for c in values):
        raise ValueError("cutoffs must be integers in [1, %d], got %r" % (MAX_CUTOFF, cutoffs))
    if diversity and max(values) > backend.EVAL_ILD_KMAX:
        raise ValueError("diversity needs every cutoff <= %d, got %d" % (backend.EVAL_ILD_KMAX, max(values)))
    return np.unique(np.asarray(values, dtype=np.int32))


def truth_csr(test, num_rows, num_items):
    """(END offsets int64, keys int32, evaluated rows int64) of a scipy sparse (num_rows, num_items) held-out matrix:
    row r's ground truth is its distinct columns whose value, after duplicates are summed, is nonzero (ascending);
    the evaluated rows are those with at least one such column."""
    if not scipy.sparse.issparse(test):
        raise ValueError("test must be a scipy sparse (%d, %d) matrix, got %s" % (num_rows, num_items,
                                                                                  type(test).__name__))
    if test.shape != (num_rows, num_items):
        raise ValueError("test must be a (%d, %d) matrix, got %s" % (num_rows, num_items, test.shape))
    m = scipy.sparse.csr_matrix(test, dtype=np.float64, copy=True)
    m.sum_duplicates()
    m.eliminate_zeros()
    keys = np.asarray(m.indices[:int(m.indptr[-1])])
    if keys.size and (int(keys.min()) < 0 or int(keys.max()) >= num_items):
        raise ValueError("test holds a column outside [0, %d)" % num_items)
    return (np.asarray(m.indptr[1:], dtype=np.int64), np.ascontiguousarray(keys, dtype=np.int32),
            np.flatnonzero(np.diff(m.indptr) > 0))


def check_slab_memory(n_cut, n):
    """MemoryError, before any allocation, when the per-row terms of every evaluated row (one [n, 8] fp64 slab per
    cutoff, kept on the device for the whole call so that the sums run in one fixed order) do not fit in MEM_FRACTION
    of the free device memory."""
    need = 64 * int(n_cut) * int(n)
    free = backend.device_free_bytes()
    if need > MEM_FRACTION * free:
        raise MemoryError("the per-row terms of %d rows at %d cutoffs need %.2f GB of device memory, more than %.0f%% "
                          "of the %.2f GB free: evaluate fewer rows per call or fewer cutoffs"
                          % (n, n_cut, need / 1e9, 100 * MEM_FRACTION, free / 1e9))


def batch_rows(per_row, n):
    """Rows per batch: per_row device bytes each within MEM_FRACTION of the free device memory (and BATCH_ROWS)."""
    b = max(1, int(MEM_FRACTION * backend.device_free_bytes() // max(per_row, 1)))
    if BATCH_ROWS:
        b = min(b, int(BATCH_ROWS))
    return max(1, min(b, n))


class _MetricPass(object):
    """The metric pass over the n evaluated rows: `add` one batch of ranked lists at a time, then `result`."""

    def __init__(self, cuts, n, num_items, items, timer, dev):
        import torch
        self.cuts, self.n, self.num_items, self.items, self.timer = cuts, n, num_items, items, timer
        self.kmax = int(cuts[-1])
        gains = 1.0 / np.log2(np.arange(2, self.kmax + 2))
        self.d_cuts = to_device(cuts, np.int32, dev)
        self.gains, self.ideal = to_device(gains, np.float64, dev), to_device(np.cumsum(gains), np.float64, dev)
        # bucket[p]: the smallest cutoff index whose cutoff exceeds position p
        self.bucket = to_device(np.searchsorted(cuts, np.arange(1, self.kmax + 1)), np.int32, dev)
        self.first = torch.full((num_items,), len(cuts), dtype=torch.int32, device=dev)
        self.terms = torch.zeros((len(cuts), n, 8), dtype=torch.float64, device=dev)

    def add(self, s, ranked, truth):
        """ranked: int32 [nb, k] device lists of evaluated rows s .. s + nb; truth: (indptr, keys, row) of their rows."""
        view = self.terms[:, s:s + ranked.shape[0]]
        with self.timer("terms"):
            backend.eval_cutoff_terms(ranked, *truth, self.d_cuts, self.gains, self.ideal, view)
        if self.items is not None:
            with self.timer("ild"):
                backend.eval_ild(ranked, self.kmax, self.items, self.d_cuts, view)
        with self.timer("coverage"):
            backend.eval_coverage_mark(ranked, self.bucket, self.first)

    def result(self, rows, per_user):
        with self.timer("coverage"):
            covered = np.cumsum(backend.eval_coverage_count(self.first, len(self.cuts)))
        with self.timer("sum"):
            sums = [backend.eval_sum(self.terms[c]) for c in range(len(self.cuts))]
        self.timer.close()
        n = self.n
        res = {"users": n}
        for c, K in enumerate(self.cuts):
            for j, name in enumerate(MEAN_METRICS):
                res["%s@%d" % (name, K)] = float(sums[c][j] / n) if n else float("nan")
            res["coverage@%d" % K] = float(covered[c] / self.num_items)
            if self.items is not None:
                res["ild@%d" % K] = float(sums[c][6] / sums[c][7]) if sums[c][7] else float("nan")
        if per_user:
            T = self.terms.cpu().numpy()
            res["rows"] = np.asarray(rows, dtype=np.int32)
            res["per_user"] = {}
            for c, K in enumerate(self.cuts):
                for j, name in enumerate(MEAN_METRICS):
                    res["per_user"]["%s@%d" % (name, K)] = T[c, :, j].copy()
                if self.items is not None:
                    res["per_user"]["ild@%d" % K] = np.where(T[c, :, 7] > 0, T[c, :, 6], np.nan)
        return res


def _device():
    import torch
    return torch.device("cuda", torch.cuda.current_device())


def evaluate_lists(ranked, test, cutoffs=(10,), item_factors=None, per_user=False, stages=None):
    """Ranking metrics of ranked lists made elsewhere against held-out items, on the GPU.

    ranked: an (n, K) integer array of item indexes, -1 for padding (what ParALS.topk_recommendation, with or without
    nprobe or a pool, and fold_in_recommendation return).  test: a scipy sparse (n, num_items) matrix aligned with
    ranked row for row; row r's ground truth is its distinct columns with a nonzero value after duplicates are summed,
    and only rows with at least one are evaluated.  cutoffs: integers in [1, min(K, 4096)].  item_factors: None, or a
    (num_items, d) array whose rows give intra-list diversity (every cutoff <= 256 then).

    Returns {"users": rows evaluated} and, per cutoff K, the means over those rows of hit@K, recall@K, precision@K,
    ndcg@K, map@K and mrr@K, coverage@K (distinct items in the first K entries of all evaluated lists over num_items)
    and, with item_factors, ild@K (mean 1 - cosine over the pairs of valid entries among the first K, over the rows with
    at least two).  per_user=True adds "rows" (int32 indexes of the evaluated rows) and "per_user", a dict of float64
    arrays per evaluated row under the same names (ild NaN where a row has fewer than two valid entries).  stages:
    optional dict receiving device milliseconds per stage.  GPU only: without one the backend's "no CPU fallback"
    error is raised after the argument checks.  The per-row terms (64 bytes per row and cutoff) stay on the device for
    the whole call; MemoryError before any allocation when they do not fit in half the free device memory."""
    ranked = np.asarray(ranked)
    if ranked.ndim != 2 or not np.issubdtype(ranked.dtype, np.integer) or ranked.shape[1] < 1:
        raise ValueError("ranked must be an (n, K) integer array with K >= 1, got %s %s" % (ranked.dtype, ranked.shape))
    if not scipy.sparse.issparse(test) or test.ndim != 2:
        raise ValueError("test must be a scipy sparse (n, num_items) matrix, got %s" % type(test).__name__)
    n_all, num_items = ranked.shape[0], test.shape[1]
    cuts = check_cutoffs(cutoffs, item_factors is not None)
    if cuts[-1] > ranked.shape[1]:
        raise ValueError("cutoffs must not exceed the lists' width %d, got %d" % (ranked.shape[1], cuts[-1]))
    if ranked.size and (int(ranked.min()) < -1 or int(ranked.max()) >= num_items):
        raise ValueError("ranked holds an index outside [-1, %d)" % num_items)
    if item_factors is not None:
        item_factors = np.asarray(item_factors)
        if item_factors.ndim != 2 or item_factors.shape[0] != num_items or item_factors.shape[1] < 1:
            raise ValueError("item_factors must be a (%d, d) array, got %s" % (num_items, item_factors.shape))
    t_ptr, t_keys, rows = truth_csr(test, n_all, num_items)
    backend.require_device()
    check_slab_memory(len(cuts), len(rows))
    dev = _device()
    timer = _StageTimer(stages)
    items = None if item_factors is None else to_device(item_factors, np.float32, dev)
    lists = np.ascontiguousarray(ranked[rows][:, :cuts[-1]], dtype=np.int32)
    truth = SortedRows(t_ptr, t_keys, rows, dev, num_items)
    mp = _MetricPass(cuts, len(rows), num_items, items, timer, dev)
    per_row = lists.shape[1] * 4 + (0 if truth.resident else 4 * truth.mean_len() + 12)
    b = batch_rows(per_row, len(rows))
    for s in range(0, len(rows), b):
        with timer("upload"):
            d_lists = to_device(lists[s:s + b], np.int32, dev)
            t = truth.rows_for(np.arange(s, min(s + b, len(rows))))
        mp.add(s, d_lists, t)
    return mp.result(rows, per_user)


def evaluate_model(model, test, cutoffs=(10,), exclude_seen=True, diversity=False, per_user=False, stages=None):
    """Evaluable.evaluate: each evaluated user's list of the largest cutoff from the masked top-k of the validation
    path (bfl_eval_topk_masked_device, the model's item bias included where its ranking adds one), then the metric
    pass of evaluate_lists.  stages: optional dict receiving device milliseconds per stage."""
    hook = getattr(model, "_device_eval_model", None)
    if hook is None:
        raise NotImplementedError("evaluate needs a model with device ranking (ALS, BPRMF, WARP, PLSI), not %s"
                                  % type(model).__name__)
    em = hook()
    if em.l2:
        raise ValueError("evaluate has no device ranking for score_func='l2'; use a dot-product model")
    cuts = check_cutoffs(cutoffs, diversity)
    P, Q = em.P, em.Q
    num_users, num_items = P.shape[0], Q.shape[0]
    t_ptr, t_keys, rows = truth_csr(test, num_users, num_items)
    if scipy.sparse.issparse(exclude_seen) or exclude_seen:
        from buffalo_b200.parallel.base import seen_csr
        s_ptr, s_keys = seen_csr(model, exclude_seen)
    else:
        s_ptr, s_keys = np.zeros(num_users, np.int64), np.zeros(0, np.int32)
    backend.require_device()
    check_slab_memory(len(cuts), len(rows))
    dev = _device()
    timer = _StageTimer(stages)
    with timer("upload"):
        d_Q = to_device(Q, np.float32, dev)
        bias = None if em.rank_bias is None else to_device(np.asarray(em.rank_bias).reshape(-1), np.float32, dev)
        truth = SortedRows(t_ptr, t_keys, rows, dev, num_items)
        seen = SortedRows(s_ptr, s_keys, rows, dev, num_items)
    mp = _MetricPass(cuts, len(rows), num_items, d_Q if diversity else None, timer, dev)
    k = mp.kmax
    nslices = -(-num_items // 4096)
    per_row = nslices * (k * 8 + 4) + k * 4 + d_Q.shape[1] * 4 + 48
    for st in (truth, seen):
        per_row += 0 if st.resident else 4 * st.mean_len() + 12
    b = batch_rows(per_row, len(rows))
    for s in range(0, len(rows), b):
        local = np.arange(s, min(s + b, len(rows)))
        with timer("upload"):
            queries = to_device(np.asarray(P)[rows[local]], np.float32, dev)
            t, sn = truth.rows_for(local), seen.rows_for(local)
        with timer("topk"):
            ranked = backend.eval_topk_masked(queries, d_Q, bias, k, *sn)
        mp.add(s, ranked, t)
    return mp.result(rows, per_user)

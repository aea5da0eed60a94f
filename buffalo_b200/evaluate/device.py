"""Validation metrics on the device (csrc/evaluate.cu, DESIGN.md 4.8): the same values as Evaluable's host loop, from
the held-out triples and the training rows of the validation users, without the per-user Python sets.

State built once per Data (`ValidationState`): the held-out CSR by user, the triples with their rows renumbered over
the validation users, and the validation users' training rows as sorted copies, on the device when they fit in half
the free device memory.  Each evaluation uploads Q, the item bias and the validation users' rows of P once."""
import collections

import numpy as np

from buffalo_b200 import backend

# What a trainer hands the device path (Evaluable._device_eval_model): the factor arrays as its host path reads them,
# the item bias its ranking adds (or None), the one its _get_scores adds (or None), and whether scores are 1 - |p - q|^2
# (then ranking stays on the host and only the score metrics run here).
EvalModel = collections.namedtuple("EvalModel", "P Q rank_bias score_bias l2")

MEM_FRACTION = 0.5   # share of the free device memory the user batches and the resident seen rows may take


def _nonempty(keys):
    # a device pointer must exist even when every row is empty
    return keys if len(keys) else np.zeros(1, dtype=np.int32)


def _gather_positions(indptr, rows):
    """(END offsets int64, entry positions int64) of the CSR rows `rows` (in that order) of a host CSR of END offsets:
    row i of the gathered CSR is entries pos[out_ptr[i - 1]:out_ptr[i]] of the source."""
    rows = np.asarray(rows, dtype=np.int64)
    ends = indptr[rows]
    begs = np.where(rows > 0, indptr[np.maximum(rows - 1, 0)], 0)
    lens = ends - begs
    out_ptr = np.cumsum(lens).astype(np.int64)
    pos = np.arange(int(out_ptr[-1]) if len(out_ptr) else 0, dtype=np.int64)
    pos += np.repeat(begs - (out_ptr - lens), lens)
    return out_ptr, pos


def _gather_rows(indptr, keys, rows):
    """(END offsets int64, keys int32) of the CSR rows `rows` (in that order) of a host CSR of END offsets."""
    out_ptr, pos = _gather_positions(indptr, rows)
    return out_ptr, np.ascontiguousarray(keys[pos], dtype=np.int32)


def to_device(a, dtype, dev):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).to(dev)


class SortedRows(object):
    """Rows `rows` (in that order) of a host CSR of END offsets, handed to device calls that need every row in ascending
    order: the validation users' training rows here, the truth and exclusion rows of evaluate/offline.py.  With
    resident=True the rows stay on the device when they fit in MEM_FRACTION of the free device memory; otherwise each
    batch gathers, uploads and sorts its own."""

    def __init__(self, indptr, keys, rows, dev, num_items, resident=True):
        self.dev, self.num_items = dev, num_items
        nnz = int(indptr[-1]) if len(indptr) else 0
        self.indptr, self.keys = _gather_rows(np.asarray(indptr, dtype=np.int64), np.asarray(keys[:nnz]), rows)
        nbytes = self.keys.nbytes + self.indptr.nbytes
        self.resident = resident and nbytes < MEM_FRACTION * backend.device_free_bytes()
        if self.resident:
            self.d_rows = self._sorted(to_device(self.indptr, np.int64, dev), to_device(_nonempty(self.keys), np.int32, dev))

    def mean_len(self):
        return int(np.ceil(len(self.keys) / max(len(self.indptr), 1)))

    def _sorted(self, indptr, keys):
        """The CSR with every row sorted: unchanged when the device check finds all rows sorted (the rows of a
        "matrix" database), else rebuilt by the device radix sort (a "stream" database keeps session order)."""
        import torch
        if backend.eval_unsorted_rows(indptr, keys) == 0:
            return indptr, keys
        lens = torch.diff(indptr, prepend=indptr.new_zeros(1))
        major = torch.repeat_interleave(torch.arange(indptr.shape[0], dtype=torch.int32, device=self.dev), lens)
        ones = torch.ones(keys.shape[0], dtype=torch.float32, device=self.dev)
        sorted_indptr, sorted_keys, _ = backend.csr_from_triples_device(major, keys, ones, indptr.shape[0],
                                                                        self.num_items)
        return sorted_indptr, sorted_keys

    def rows_for(self, local):
        """(indptr, keys, row) device tensors: query q of a batch reads CSR row row[q], which holds rows[local[q]]."""
        if self.resident:
            return self.d_rows + (to_device(local, np.int32, self.dev),)
        ptr, keys = _gather_rows(self.indptr, self.keys, local)
        indptr, keys = self._sorted(to_device(ptr, np.int64, self.dev), to_device(_nonempty(keys), np.int32, self.dev))
        return indptr, keys, to_device(np.arange(len(local)), np.int32, self.dev)


class ValidationState(object):
    def __init__(self, data, dev, max_users=None):
        import torch
        self.dev = dev
        h = data.get_header()
        self.num_users, self.num_items = int(h["num_users"]), int(h["num_items"])
        v = data.get_group("vali")
        row, col, val = (np.asarray(v[k][:]) for k in ("row", "col", "val"))
        self.vali_rows = np.unique(row)
        self.n_triples = len(row)
        t = self._to_dev
        self.cols, self.vals = t(col, np.int32), t(val, np.float32)
        self.rows_local = t(np.searchsorted(self.vali_rows, row), np.int32)
        self.gt_indptr, self.gt_keys, _ = backend.csr_from_triples_device(t(row, np.int32), self.cols, self.vals,
                                                                          self.num_users, self.num_items)
        grp = data.get_group("rowwise")
        self.max_users = max_users
        # every validation user's training row on the device for the life of the Data, when it fits
        self.seen = SortedRows(grp["indptr"][:], grp["key"], self.vali_rows, dev, self.num_items,
                               resident=max_users is None)
        self.seen_indptr, self.seen_keys, self.resident = self.seen.indptr, self.seen.keys, self.seen.resident
        torch.cuda.current_stream(dev).synchronize()

    def _to_dev(self, a, dtype):
        return to_device(a, dtype, self.dev)

    def seen_for(self, local):
        """(seen_indptr, seen_keys, seen_row) device tensors covering the validation users vali_rows[local]."""
        return self.seen.rows_for(local)


def state_of(data, dev, max_users=None):
    st = getattr(data, "_b200_validation_state", None)
    if st is None or st.max_users != max_users or st.dev != dev:
        st = ValidationState(data, dev, max_users)
        data._b200_validation_state = st
    return st


def _zero_division(what):
    raise ZeroDivisionError("float division by zero (%s)" % what)


class Evaluation(object):
    """One evaluation of one model: the factors uploaded once, then the ranking and score metrics."""

    def __init__(self, data, model, max_users=None):
        import torch
        self.dev = torch.device("cuda", torch.cuda.current_device())
        self.st = state_of(data, self.dev, max_users)
        t = self.st._to_dev
        self.model = model
        self.Q = t(model.Q, np.float32)
        self.P = t(np.asarray(model.P)[self.st.vali_rows], np.float32)   # rows of the validation users only
        self.rank_bias = None if model.rank_bias is None else t(np.asarray(model.rank_bias).reshape(-1), np.float32)
        self.score_bias = None if model.score_bias is None else t(np.asarray(model.score_bias).reshape(-1), np.float32)

    def batch_users(self, topk, queued):
        """Users per batch of the masked top-k: its candidate lists, output and query rows (and the batch's seen rows
        when they are not resident) within MEM_FRACTION of the free device memory."""
        nslices = -(-self.st.num_items // 4096)
        per_user = nslices * (topk * 8 + 4) + topk * 4 + self.P.shape[1] * 4 + 48
        if not self.st.resident:
            per_user += 4 * max(1, int(np.ceil(len(self.st.seen_keys) / max(len(self.st.vali_rows), 1)))) + 8
        b = max(1, int(MEM_FRACTION * backend.device_free_bytes() // per_user))
        if self.st.max_users:
            b = min(b, int(self.st.max_users))
        return min(b, queued)

    def ranking(self, topk, eval_samples, stages=None):
        """NDCG, MAP, accuracy and AUC of the validation users (an eval_samples draw of them, from np.random like the
        host path) against their held-out items.  stages: optional dict receiving device milliseconds per stage."""
        import torch
        st = self.st
        rows = st.vali_rows
        if eval_samples:
            rows = np.random.choice(rows, size=min(eval_samples, len(rows)), replace=False)
        local = np.searchsorted(st.vali_rows, rows)
        gains = 1.0 / np.log2(np.arange(2, topk + 2))
        d_gains, d_ideal = st._to_dev(gains, np.float64), st._to_dev(np.cumsum(gains), np.float64)
        terms = torch.empty((len(rows), 6), dtype=torch.float64, device=self.dev)
        timer = _StageTimer(stages)
        b = self.batch_users(topk, max(len(rows), 1))
        for s in range(0, len(rows), b):
            lb = local[s:s + b]
            with timer("seen"):
                seen_indptr, seen_keys, seen_row = st.seen_for(lb)
                users = st._to_dev(rows[s:s + b], np.int32)
                queries = self.P[st._to_dev(lb, np.int64)]
            with timer("topk"):
                ranked = backend.eval_topk_masked(queries, self.Q, self.rank_bias, topk, seen_indptr, seen_keys,
                                                  seen_row)
            with timer("terms"):
                backend.eval_ranking_terms(ranked, users, seen_indptr, seen_row, st.gt_indptr, st.gt_keys, d_gains,
                                           d_ideal, st.num_items, terms[s:s + b])
        with timer("sum"):
            tot = backend.eval_sum(terms)
        timer.close()
        if tot[5] > 0:
            _zero_division("a validation user holds out every item")
        if tot[4] == 0:
            _zero_division("no validation user has training items")
        return {"ndcg": float(tot[0] / tot[4]), "map": float(tot[1] / tot[4]), "accuracy": float(tot[2] / tot[4]),
                "auc": float(tot[3] / tot[4])}

    def scores(self, stages=None):
        """RMSE and mean absolute error of the model's scores over every held-out triple."""
        st = self.st
        timer = _StageTimer(stages)
        with timer("scores"):
            mode = "l2" if self.model.l2 else ("dot_bias" if self.score_bias is not None else "dot")
            terms = backend.eval_score_terms(self.P, self.Q, self.score_bias, mode, st.rows_local, st.cols, st.vals)
            tot = backend.eval_sum(terms)
        timer.close()
        n = st.n_triples
        if n == 0:
            return {"rmse": float("nan"), "error": float("nan")}
        return {"rmse": float(np.sqrt(tot[0] / n)), "error": float(tot[1] / n)}


class _StageTimer(object):
    """Device milliseconds per named stage (CUDA events), summed over batches; a no-op when stages is None."""

    def __init__(self, stages):
        self.stages, self.marks = stages, []

    def __call__(self, name):
        timer = self

        class _Span(object):
            def __enter__(self):
                if timer.stages is not None:
                    import torch
                    self.a = torch.cuda.Event(enable_timing=True)
                    self.a.record()

            def __exit__(self, *exc):
                if timer.stages is not None:
                    import torch
                    b = torch.cuda.Event(enable_timing=True)
                    b.record()
                    timer.marks.append((name, self.a, b))
        return _Span()

    def close(self):
        if self.stages is None:
            return
        import torch
        torch.cuda.synchronize()
        for name, a, b in self.marks:
            self.stages[name] = self.stages.get(name, 0.0) + a.elapsed_time(b)
        self.marks = []

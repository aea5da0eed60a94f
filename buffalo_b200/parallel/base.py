"""Batch query helpers (buffalo/parallel/base.py): ParALS / ParBPRMF, the dot_topn semantics of
buffalo/parallel/_core.hpp:88-142 (best-first indexes, -1 padded).  With a GPU the queries run on a backend.Serve
handle that keeps the item factors resident (DESIGN.md 4.9); without one, or above its limits, the NumPy
implementation below runs."""
import numpy as np

from buffalo_b200 import backend


def quickselect(scores, result, sorted=True, num_threads=4):
    k = result.shape[1]
    part = np.argpartition(-scores, min(k, scores.shape[1]) - 1, axis=1)[:, :k]
    if sorted:
        vals = np.take_along_axis(scores, part, axis=1)
        part = np.take_along_axis(part, np.argsort(-vals, axis=1, kind="stable"), axis=1)
    result[:, :part.shape[1]] = part


def dot_topn(indexes, P, Q, Qb, out_keys, out_scores, pool, topk, num_workers=4):
    cand = Q if pool is None or len(pool) == 0 else Q[pool]
    scores = P[indexes].dot(cand.T)
    if Qb is not None and Qb.size:
        scores = scores + (Qb if pool is None or len(pool) == 0 else Qb[pool]).reshape(1, -1)
    k = min(topk, scores.shape[1])
    part = np.argpartition(-scores, k - 1, axis=1)[:, :k]
    vals = np.take_along_axis(scores, part, axis=1)
    order = np.argsort(-vals, axis=1, kind="stable")
    part, vals = np.take_along_axis(part, order, axis=1), np.take_along_axis(vals, order, axis=1)
    out_keys[:] = -1
    out_scores[:] = 0
    out_keys[:, :k] = part if pool is None or len(pool) == 0 else np.asarray(pool)[part]
    out_scores[:, :k] = vals


class Parallel(object):
    def __init__(self, algo, *argv, **kwargs):
        self.algo = algo
        self.num_workers = int(kwargs.get("num_workers", algo.opt.num_workers))

    @staticmethod
    def _fingerprint(*arrays):
        """Checksum of the arrays' bits, one pass over the data: the xor of all 32-bit words and the sum of the row
        sums weighted by odd row numbers (so a changed value, and rows that changed places, both show)."""
        out = []
        for x in arrays:
            if x is None:
                out.append(None)
                continue
            w = x.view(np.uint32).reshape(x.shape[0], -1)
            rows = w.sum(axis=1, dtype=np.uint64)
            out.append((x.shape, int(np.bitwise_xor.reduce(w, axis=None)),
                        int((rows * (np.arange(len(rows), dtype=np.uint64) * np.uint64(2) + np.uint64(1))).sum(dtype=np.uint64))))
        return tuple(out)

    def _serve_handle(self, B, Bb):
        """The handle holding items B (and bias Bb) on the device.  The factor arrays are the model's live arrays and
        training, normalize() or the user may rewrite them, in place or not, between two calls; so every call
        checksums them and uploads again when they differ from what is resident."""
        key = self._fingerprint(B, Bb)
        if getattr(self, "_serve_key", None) != key:
            if getattr(self, "_serve", None) is None:
                self._serve = backend.Serve()
            self._serve_key = None
            self._serve.set_items(B, Bb)
            self._serve_key = key
        return self._serve

    def _run(self, indexes, A, B, Bb, topk, pool):
        if Bb is not None and not Bb.size:
            Bb = None
        # On the device when one is present and the call is within the kernels' limits.  The items must fit in device
        # memory next to the gathered query rows: an allocation failure is an error, not a silent switch to NumPy.
        on_device = (backend.device_available() and len(indexes) and 0 < topk <= backend.SERVE_KMAX
                     and B.shape[0] < 2 ** 31
                     and all(x.dtype == np.float32 and x.flags["C_CONTIGUOUS"] for x in (A, B)))
        if on_device:
            h = self._serve_handle(B, None if Bb is None else np.ascontiguousarray(Bb, dtype=np.float32))
            # only the rows asked for go to the device, read from the live array at every call
            h.set_queries(np.ascontiguousarray(A[indexes]))
            h.set_pool(None if pool is None or len(pool) == 0 else pool)
            return h.topk(np.arange(len(indexes), dtype=np.int32), topk)
        keys = np.zeros((len(indexes), topk), dtype=np.int32)
        scores = np.zeros((len(indexes), topk), dtype=np.float32)
        dot_topn(indexes, A, B, Bb, keys, scores, pool, topk, self.num_workers)
        return keys, scores


class ParALS(Parallel):
    _bias = False

    def _resolve(self, keys, pool, group):
        idx = self.algo.get_index_pool(keys, group=group) if isinstance(keys, list) else keys
        kept = [k for k, i in zip(keys, idx) if i is not None]
        idx = np.array([i for i in idx if i is not None], dtype=np.int32)
        if pool is not None:
            pool = self.algo.get_index_pool(pool, group="item" if group == "user" else group)
            if len(pool) == 0:
                raise RuntimeError("pool is empty")
        return kept, idx, pool

    def most_similar(self, keys, topk=10, group="item", pool=None, repr=False, ef_search=-1, use_mmap=True):
        self.algo.normalize(group=group)
        _, idx, pool = self._resolve(keys, pool, group)
        if group not in ("item", "user"):
            raise ValueError(f"Not supported group: {group}")
        F = self.algo.Q if group == "item" else self.algo.P
        names = self.algo._idmanager.itemids if group == "item" else self.algo._idmanager.userids
        topks, scores = self._run(idx, F, F, None, topk, pool)
        if repr:
            topks = [[names[t] for t in tt if t != -1] for tt in topks]
        return topks, scores

    def topk_recommendation(self, keys, topk=10, pool=None, repr=False):
        if self.algo.opt._nrz_P or self.algo.opt._nrz_Q:
            raise RuntimeError("Cannot make topk recommendation with normalized factors")
        kept, idx, pool = self._resolve(keys, pool, "user")
        Qb = self.algo.Qb if self._bias and self.algo.opt.get("use_bias") else None
        topks, scores = self._run(idx, self.algo.P, self.algo.Q, Qb, topk, pool)
        if repr:
            topks = [[self.algo._idmanager.itemids[t] for t in tt if t != -1] for tt in topks]
        return kept, topks, scores


class ParBPRMF(ParALS):
    _bias = True


def _unsupported(name):
    def ctor(*a, **k):
        raise NotImplementedError(name + " is outside the H100 hot-path scope")
    return ctor


ParW2V = _unsupported("ParW2V")
ParCFR = _unsupported("ParCFR")

"""Batch query helpers (buffalo/parallel/base.py): ParALS / ParBPRMF.  Serving-side brute-force MIPS is outside
the training hot path (SURVEY.md 2.1 #10); this is a NumPy implementation of the same interface
(dot_topn semantics of buffalo/parallel/_core.hpp:88-142: best-first indexes, -1 padded)."""
import numpy as np


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

    def _run(self, indexes, A, B, Bb, topk, pool):
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

"""WARP trainer (buffalo/algo/warp.py) on the H100 backend.  The reference has no GPU WARP
(warp.py:30-32 raises NotImplementedError for accelerator=True); here the GPU path is the only path."""
import numpy as np

from buffalo_b200.algo.bpr import BPRMF
from buffalo_b200.algo.options import _WARP, WARPOption
from buffalo_b200.evaluate.device import EvalModel


class WARP(BPRMF):
    """drop-in for buffalo.algo.warp.WARP; shares the BPRMF driver, WARP's option table and backend kind."""
    _KIND, _NAME, _OPT = "warp", "WARP", WARPOption
    _specific = _WARP          # option defaults/validation resolve to WARPOption's table

    def __init__(self, opt_path=None, *args, **kwargs):
        super().__init__(opt_path, *args, **kwargs)
        if isinstance(self.opt.score_func, str):
            self.opt.score_func = self.opt.score_func.lower()

    @staticmethod
    def new(path, data_fields=[]):
        return WARP.instantiate(WARPOption, path, data_fields)

    def _draw(self, rows, cols, rng=np.random):
        return rng.normal(scale=1.0 / (self.opt.d ** 2), size=(rows, cols)).astype("float32")   # warp.py:83-88 (signed)

    def prepare_sampling(self):
        pass  # warp.py:72-77: uniform negatives only

    def normalize(self, group="item"):
        if self.opt["score_func"] == "l2":
            self.logger.warning("Normalization will harm performance if score func is L2")
        super().normalize(group)

    def _l2(self):
        return self.opt.score_func == "l2"

    def _get_topk_recommendation(self, rows, topk, pool=None):
        if not self._l2():
            topks = super(BPRMF, self)._get_topk_recommendation(self.P[rows], self.Q, pb=None, Qb=None, pool=pool,
                                                                topk=topk, num_workers=self.opt.num_workers)
            return zip(rows, topks)
        p = self.P[rows]
        Q = self.Q if pool is None else self.Q[pool]
        scores = -((p ** 2).sum(1)[:, None] - 2 * p.dot(Q.T) + (Q ** 2).sum(1)[None, :])
        topks = self.get_topk(scores, topk, num_threads=self.opt.num_workers)
        if pool is not None:
            topks = np.array([pool[t] for t in topks])
        return zip(rows, topks)

    def _get_most_similar_item(self, col, topk, pool):
        if not self._l2():
            return super()._get_most_similar_item(col, topk, pool)
        if isinstance(col, np.ndarray):
            if col.ndim != 1:
                raise ValueError("query vector must be a 1d numpy array")
            q = col
        else:
            topk += 1
            q = self.Q[col]
        cand = self.Q if pool is None else self.Q[pool]
        scores = -((cand - q) ** 2).sum(-1)
        topks = self.get_topk(scores, topk, num_threads=self.opt.num_workers)
        out = -scores[topks]
        return (topks if pool is None else pool[topks]), out

    def get_scores(self, row_col_pairs):
        if self._l2():
            return {(r, c): -((self.P[r] - self.Q[c]) ** 2).sum() for r, c in row_col_pairs}
        return {(r, c): self.P[r].dot(self.Q[c]) for r, c in row_col_pairs}

    def _device_eval_model(self):
        return EvalModel(self.P, self.Q, None, None, self._l2())

    def _get_scores(self, row, col):
        if self._l2():
            return 1.0 - ((self.P[row] - self.Q[col]) ** 2).sum(-1)
        return (self.P[row] * self.Q[col]).sum(axis=1)

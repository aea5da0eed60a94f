"""BPRMF trainer (buffalo/algo/bpr.py) on the H100 backend."""

import numpy as np

from buffalo_b200.algo.base import Algo, Serializable
from buffalo_b200.algo.options import BPRMFOption
from buffalo_b200.algo.sgd_common import SGDTrainerMixin
from buffalo_b200.backend import CuSGD
from buffalo_b200.data.base import Data
from buffalo_b200.evaluate import Evaluable
from buffalo_b200.evaluate.device import EvalModel

inited_CUBPR = True


class BPRMF(SGDTrainerMixin, Algo, BPRMFOption, Evaluable, Serializable):
    """Bayesian Personalized Ranking MF -- drop-in for buffalo.algo.bpr.BPRMF."""
    _KIND, _NAME, _OPT = "bpr", "BPRMF", BPRMFOption

    def __init__(self, opt_path=None, *args, **kwargs):
        Algo.__init__(self, *args, **kwargs)
        self._OPT.__init__(self, *args, **kwargs)
        Evaluable.__init__(self, *args, **kwargs)
        Serializable.__init__(self, *args, **kwargs)
        self._init_trainer(self._NAME, self._OPT, lambda: CuSGD(self._KIND), opt_path,
                           lambda path, err: "cannot parse option file: %s (%s)" % (path, err), kwargs)

    @staticmethod
    def new(path, data_fields=[]):
        return BPRMF.instantiate(BPRMFOption, path, data_fields)

    def set_data(self, data):
        assert isinstance(data, Data), "Wrong instance: {}".format(type(data))
        self.data = data

    def normalize(self, group="item"):
        if group == "item" and not self.opt._nrz_Q:
            self.Q = self._normalize(self.Q)
            self.opt._nrz_Q = True
        elif group == "user" and not self.opt._nrz_P:
            self.P = self._normalize(self.P)
            self.opt._nrz_P = True

    def initialize(self):
        super().initialize()
        assert self.data, "Data is not set"
        self._init_buffer()
        self.init_factors()
        self.prepare_sampling()

    def _draw(self, rows, cols):
        return np.abs(np.random.normal(scale=1.0 / (self.opt.d ** 2), size=(rows, cols)).astype("float32"))   # bpr.py:88-93

    def init_factors(self):
        h = self.data.get_header()
        self.num_nnz = h["num_nnz"]
        self.P = self._pad(self._draw(h["num_users"], self.opt.d))
        self.Q = self._pad(self._draw(h["num_items"], self.opt.d))
        self.Qb = np.ascontiguousarray(self._draw(h["num_items"], 1))
        if not self.opt.get("use_bias"):
            self.Qb *= 0
        self.obj.initialize_model(self.P, self.Q, self.Qb, self.num_nnz)

    def prepare_sampling(self):
        """Cumulative popularity table (bpr.py:99-111), vectorised; `**= int(power)` is the reference's own
        truncation of fractional powers (0.75 -> 0 -> uniform weights)."""
        self.logger.info("Preparing sampling ...")
        n_items = self.data.get_header()["num_items"]
        table = np.zeros(n_items, dtype=np.int64)
        if self.opt.sampling_power > 0.0:
            grp = self.data.get_group("rowwise")
            nnz = int(grp["indptr"][-1]) if len(grp["indptr"]) else 0
            from buffalo_b200 import backend
            if backend.device_available():   # histogram + integer power + scan on the device (csrc/ingest.cu)
                table = backend.popularity_table_host(grp["key"][:nnz], n_items, int(self.opt.sampling_power))
            else:
                table = np.bincount(grp["key"][:nnz], minlength=n_items).astype(np.int64)
                table **= int(self.opt.sampling_power)
                table = np.cumsum(table).astype(np.int64)
        self.sampling_table_ = table
        self.obj.set_cumulative_table(self.sampling_table_, n_items)

    def _get_topk_recommendation(self, rows, topk, pool=None):
        Qb = self.Qb if self.opt.get("use_bias") else None
        topks = super()._get_topk_recommendation(self.P[rows], self.Q, pb=None, Qb=Qb, pool=pool, topk=topk,
                                                 num_workers=self.opt.num_workers)
        return zip(rows, topks)

    def _get_most_similar_item(self, col, topk, pool):
        return super()._get_most_similar_item(col, topk, self.Q, self.opt._nrz_Q, pool)

    def get_scores(self, row_col_pairs):
        return {(r, c): self.P[r].dot(self.Q[c]) + self.Qb[c][0] for r, c in row_col_pairs}

    def _get_scores(self, row, col):
        return (self.P[row] * self.Q[col]).sum(axis=1) + self.Qb[col][:, 0]

    def _get_feature(self, index, group="item"):
        return {"item": self.Q, "user": self.P}[group][index] if group in ("item", "user") else None

    def _device_eval_model(self):
        # ranking adds Qb only with use_bias (_get_topk_recommendation); _get_scores always adds it
        return EvalModel(self.P, self.Q, self.Qb if self.opt.get("use_bias") else None, self.Qb, False)

    def _get_data(self):
        return super()._get_data() + [("opt", self.opt), ("Q", self.Q), ("Qb", self.Qb), ("P", self.P)]

    def get_evaluation_metrics(self):
        return ["val_rmse", "val_ndcg", "val_map", "val_accuracy", "val_error", "train_loss"]

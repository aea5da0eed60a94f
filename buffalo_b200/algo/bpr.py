"""BPRMF trainer (buffalo/algo/bpr.py) on the H100 backend."""

import numpy as np

from buffalo_b200.algo import fold_in
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

    def _draw(self, rows, cols, rng=np.random):
        return np.abs(rng.normal(scale=1.0 / (self.opt.d ** 2), size=(rows, cols)).astype("float32"))   # bpr.py:88-93

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
        self.logger.info("Preparing sampling ...")
        self.sampling_table_ = self._popularity_table()
        self.obj.set_cumulative_table(self.sampling_table_, len(self.sampling_table_))

    def _popularity_table(self):
        """Cumulative popularity table (bpr.py:99-111), vectorised; `**= int(power)` is the reference's own
        truncation of fractional powers (0.75 -> 0 -> uniform weights)."""
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
        return table

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

    # ---- item fold-in (DESIGN.md 4.16) --------------------------------------------------------
    def fold_in_items(self, histories, init=None, epochs=None):
        """(rows float32 [n, d], bias float32 [n]) for n new items, with everything trained frozen: `epochs` (default
        num_iters) epochs of the item side of training restricted to the new rows.  Each history entry (u, x) is a
        positive, visited in CSR order; its negatives come from the trained catalogue through the model's own sampler
        (uniform or the popularity table, verify_neg against u's row of the attached training data; WARP's rank
        sampling with max_trials and threshold), and only the positive side's terms are applied, to x and its bias:
        plain-SGD BPR after every sample at training's linearly decayed rate, adagrad / adam one step per epoch from the
        epoch's gradient (WARP then projects x into the unit ball).  histories: a scipy sparse (n, num_users) matrix
        or a list of n lists of user ids (unknown ids dropped).  init: None (training's initial draw, seeded from
        random_seed) or an (n, d) array of start rows; the bias starts at 0 and stays 0 without use_bias.  P, Q, Qb and
        the training holder are not written; serve the rows with add_items(ids, rows, bias).  Needs the training data
        attached (set_data).  On the GPU only: without one the backend's "no CPU fallback" error is raised."""
        tX, tXb, _ = self._fold_in_items_device(histories, init, epochs)
        return tX[:, :self.opt.d].cpu().numpy(), tXb.cpu().numpy()

    def _fold_in_items_device(self, histories, init=None, epochs=None, trace=False):
        """fold_in_items' rows [n, vdim] and biases [n] as torch CUDA tensors, and with `trace` the draws (negatives
        [epochs, nnz * samples per positive], -1 for a WARP discard; WARP trial counts [epochs, nnz], 0 for a discard;
        None for BPR) as the kernel recorded them."""
        if self.opt._nrz_P or self.opt._nrz_Q:
            raise RuntimeError("Cannot fold in items with normalized factors")
        epochs = fold_in.positive_int(self.opt.num_iters if epochs is None else epochs, "epochs")
        if self.data is None:
            raise ValueError("fold_in_items needs the training data attached (set_data): negatives are checked "
                             "against each user's training row")
        header = self.data.get_header()
        num_items = header["num_items"]      # the trained catalogue: rows added by add_items are not negatives
        if header["num_users"] != self.P.shape[0] or num_items > self.Q.shape[0]:
            raise ValueError("the attached data (%d users, %d items) does not match the factors (%d, %d)"
                             % (header["num_users"], num_items, self.P.shape[0], self.Q.shape[0]))
        indptr, users, _ = fold_in.history_csr(self, histories, *fold_in.columns(self, "P"))
        n = len(indptr)
        per = 1 if self._KIND == "warp" else max(int(self.opt.num_negative_samples), 1)
        if n and int(np.diff(indptr, prepend=0).max()) * per >= 1 << 32:
            raise ValueError("a history row holds more than 2^32 samples per epoch")
        if init is None:
            init = self._draw(n, self.opt.d, np.random.RandomState(self.opt.random_seed))
        X0 = fold_in.start_rows(init, n, self.opt.d, 0.0)
        import torch
        st, h = fold_in.resident_state(self, lambda: CuSGD(self._KIND), side="P")
        dev = fold_in.device()
        Qc = np.ascontiguousarray(self.Q[:num_items], dtype=np.float32)
        Qbc = np.ascontiguousarray(np.asarray(self.Qb, dtype=np.float32).reshape(-1)[:num_items])
        Q = st.cached("Q", fold_in.fingerprint(Qc), lambda: fold_in.padded(Qc, h.get_vdim(), self.opt.d))
        Qb = st.cached("Qb", fold_in.fingerprint(Qbc), lambda: torch.from_numpy(Qbc).to(dev))
        # the training data does not change once created: keyed by the object and its size
        train = st.cached("train", (id(self.data), header["num_nnz"]), lambda: self._csr_to_device("rowwise", dev)[:2])
        cum = None
        if self._KIND == "bpr" and self.opt.sampling_power > 0.0:
            table = getattr(self, "sampling_table_", None)
            table = self._popularity_table() if table is None or len(table) != num_items else table
            if table[-1] > 0:             # an all-zero table means uniform sampling, as in training
                cum = st.cached("cum", fold_in.fingerprint(table), lambda: torch.from_numpy(table).to(dev))
        ind_t, users_t, _, tX = fold_in.to_device(indptr, users, np.ones(len(users), np.float32), X0, h.get_vdim())
        tXb = torch.zeros(n, dtype=torch.float32, device=dev)
        tr = None
        if trace:
            nnz = len(users)
            tr = (torch.full((epochs, nnz * per), -2, dtype=torch.int32, device=dev),
                  torch.zeros((epochs, nnz), dtype=torch.int32, device=dev) if self._KIND == "warp" else None)
        if n:
            h.fold_in_items_device(st.F, Q, Qb, train[0], train[1], cum, ind_t, users_t, tX, tXb, epochs,
                                   trace=tr if len(users) else None)
        return tX, tXb, tr


    def get_evaluation_metrics(self):
        return ["val_rmse", "val_ndcg", "val_map", "val_accuracy", "val_error", "train_loss"]

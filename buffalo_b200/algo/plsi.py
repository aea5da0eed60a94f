"""pLSI trainer: the reference's Python EM driver (buffalo/algo/plsi.py) on top of the H100 backend.

Two feeding modes, same results:
  * resident (default when the rowwise CSR and the factors fit in device memory): the CSR and the factor matrices live
    on the GPU for the whole of train(); one update / normalize / swap launch set per iteration;
  * chunked: the reference's own protocol -- reset, obj.partial_update(start_x, next_x, indptr, keys, vals) per
    BufferedDataMatrix chunk, normalize, swap (plsi.py:132-160).
The factor arrays are [rows, d] (plsi.py:107-111: not padded).

With the option `deterministic` (a backend key, false when absent) the new item rows are built by an item pass over
the colwise CSR before the row pass, without atomics, so a fixed random_seed gives bitwise the same model in either
feeding mode.  The resident mode then also holds the colwise CSR and the segment partial rows of long items.
"""
import time

import numpy as np

from buffalo_b200.algo import fold_in
from buffalo_b200.algo.base import Algo, Serializable
from buffalo_b200.algo.options import PLSIOption
from buffalo_b200.backend import CuPLSI
from buffalo_b200.data.base import Data
from buffalo_b200.data.buffered_data import BufferedDataMatrix
from buffalo_b200.evaluate import Evaluable
from buffalo_b200.evaluate.device import EvalModel


class PLSI(Algo, PLSIOption, Evaluable, Serializable):
    """Probabilistic latent semantic indexing trained by EM -- drop-in for buffalo.algo.plsi.PLSI."""

    def __init__(self, opt_path=None, *args, **kwargs):
        Algo.__init__(self, *args, **kwargs)
        PLSIOption.__init__(self, *args, **kwargs)
        Evaluable.__init__(self, *args, **kwargs)
        Serializable.__init__(self, *args, **kwargs)
        self._init_trainer("PLSI", PLSIOption, CuPLSI, opt_path,
                           lambda path, err: "putting parameter to cython object failed (%s)" % err, kwargs)

    @staticmethod
    def new(path, data_fields=[]):
        return PLSI.instantiate(PLSIOption, path, data_fields)

    def set_data(self, data):
        assert isinstance(data, Data), "Wrong instance: {}".format(type(data))
        self.data = data

    def normalize(self, group="item"):
        if group == "item":
            self.Q /= (np.sum(self.Q, axis=0, keepdims=True) + self.opt.eps)
        elif group == "user":
            self.P /= (np.sum(self.P, axis=1, keepdims=True) + self.opt.eps)

    def inherit(self):
        """Copies the rows of a saved model whose ids also occur here (plsi.py:62-89)."""
        def _inherit(key):
            if key == "user":
                self.build_userid_map()
            else:
                self.build_itemid_map()
            curr_idmap = self._idmanager.userid_map if key == "user" else self._idmanager.itemid_map
            prev_idmap = prev_model._idmanager.userid_map if key == "user" else prev_model._idmanager.itemid_map
            curr_obj = self.P if key == "user" else self.Q
            prev_obj = prev_model.P if key == "user" else prev_model.Q
            curr_d, prev_d = curr_obj.shape[1], prev_obj.shape[1]
            assert curr_d == prev_d, f"Dimension mismatch. Current dimension: {curr_d} / Previous dimension: {prev_d}"
            for k, curr_idx in curr_idmap.items():
                if k in prev_idmap:
                    curr_obj[curr_idx] = prev_obj[prev_idmap[k]]

        if not self.opt["inherit_opt"]:
            return
        inherit_opt = self.opt.inherit_opt
        prev_model = PLSI.new(inherit_opt.model_path)
        if inherit_opt.get("inherit_user", False):
            self.logger.info("Inherit from previous user matrix")
            _inherit("user")
        if inherit_opt.get("inherit_item", False):
            self.logger.info("Inherit from previous item matrix")
            _inherit("item")

    def initialize(self):
        super().initialize()
        self.buf = BufferedDataMatrix()
        self.buf.initialize(self.data)
        self.buf.set_group("rowwise")
        self.init_factors()
        self.inherit()

    def init_factors(self):
        assert self.data, "Did not set data"
        header = self.data.get_header()
        self.num_items = header["num_items"]
        self.num_users = header["num_users"]
        self.num_nnz = header["num_nnz"]
        self.vdim = self.obj.get_vdim()
        for name, rows in [("P", self.num_users), ("Q", self.num_items)]:
            setattr(self, name, None)
            setattr(self, name, np.zeros((rows, self.opt.d), dtype="float32"))
        self.obj.initialize_model(self.P, self.Q)

    # ---- queries (host) -----------------------------------------------------------------------
    def _get_topk_recommendation(self, rows, topk, pool=None):
        topks = super()._get_topk_recommendation(self.P[rows], self.Q, pb=None, Qb=None, pool=pool, topk=topk,
                                                 num_workers=self.opt.num_workers)
        return zip(rows, topks)

    def _get_most_similar_item(self, col, topk, pool):
        return super()._get_most_similar_item(col, topk, self.Q, True, pool)      # plsi.py:121-122

    def get_scores(self, row_col_pairs):
        return {(r, c): self.P[r].dot(self.Q[c]) for r, c in row_col_pairs}

    def _get_scores(self, row, col):
        return (self.P[row] * self.Q[col]).sum(axis=1)

    def _get_feature(self, index, group="item"):
        if group == "item":
            return self.Q[index]
        elif group == "user":
            return self.P[index]
        return None

    def _device_eval_model(self):
        return EvalModel(self.P, self.Q, None, None, False)

    # ---- fold-in (DESIGN.md 4.10) -------------------------------------------------------------
    def fold_in(self, histories, init=None, iters=None):
        """float32 [n, d] rows p(z|u) for n histories by Hofmann's folding-in: `iters` EM iterations on each row with
        the item factors Q fixed.  An iteration is the row pass of training (acc = sum v * l / sum(l),
        l = max(p * q, 1e-10)) followed by its row normalisation ((acc + alpha1 / d) / sum).  histories: a scipy sparse
        (n, num_items) matrix or a list of n lists of item ids (unknown ids dropped, value 1.0).  init: None (the
        uniform row 1/d) or an (n, d) array; iters: None means opt.num_iters.  Rows without history keep their start
        row.  P, Q and the training holder are not touched.  On the GPU only (kernel plsi_fold_in_kernel)."""
        tX, _ = self._fold_in_device(histories, init, iters)
        return tX[:, :self.opt.d].cpu().numpy()

    def _fold_in_device(self, histories, init=None, iters=None):
        """fold_in's rows as a torch CUDA tensor [n, vdim] (padding zero), and the histories' device CSR."""
        iters = fold_in.positive_int(self.opt.num_iters if iters is None else iters, "iters")
        st, h, (ind_t, keys_t, vals_t, tX) = fold_in.begin(self, CuPLSI, histories, init, 1.0 / self.opt.d)
        h.fold_in_device(st.F, ind_t, keys_t, vals_t, tX, iters, self.opt.alpha1)
        return tX, (ind_t, keys_t, vals_t)

    # ---- training -----------------------------------------------------------------------------
    def _deterministic(self):
        return bool(self.opt.get("deterministic", False))

    def _iterate(self):
        """The reference protocol: reset, partial_update per rowwise chunk, normalize, swap (plsi.py:132-160).
        Deterministic mode sends the colwise chunks through partial_update_items first."""
        self.obj.reset()
        loss_nume, loss_deno = 0.0, 0.0
        feed_t, update_t, updated = 0.0, 0.0, 0
        if self._deterministic():
            self.buf.set_group("colwise")
            for sz in self.buf.fetch_batch():
                st = time.time()
                start_x, next_x, indptr, keys, vals = self.buf.get()
                feed_t += time.time() - st
                st = time.time()
                self.obj.partial_update_items(start_x, next_x, indptr, keys, vals)
                update_t += time.time() - st
            self.buf.set_group("rowwise")
        for sz in self.buf.fetch_batch():
            st = time.time()
            start_x, next_x, indptr, keys, vals = self.buf.get()
            feed_t += time.time() - st
            st = time.time()
            loss_nume += self.obj.partial_update(start_x, next_x, indptr, keys, vals)
            update_t += time.time() - st
            loss_deno += np.sum(vals)
            updated += sz
        self.obj.normalize(self.opt.alpha1, self.opt.alpha2)
        self.obj.swap()
        self.logger.debug(f"updated processed({updated}) elapsed(data feed: {feed_t:0.5f} update: {update_t:0.5f})")
        return loss_nume, loss_deno

    def _train_resident(self, training_callback):
        import torch
        dev = torch.device("cuda", torch.cuda.current_device())
        d = self.opt.d

        def padded(F):
            T = torch.zeros((F.shape[0], self.vdim), dtype=torch.float32, device=dev)
            T[:, :d] = torch.from_numpy(F).to(dev)
            return T
        tP, tQ = padded(self.P), padded(self.Q)
        self.obj.bind_factors(tP, tQ)
        indptr, keys, vals = self._csr_to_device("rowwise", dev)
        self.obj.bind_csr(indptr, keys, vals)
        deterministic = self._deterministic()
        if deterministic:
            self.obj.bind_colwise_csr(*self._csr_to_device("colwise", dev))
        loss_deno = float(np.sum(vals.cpu().numpy(), dtype=np.float64))
        loss = torch.zeros(1, dtype=torch.float64, device=dev)
        rows, items = self.P.shape[0], self.Q.shape[0]

        def sync_back():
            self.P[:] = tP[:, :d].cpu().numpy()
            self.Q[:] = tQ[:, :d].cpu().numpy()

        def one_iteration():
            loss.zero_()
            if deterministic:
                self.obj.update_items_device(0, items)
            self.obj.update_device(0, rows, loss)
            self.obj.normalize_device(self.opt.alpha1, self.opt.alpha2)
            self.obj.swap_device()
            return self._loss(float(loss.cpu().numpy()[0]), loss_deno)
        try:
            return self._epoch_loop(one_iteration, sync_back, training_callback, "Loss", 1e+10)
        finally:
            sync_back()
            self.obj.set_model(self.P, self.Q)   # leave the holder on host-pointer semantics

    def _train_chunked(self, training_callback):
        return self._epoch_loop(lambda: self._loss(*self._iterate()), lambda: None, training_callback, "Loss", 1e+10)

    def _loss(self, nume, deno):
        return nume / (deno + self.opt.eps)                              # plsi.py:171

    def train(self, training_callback=None):
        self.logger.info(f"Train pLSI, K: {self.opt.d}, alpha1: {self.opt.alpha1}, "
                         f"alpha2: {self.opt.alpha2}, num_workers: {self.opt.num_workers}")
        for name in ("P", "Q"):          # factors replaced or inherited by the user: the backend needs float32 [rows, d]
            setattr(self, name, np.ascontiguousarray(getattr(self, name), dtype=np.float32))
        self.obj.set_model(self.P, self.Q)
        deterministic = self._deterministic()
        resident = self._resident_capable(self._resident_bytes())
        self.logger.info("pLSI feeding: %s, item rows: %s" % ("resident" if resident else "chunked",
                                                               "deterministic item pass" if deterministic else "atomics"))
        if resident:
            loss = self._train_resident(training_callback)
        else:
            loss = self._train_chunked(training_callback)
        ret = {"train_loss": loss}
        ret.update({"val_%s" % k: v for k, v in self.validation_result.items()})
        return ret

    def _resident_bytes(self):
        """Device bytes of the resident mode: the rowwise CSR, the factors and the item accumulator; in deterministic
        mode also the colwise CSR, the per-row losses and the partial rows of the segments of long items."""
        h = self.data.get_header()
        need = h["num_nnz"] * 8 + h["num_users"] * (self.vdim * 4 + 9) + h["num_items"] * self.vdim * 8
        if self._deterministic():
            seg = self.obj.item_segment_len()
            cind = np.asarray(self.data.get_group("colwise")["indptr"][:], dtype=np.int64)
            lens = np.diff(cind, prepend=0)
            segments = int(np.sum((lens[lens > seg] + seg - 1) // seg))
            need += h["num_nnz"] * 8 + h["num_items"] * 8 + h["num_users"] * 8 + segments * self.vdim * 4
        return need

    def _get_data(self):
        return super()._get_data() + [("opt", self.opt), ("Q", self.Q), ("P", self.P)]

    def get_evaluation_metrics(self):
        return ["train_loss", "val_rmse", "val_ndcg", "val_map", "val_accuracy", "val_error"]

"""ALS trainer: the reference's Python epoch driver (buffalo/algo/als.py) on top of the H100 backend.

Two feeding modes, same results:
  * resident (default when the CSR fits in device memory): both CSR orientations and the factor matrices live
    on the GPU for the whole of train(); one launch set per half-epoch, no host traffic inside the loop;
  * chunked: the reference's own protocol -- BufferedDataMatrix chunks pushed through
    obj.partial_update(start_x, next_x, indptr, keys, vals, axis) (als.py:115-142).
The backend is GPU-only; `accelerator` is accepted and ignored (both values run the sm_90a kernels).
"""
import time

import numpy as np

from buffalo_b200.algo import fold_in
from buffalo_b200.algo.base import Algo, Serializable
from buffalo_b200.algo.options import ALSOption
from buffalo_b200.backend import CuALS
from buffalo_b200.data.base import Data
from buffalo_b200.data.buffered_data import BufferedDataMatrix
from buffalo_b200.evaluate import Evaluable
from buffalo_b200.evaluate.device import EvalModel

inited_CUALS = True


class ALS(Algo, ALSOption, Evaluable, Serializable):
    """Collaborative Filtering for Implicit Feedback datasets (Hu, Koren, Volinsky) -- drop-in for buffalo.algo.als.ALS."""

    def __init__(self, opt_path=None, *args, **kwargs):
        Algo.__init__(self, *args, **kwargs)
        ALSOption.__init__(self, *args, **kwargs)
        Evaluable.__init__(self, *args, **kwargs)
        Serializable.__init__(self, *args, **kwargs)
        self._init_trainer("ALS", ALSOption, CuALS, opt_path,
                           lambda path, err: "cannot parse option file: %s (%s)" % (path, err), kwargs)

    @staticmethod
    def new(path, data_fields=[]):
        return ALS.instantiate(ALSOption, path, data_fields)

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
        self.init_factors()

    def init_factors(self):
        assert self.data, "Data is not set"
        self.vdim = self.obj.get_vdim()
        header = self.data.get_header()
        for name, rows in (("P", header["num_users"]), ("Q", header["num_items"])):
            setattr(self, name, None)
            F = np.zeros((rows, self.vdim), dtype=np.float32)
            # abs(N(0, 1/d^2)) (als.py:85-86); drawn at width d so a seed gives the reference's values
            F[:, :self.opt.d] = np.abs(np.random.normal(scale=1.0 / (self.opt.d ** 2), size=(rows, self.opt.d)))
            setattr(self, name, F)
        self.obj.initialize_model(self.P, self.Q)

    # ---- queries (host) -----------------------------------------------------------------------
    def _get_topk_recommendation(self, rows, topk, pool=None):
        topks = super()._get_topk_recommendation(self.P[rows], self.Q, pb=None, Qb=None, pool=pool, topk=topk,
                                                 num_workers=self.opt.num_workers)
        return zip(rows, topks)

    def _get_most_similar_item(self, col, topk, pool):
        return super()._get_most_similar_item(col, topk, self.Q, self.opt._nrz_Q, pool)

    def get_scores(self, row_col_pairs):
        return {(r, c): self.P[r].dot(self.Q[c]) for r, c in row_col_pairs}

    def _get_scores(self, row, col):
        return (self.P[row] * self.Q[col]).sum(axis=1)

    def _get_feature(self, index, group="item"):
        return {"item": self.Q, "user": self.P}[group][index] if group in ("item", "user") else None

    def _device_eval_model(self):
        return EvalModel(self.P, self.Q, None, None, False)

    # ---- fold-in (DESIGN.md 4.10) -------------------------------------------------------------
    def fold_in(self, histories, init=None, sweeps=1):
        """float32 [n, d] user rows for n histories, with the item factors fixed: `sweeps` applications of the row
        solve that train()'s user half-epoch applies (the model's optimizer and options, against the Gram of the current
        Q).  histories: a scipy sparse (n, num_items) matrix in the units of the training data, or a list of n lists of
        item ids (unknown ids dropped, value 1.0).  init: None (zero rows) or an (n, d) array of start rows, e.g.
        self.P[rows] for returning users.  Rows without history keep their start row.  P, Q and the training holder
        are not touched.  On the GPU only: without one the backend's "no CPU fallback" error is raised."""
        tX, _ = self._fold_in_device(histories, init, sweeps)
        return tX[:, :self.opt.d].cpu().numpy()

    def _fold_in_device(self, histories, init=None, sweeps=1):
        """fold_in's rows as a torch CUDA tensor [n, vdim] (padding zero), and the histories' device CSR
        (END offsets int64, keys int32, vals float32; keys / vals hold at least one element)."""
        if self.opt._nrz_Q:
            raise RuntimeError("Cannot fold in users with normalized item factors")
        sweeps = fold_in.positive_int(sweeps, "sweeps")
        st, h, (ind_t, keys_t, vals_t, tX) = fold_in.begin(self, CuALS, histories, init, 0.0)
        n = tX.shape[0]
        if n:
            import torch
            try:
                self._bind_fold_items(st, h, tX)
                h.bind_csr(0, ind_t, keys_t, vals_t)
                # the loss pair train() passes as well, so the solve is the very instantiation of the user half-epoch
                loss = torch.zeros(2, dtype=torch.float64, device=tX.device)
                for _ in range(sweeps):
                    h.update_device(0, 0, n, loss)
            finally:
                # the rows and the CSR belong to this call and are freed with its results (every call binds its own
                # before it solves); the holder keeps only its scratch, the resident Q is st.F
                h._keep = []
        return tX, (ind_t, keys_t, vals_t)

    @staticmethod
    def _bind_fold_items(st, h, X):
        """Binds rows X and the state's resident Q to the fold-in holder h, with the Gram of this Q computed once."""
        h.bind_factors(X, st.F)
        ALS._fold_gram(st, h, 0)

    @staticmethod
    def _fold_gram(st, h, axis):
        """The Gram of the state's resident factors, computed on the holder once per upload of them."""
        if st.derived_key != st.key:
            st.derived_key = None
            h.precompute_device(axis)
            st.derived_key = st.key

    def fold_in_items(self, histories, init=None, sweeps=1):
        """float32 [n, d] item rows for n new items, with the user factors fixed: `sweeps` applications of the row
        solve that train()'s item half-epoch applies (the model's optimizer and options -- reg_i, adaptive_reg with the
        item's entry count, the split-row path for long rows -- against the Gram of the current P).  histories: a scipy
        sparse (n, num_users) matrix in the units of the training data, or a list of n lists of user ids (unknown ids
        dropped, value 1.0).  init: None (zero rows) or an (n, d) array of start rows.  Rows without history keep their
        start row.  P, Q and the training holder are not written; serve the rows with add_items().  The padded P and its
        Gram stay on the device between calls until P or the options change (rows * vdim * 4 bytes: 5 GB at 10M users
        and d = 128).  On the GPU only: without one the backend's "no CPU fallback" error is raised."""
        if self.opt._nrz_P:
            raise RuntimeError("Cannot fold in items with normalized user factors")
        sweeps = fold_in.positive_int(sweeps, "sweeps")
        st, h, (ind_t, keys_t, vals_t, tX) = fold_in.begin(self, CuALS, histories, init, 0.0, side="P")
        n = tX.shape[0]
        if n:
            import torch
            try:
                h.bind_factors(st.F, tX)
                h.bind_csr(1, ind_t, keys_t, vals_t)
                self._fold_gram(st, h, 1)
                loss = torch.zeros(2, dtype=torch.float64, device=tX.device)
                for _ in range(sweeps):
                    h.update_device(1, 0, n, loss)
            finally:
                h._keep = []
        return tX[:, :self.opt.d].cpu().numpy()

    # ---- explanations (DESIGN.md 4.11) --------------------------------------------------------
    EXPLAIN_DMAX, EXPLAIN_KMAX, EXPLAIN_TOPM_MAX = 256, 4096, 64

    def explain(self, histories, items, topm=5):
        """Why each target item scores what it does for each history row: Hu, Koren and Volinsky's section 5 split of
        the score q_i . x_r into one term per history item j, (q_i' A_r^-1 q_j) * (1 + alpha v_j), where
        A_r = Q'Q + alpha sum v_j q_j q_j' + reg_u kappa I and x_r = A_r^-1 sum (1 + alpha v_j) q_j is the exact
        least-squares row of the user half-epoch (kappa = the row's entry count with adaptive_reg, else 1).  Entries of
        one item are summed into one term.  x_r is the exact solve whatever the optimizer: it is fold_in(histories)'s
        row for llt / ldlt at d < 128, while manual_cg and iALS++ (every d >= 128) only approach it, so P[u] . q_i
        after train() is in general not this score.

        histories: as fold_in takes them.  items: an (n, k) integer array of item indexes with -1 for no target (what
        ParALS.topk_recommendation returns), or n lists of item ids (unknown ids become -1; rows padded with -1).
        Returns (scores float32 [n, k], keys int32 [n, k, topm], contributions float32 [n, k, topm]): the topm items
        with the largest contributions, descending, ties to the smaller item index; -1 / 0.0 pad.  A -1 target or an
        empty history gives score 0.0 and keys -1; a row whose A_r meets a non-positive Cholesky pivot gets NaN scores
        and keys -1.  On the GPU only: without one the backend's "no CPU fallback" error is raised."""
        if self.opt._nrz_Q:
            raise RuntimeError("Cannot explain scores with normalized item factors")
        if isinstance(topm, bool) or not isinstance(topm, (int, np.integer)) or not 1 <= topm <= self.EXPLAIN_TOPM_MAX:
            raise ValueError("topm must be an integer in [1, %d], got %r" % (self.EXPLAIN_TOPM_MAX, topm))
        if self.opt.d > self.EXPLAIN_DMAX:
            raise ValueError("explain supports d <= %d, got %d" % (self.EXPLAIN_DMAX, self.opt.d))
        num_items = self.Q.shape[0]
        indptr, keys, vals = fold_in.history_csr(self, histories, num_items)
        targets = fold_in.target_matrix(self, items, len(indptr), num_items, self.EXPLAIN_KMAX)
        st, h = fold_in.resident_state(self, CuALS)
        n, k = targets.shape
        if n == 0 or k == 0:
            return (np.zeros((n, k), np.float32), np.full((n, k, topm), -1, np.int32),
                    np.zeros((n, k, topm), np.float32))
        import torch
        ind_t, keys_t, vals_t = fold_in.csr_to_device(indptr, keys, vals)
        try:
            # the explanation reads Q and its Gram only; the bound rows are a placeholder
            self._bind_fold_items(st, h, torch.zeros((1, h.get_vdim()), dtype=torch.float32, device=ind_t.device))
            out = h.explain_device(ind_t, keys_t, vals_t, torch.from_numpy(targets).to(ind_t.device), topm)
        finally:
            h._keep = []
        return tuple(t.cpu().numpy() for t in out)

    # ---- exploration (DESIGN.md 4.17) ---------------------------------------------------------
    def posterior_sample(self, histories, mean, scale=1.0, seed=0, draw_keys=None):
        """float32 [n, d]: one draw per history row from the Gaussian posterior of its user row, for Thompson sampling.
        Read as Bayesian least squares -- observations p_j with noise precision c_j / sigma^2 and the prior
        N(0, sigma^2 / (reg_u kappa) I) -- the objective of the user half-epoch gives, with the item factors fixed, the
        posterior N(A_r^-1 b_r, sigma^2 A_r^-1), A_r = Q'Q + alpha sum v_j q_j q_j' + reg_u kappa I (kappa = the row's
        entry count with adaptive_reg, else 1).  A draw here is mean[r] + scale L_r^-T z with A_r = L_r L_r' and
        z ~ N(0, I): the caller's mean (P[u], or a fold_in row) with the spread of that posterior.  scale is sigma, the
        caller's choice (not estimated): smaller explores less, 0 returns mean itself.

        histories: as fold_in takes them.  mean: an (n, d) array.  seed: an integer in [0, 2^32).  draw_keys: n distinct
        non-negative integers, default arange(n); z of a row depends only on seed and its draw key (DESIGN.md 4.17 gives
        the Philox words), so a row's draw does not depend on the other rows of the call.  A row whose A_r is not
        positive definite in fp32 comes back as its mean, with a logged warning counting such rows.  d <= 256.  On the
        GPU only: without one the backend's "no CPU fallback" error is raised."""
        tX = self._posterior_sample_device(histories, mean, scale, seed, draw_keys)
        return tX[:, :self.opt.d].cpu().numpy()

    def _posterior_sample_device(self, histories, mean, scale=1.0, seed=0, draw_keys=None):
        """posterior_sample's rows as a torch CUDA tensor [n, vdim] (padding zero); every check before device work."""
        if self.opt._nrz_Q:
            raise RuntimeError("Cannot sample posterior rows with normalized item factors")
        if self.opt.d > self.EXPLAIN_DMAX:
            raise ValueError("posterior_sample supports d <= %d, got %d" % (self.EXPLAIN_DMAX, self.opt.d))
        scale, seed = fold_in.posterior_args(scale, seed)
        indptr, keys, vals = fold_in.history_csr(self, histories, self.Q.shape[0])
        n, d = len(indptr), self.opt.d
        M = np.asarray(mean)
        if M.shape != (n, d) or (M.size and not np.issubdtype(M.dtype, np.number)):
            raise ValueError("mean must be an (%d, %d) array, got %s %s" % (n, d, M.dtype, M.shape))
        K = fold_in.draw_key_array(draw_keys, n)
        st, h = fold_in.resident_state(self, CuALS)
        import torch
        ind_t, keys_t, vals_t, tM = fold_in.to_device(indptr, keys, vals, M.astype(np.float32), h.get_vdim())
        if n == 0:
            return tM
        return self._sample_rows(st, h, (ind_t, keys_t, vals_t), tM, torch.from_numpy(K).to(tM.device), seed, scale)

    def _sample_rows(self, st, h, csr, tM, tK, seed, scale):
        """tM (CUDA [n, vdim], the means) replaced in place by the posterior draws of the device history CSR csr with draw
        keys tK (int64 CUDA [n]); arguments already checked.  Returns tM."""
        import torch
        n = tM.shape[0]
        try:
            # the draws read Q and its Gram only; the bound rows are a placeholder
            self._bind_fold_items(st, h, torch.zeros((1, h.get_vdim()), dtype=torch.float32, device=tM.device))
            _, failed = h.posterior_sample_device(*csr, tM, tK, seed, scale, out=tM)
        finally:
            h._keep = []
        failed = int(failed.item())
        if failed:
            self.logger.warning("posterior_sample: %d of %d rows left at their mean (A_r not positive definite in fp32)"
                                % (failed, n))
        return tM

    # ---- training -----------------------------------------------------------------------------
    def _get_buffer(self):
        buf = BufferedDataMatrix()
        buf.initialize(self.data)
        return buf

    def _iterate(self, buf, group="rowwise"):
        """The reference protocol: precompute, then one partial_update per chunk (als.py:115-142)."""
        axis = 0 if group == "rowwise" else 1
        t0 = time.time()
        self.obj.precompute(axis)
        nume = deno = 0.0
        buf.set_group(group)
        updated = 0
        for sz in buf.fetch_batch():
            updated += sz
            start_x, next_x, indptr, keys, vals = buf.get()
            n_, d_ = self.obj.partial_update(start_x, next_x, indptr, keys, vals, axis)
            nume += n_
            deno += d_
        self.logger.debug(f"{group} updated: processed({updated}) elapsed({time.time() - t0:0.3f}s)")
        return nume, deno

    def _rmse(self, nume, deno):
        return (nume / (deno + self.opt.eps)) ** 0.5           # als.py:171

    def _train_resident(self, training_callback):
        import torch
        dev = torch.device("cuda", torch.cuda.current_device())
        h = self.data.get_header()
        U, I = h["num_users"], h["num_items"]
        tP, tQ = torch.from_numpy(self.P).to(dev), torch.from_numpy(self.Q).to(dev)
        self.obj.bind_factors(tP, tQ)
        for axis, G in enumerate(("rowwise", "colwise")):
            self.obj.bind_csr(axis, *self._csr_to_device(G, dev))
        loss = torch.zeros(2, dtype=torch.float64, device=dev)

        def sync_back():
            self.P[:], self.Q[:] = tP.cpu().numpy(), tQ.cpu().numpy()

        def one_iteration():
            loss.zero_()
            for axis, rows in ((0, U), (1, I)):
                self.obj.precompute_device(axis)
                self.obj.update_device(axis, 0, rows, loss)
            n_, d_ = loss.cpu().numpy()
            return self._rmse(float(n_), float(d_))
        try:
            return self._timed_epochs(one_iteration, sync_back, training_callback)
        finally:
            sync_back()
            self.obj.initialize_model(self.P, self.Q)   # leave the holder on host-pointer semantics

    def _train_chunked(self, training_callback):
        buf = self._get_buffer()
        lindptr, rindptr, batch_size = buf.get_indptrs()
        self.obj.set_placeholder(lindptr, rindptr, batch_size)

        def one_iteration():
            n1, d1 = self._iterate(buf, group="rowwise")
            n2, d2 = self._iterate(buf, group="colwise")
            return self._rmse(n1 + n2, d1 + d2)
        return self._timed_epochs(one_iteration, lambda: None, training_callback)

    def _timed_epochs(self, one_iteration, sync_back, training_callback):
        t_all = time.time()
        rmse = self._epoch_loop(one_iteration, sync_back, training_callback, "RMSE", float("inf"))
        self.logger.info(f"elapsed for full epochs: {time.time() - t_all:.2f} sec")
        return rmse

    def train(self, training_callback=None):
        self._check_catalogue()
        if self.P.shape[1] != self.vdim:      # factors replaced by the user at width d: re-pad
            for name in ("P", "Q"):
                F = getattr(self, name)
                G = np.zeros((F.shape[0], self.vdim), dtype=np.float32)
                G[:, :self.opt.d] = F[:, :self.opt.d]
                setattr(self, name, G)
        self.obj.initialize_model(self.P, self.Q)
        h = self.data.get_header()
        # option `deterministic` (a backend key, false when absent): bitwise repeatable factors and loss on one GPU
        det = bool(self.opt.get("deterministic", False))
        self.logger.info("split rows and loss: %s" % ("deterministic (ordered chunk sums)" if det else "atomics"))
        need = 2 * h["num_nnz"] * 8 + (h["num_users"] + h["num_items"]) * (self.vdim * 4 + 8)
        if det:
            need += self.deterministic_bytes(h["num_users"], h["num_items"], self.opt.get("_b200_det_scratch_mb", 0))
        rmse = self._train_resident(training_callback) if self._resident_capable(need) else self._train_chunked(training_callback)
        if self.opt.d < self.vdim:            # als.py:191-193
            self.P = np.ascontiguousarray(self.P[:, :self.opt.d])
            self.Q = np.ascontiguousarray(self.Q[:, :self.opt.d])
        ret = {"train_loss": rmse}
        ret.update({"val_%s" % k: v for k, v in self.validation_result.items()})
        return ret

    @staticmethod
    def deterministic_bytes(num_users, num_items, scratch_mb=0):
        """Upper bound of the device memory the deterministic mode adds: 16 B of loss terms per row of the longer axis,
        and the scratch budget of one batch of split rows (scratch_mb, fractions allowed, or when 0 the backend's cap
        of 2 GiB).  The backend takes min(free / 4, 2 GiB) and allocates only what the split rows need (0.97 GB at C2),
        so near the residency limit this bound can choose the chunked feed where the resident one would have fitted."""
        return 16 * max(num_users, num_items) + (int(scratch_mb * (1 << 20)) if scratch_mb else 2 << 30)

    def _get_data(self):
        return super()._get_data() + [("opt", self.opt), ("Q", self.Q), ("P", self.P)]

    def get_evaluation_metrics(self):
        return ["train_loss", "val_rmse", "val_ndcg", "val_map", "val_accuracy", "val_error"]

"""Shared driver for the two negative-sampling trainers (BPRMF, WARP): the epoch loop of
buffalo/algo/bpr.py:170-252 / warp.py:187-267 on the H100 backend."""
import time

import numpy as np

from buffalo_b200.data.buffered_data import BufferedDataMatrix


class SGDTrainerMixin(object):
    """Expects: self.obj (CuSGD), self.opt, self.data, self.buf, self.P/Q/Qb, self.logger, self.num_nnz."""

    def _init_buffer(self):
        self.buf = BufferedDataMatrix()
        self.buf.initialize(self.data)

    def sampling_loss_samples(self):
        """sqrt(U) probe triples (bpr.py:135-161): one observed item and one unseen item per sampled user."""
        users, positives, negatives = [], [], []
        if self.opt.compute_loss_on_training:
            self.logger.info("Sampling loss samples...")
            num_users, num_items = self.P.shape[0], self.Q.shape[0]
            for u in np.random.choice(num_users, size=int(num_users ** 0.5), replace=False):
                keys, *_ = self.data.get(int(u))
                if len(keys) == 0:
                    continue
                seen = set(int(k) for k in keys)
                cand = [n for n in np.random.choice(num_items, size=min(len(seen) + 1, num_items), replace=False)
                        if int(n) not in seen]
                if not cand:
                    continue
                users.append(int(u))
                positives.append(int(keys[0]))
                negatives.append(int(cand[0]))
            self.logger.info("Generated %s loss samples." % len(users))
        self._sub_samples = [np.array(a, dtype=np.int32) for a in (users, positives, negatives)]

    def compute_loss(self):
        if len(self._sub_samples[0]) == 0:
            return 0.0
        return self.obj.compute_loss(*self._sub_samples)

    def _iterate(self):
        """add_jobs per chunk, then update_parameters (bpr.py:170-188)."""
        t0 = time.time()
        updated = 0
        self.buf.set_group("rowwise")
        for sz in self.buf.fetch_batch():
            updated += sz
            start_x, next_x, indptr, keys, _ = self.buf.get()
            self.obj.add_jobs(start_x, next_x, indptr, keys)
        self.obj.update_parameters()
        self.logger.debug(f"updated processed({updated}) elapsed({time.time() - t0:0.3f})")

    def _prepare_train(self):
        indptr, _, batch_size = self.buf.get_indptrs()
        # option `deterministic` (a backend key, false when absent): gradient sums in a fixed order, bitwise repeatable
        self.logger.info("gradient accumulation: %s" % ("deterministic (fixed-order user and item passes)"
                                                        if self.opt.get("deterministic", False) else "atomics"))
        # a second train() (or user-replaced factors) arrives at width d: re-pad to vdim like bpr.py's _prepare_train,
        # the native side copies rows * vdim floats in and out
        self.P, self.Q = self._pad(self.P), self._pad(self.Q)
        self.Qb = np.ascontiguousarray(self.Qb, dtype=np.float32).reshape(self.Q.shape[0], 1)
        self.obj.initialize_model(self.P, self.Q, self.Qb, self.num_nnz, True)
        self.obj.set_placeholder(indptr, batch_size)
        if hasattr(self, "sampling_table_"):
            self.obj.set_cumulative_table(self.sampling_table_, len(self.sampling_table_))
        self.obj.launch_workers()

    def _finalize_train(self):
        loss = self.obj.join()          # drains the stream and copies P, Q, Qb back (algo.cc:474-492)
        if self.opt.d < self.P.shape[1]:
            self.P = np.ascontiguousarray(self.P[:, :self.opt.d])
            self.Q = np.ascontiguousarray(self.Q[:, :self.opt.d])
        return loss

    def train(self, training_callback=None):
        self._check_catalogue()
        self.validation_result = {}
        self.sampling_loss_samples()
        self._prepare_train()

        def one_iteration():
            self._iterate()
            self.obj.wait_until_done()
            return self.compute_loss() if self.opt.compute_loss_on_training else 0.0
        # update_parameters() already copied the factors back to the host arrays: nothing to sync
        self._epoch_loop(one_iteration, lambda: None, training_callback, "PR-Loss", float("inf"))
        ret = {"train_loss": self._finalize_train()}
        ret.update({"val_%s" % k: v for k, v in self.validation_result.items()})
        return ret

    def _pad(self, F):
        vdim = self.obj.get_vdim()
        if F.shape[1] == vdim:
            return np.ascontiguousarray(F, dtype=np.float32)
        G = np.zeros((F.shape[0], vdim), dtype=np.float32)
        G[:, :F.shape[1]] = F
        return G

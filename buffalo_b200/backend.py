"""Backend holder objects: the `self.obj` of the algo drivers.

``CuALS`` / ``CuSGD`` / ``CuPLSI`` expose exactly the method set of the reference's Cython holders
(buffalo/algo/_als.pyx:28-63, buffalo/algo/cuda/_als.pyx:25-67, buffalo/algo/_bpr.pyx:34-92,
buffalo/algo/cuda/_bpr.pyx:27-80, buffalo/algo/_warp.pyx:34-92, buffalo/algo/_plsi.pyx:13-57) on top of the C ABI, plus a
device-resident path that takes torch CUDA tensors (PyTorch is used for device memory and
streams only).
"""
import ctypes as C
import json
import os

import numpy as np

from buffalo_b200 import _cabi


def _host(a, dtype, ndim, name):
    # the Cython signatures type-check dtype/ndim and assume C contiguity (_als.pyx:42-63)
    if not isinstance(a, np.ndarray) or a.dtype != dtype or a.ndim != ndim:
        raise ValueError("Buffer dtype/ndim mismatch for %s: expected %s ndim=%d" % (name, np.dtype(dtype), ndim))
    if not a.flags["C_CONTIGUOUS"]:
        raise ValueError("%s must be C-contiguous" % name)
    return a.ctypes.data


def _dev(t, dtype_name, name):
    import torch
    if not isinstance(t, torch.Tensor) or not t.is_cuda or not t.is_contiguous() or str(t.dtype) != "torch." + dtype_name:
        raise ValueError("%s must be a contiguous CUDA tensor of dtype %s" % (name, dtype_name))
    return t.data_ptr()


def _stream_ptr(stream):
    import torch
    s = torch.cuda.current_stream() if stream is None else stream
    return s.cuda_stream


def _opt_bytes(opt):
    if isinstance(opt, (bytes, bytearray)):
        return bytes(opt), True
    if isinstance(opt, str):
        return opt.encode("utf-8"), True
    return json.dumps(dict(opt)).encode("utf-8"), False


def _device_view(ptr, shape, typestr):
    """torch CUDA tensor over `ptr` (memory the library owns) through __cuda_array_interface__."""
    import torch

    class _Arr(object):
        __cuda_array_interface__ = {"shape": tuple(shape), "typestr": typestr, "data": (ptr, False), "version": 2}
    return torch.as_tensor(_Arr(), device="cuda")


class _Holder(object):
    """Lifecycle shared by the bfl_<prefix>_* handles: create/destroy, init, get_vdim and the tensors kept alive
    while the native side holds their pointers."""

    def __init__(self, prefix, *create_args):
        self._lib = _cabi.lib()
        self._prefix = prefix
        self._h = self._fn("create")(*create_args)
        if not self._h:
            raise MemoryError("bfl_%s_create" % prefix)
        self._keep = []

    def _fn(self, name):
        return getattr(self._lib, "bfl_%s_%s" % (self._prefix, name))

    def __del__(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._fn("destroy")(h)

    # --- reference method set -------------------------------------------------------------
    def init(self, opt_path):
        """opt_path: bytes/str path of the JSON option file (als.py:43), or a dict."""
        data, is_path = _opt_bytes(opt_path)
        rc = self._fn("init")(self._h, data) if is_path else self._fn("init_json")(self._h, data)
        if rc == 1:  # BFL_ERR_OPTION: the reference's init returns False (algo.cc:22-34)
            self.last_error = self._lib.bfl_last_error().decode("utf-8", "replace")
            return False
        _cabi.check(rc, "bfl_%s_init" % self._prefix)
        if is_path:
            with open(data.decode("utf-8")) as fin:
                opt = json.load(fin)
        else:
            opt = json.loads(data.decode("utf-8"))
        self._d = int(opt["d"]) if "d" in opt else None
        return True

    def get_vdim(self):
        return self._fn("get_vdim")(self._h)

    def _check_vdim(self, P, Q):
        # the kernels stride rows by vdim, so a narrower matrix would be read and written past its end
        vdim = self.get_vdim()
        if P.ndim != 2 or Q.ndim != 2 or P.shape[1] != vdim or Q.shape[1] != vdim:
            raise ValueError("P and Q must be [rows, vdim=%d] (got %s, %s)" % (vdim, tuple(P.shape), tuple(Q.shape)))


class CuALS(_Holder):
    """ALS backend (CyALS, _als.pyx:28-63; CUDA holder cuda/_als.pyx:25-67)."""

    def __init__(self):
        super().__init__("als")

    def initialize_model(self, P, Q):
        pP, pQ = _host(P, np.float32, 2, "P"), _host(Q, np.float32, 2, "Q")
        self._check_vdim(P, Q)
        self._keep = [P, Q]  # native side retains the pointers (als.cc:78-79)
        _cabi.check(self._lib.bfl_als_initialize_model(self._h, pP, P.shape[0], pQ, Q.shape[0]), "initialize_model")

    def set_placeholder(self, lindptr, rindptr, batch_size):
        _cabi.check(self._lib.bfl_als_set_placeholder(self._h, _host(lindptr, np.int64, 1, "lindptr"),
                                                      _host(rindptr, np.int64, 1, "rindptr"), int(batch_size)),
                    "set_placeholder")

    def precompute(self, axis):
        _cabi.check(self._lib.bfl_als_precompute(self._h, int(axis)), "precompute")

    def partial_update(self, start_x, next_x, indptr, keys, vals, axis):
        nume, deno = C.c_double(0.0), C.c_double(0.0)
        _cabi.check(self._lib.bfl_als_partial_update(self._h, int(start_x), int(next_x),
                                                     _host(indptr, np.int64, 1, "indptr"),
                                                     _host(keys, np.int32, 1, "keys"),
                                                     _host(vals, np.float32, 1, "vals"), int(axis),
                                                     C.byref(nume), C.byref(deno)), "partial_update")
        return nume.value, deno.value

    # --- device-resident path ---------------------------------------------------------------
    def bind_factors(self, P, Q):
        """P, Q: torch float32 CUDA tensors [rows, vdim], updated in place."""
        self._check_vdim(P, Q)
        self._keep = [P, Q]
        _cabi.check(self._lib.bfl_als_bind_factors_device(self._h, _dev(P, "float32", "P"), P.shape[0],
                                                          _dev(Q, "float32", "Q"), Q.shape[0]), "bind_factors")

    def bind_csr(self, axis, indptr, keys, vals):
        """indptr int64[rows] END offsets, keys int32[nnz], vals float32[nnz]: torch CUDA tensors."""
        self._keep += [indptr, keys, vals]
        _cabi.check(self._lib.bfl_als_bind_csr_device(self._h, int(axis), _dev(indptr, "int64", "indptr"),
                                                      _dev(keys, "int32", "keys"), _dev(vals, "float32", "vals"),
                                                      indptr.shape[0], keys.shape[0]), "bind_csr")

    def precompute_device(self, axis, stream=None):
        _cabi.check(self._lib.bfl_als_precompute_device(self._h, int(axis), _stream_ptr(stream)), "precompute_device")

    def precompute_rows_device(self, axis, row_begin, row_end, stream=None):
        """Partial Gram over rows [row_begin,row_end) of the opposite factor (to be all-reduced via gram_tensor())."""
        _cabi.check(self._lib.bfl_als_precompute_rows_device(self._h, int(axis), int(row_begin), int(row_end),
                                                             _stream_ptr(stream)), "precompute_rows_device")

    def update_device(self, axis, row_begin, row_end, loss=None, stream=None):
        """loss: optional torch float64 CUDA tensor[2] receiving (+=) numerator, denominator."""
        lp = _dev(loss, "float64", "loss") if loss is not None else None
        _cabi.check(self._lib.bfl_als_update_device(self._h, int(axis), int(row_begin), int(row_end), lp,
                                                    _stream_ptr(stream)), "update_device")

    def set_peer_replicas(self, axis, pointers):
        """pointers: device addresses (ints), valid in this process, of the other ranks' replicas of the matrix
        updated on `axis` (buffalo_b200.parallel.dist.open_peer_replicas); [] switches the fused exchange off."""
        arr = (C.c_void_p * max(len(pointers), 1))(*[int(p) for p in pointers])
        _cabi.check(self._lib.bfl_als_set_peer_replicas(self._h, int(axis), len(pointers), arr), "set_peer_replicas")

    def explain_device(self, indptr, keys, vals, targets, topm, stream=None):
        """bfl_als_explain_device: (scores float32 [n, k], keys int32 [n, k, topm], contributions float32 [n, k, topm])
        torch CUDA tensors explaining the exact row solve of each history row (indptr int64 [n] END offsets, keys int32
        items in [0, Q_rows), ascending within a row, not checked here; vals float32) for the targets int32 [n, k], against
        the bound Q and the Gram of precompute_device(0)."""
        import torch
        if targets.ndim != 2 or indptr.shape[0] != targets.shape[0]:
            raise ValueError("targets must be [n, k] with one row per END offset (got %s for %d rows)"
                             % (tuple(targets.shape), indptr.shape[0]))
        n, k = targets.shape
        dev = targets.device
        scores = torch.empty((n, k), dtype=torch.float32, device=dev)
        out_keys = torch.empty((n, k, int(topm)), dtype=torch.int32, device=dev)
        contrib = torch.empty((n, k, int(topm)), dtype=torch.float32, device=dev)
        if n:
            _cabi.check(self._lib.bfl_als_explain_device(
                self._h, _dev(indptr, "int64", "indptr"), _dev(keys, "int32", "keys"), _dev(vals, "float32", "vals"), n,
                _dev(targets, "int32", "targets"), int(k), int(topm), scores.data_ptr(), out_keys.data_ptr(),
                contrib.data_ptr(), _stream_ptr(stream)), "bfl_als_explain_device")
        return scores, out_keys, contrib

    def posterior_sample_device(self, indptr, keys, vals, mean, draw_keys, seed, scale, out=None, stream=None):
        """bfl_als_posterior_sample_device: (rows float32 CUDA [n, ld], failed int64 CUDA [1]) -- one draw per history row
        (indptr int64 [n] END offsets, keys int32 items in [0, Q_rows), ascending within a row, not checked here; vals
        float32) from N(mean[r], scale^2 A_r^-1), against the bound Q and the Gram of precompute_device(0).  mean float32
        CUDA [n, ld] (any ld >= d: the pitch of mean and out only, Q is read at the holder's own), draw_keys int64 CUDA
        [n], seed in [0, 2^32), scale finite >= 0.  out: None (a new zero tensor, so its padding columns are zero) or a
        float32 CUDA [n, ld] tensor, which may be mean itself.  failed holds the number of rows left at their mean."""
        import torch
        if mean.ndim != 2 or indptr.ndim != 1 or indptr.shape[0] != mean.shape[0]:
            raise ValueError("mean must be [n, ld] with one row per END offset (got %s for %d rows)"
                             % (tuple(mean.shape), indptr.shape[0]))
        if draw_keys.shape != (mean.shape[0],):
            raise ValueError("draw_keys must be [%d], got %s" % (mean.shape[0], tuple(draw_keys.shape)))
        if not 0 <= int(seed) < 2 ** 32:
            raise ValueError("seed must be in [0, 2^32), got %r" % (seed,))
        n, ld = mean.shape
        if out is None:
            out = torch.zeros_like(mean)
        elif tuple(out.shape) != (n, ld):
            raise ValueError("out must be [%d, %d], got %s" % (n, ld, tuple(out.shape)))
        failed = torch.zeros(1, dtype=torch.int64, device=mean.device)
        if n:
            _cabi.check(self._lib.bfl_als_posterior_sample_device(
                self._h, _dev(indptr, "int64", "indptr"), _dev(keys, "int32", "keys"), _dev(vals, "float32", "vals"), n,
                _dev(mean, "float32", "mean"), int(ld), _dev(draw_keys, "int64", "draw_keys"), int(seed),
                float(scale), _dev(out, "float32", "out"), failed.data_ptr(), _stream_ptr(stream)),
                "bfl_als_posterior_sample_device")
        return out, failed

    def gram_tensor(self):
        """View of the current d x d Gram matrix as a torch tensor (multi-GPU all-reduce, tests)."""
        ptr = self._lib.bfl_als_gram_device_mut(self._h)
        return _device_view(ptr, (self._d * self._d,), "<f4").view(self._d, self._d)


class CuSGD(_Holder):
    """BPRMF / WARP backend (CyBPRMF _bpr.pyx:34-92, CyWARP _warp.pyx:34-92, CyBPR cuda/_bpr.pyx:27-80)."""

    KIND = {"bpr": 0, "warp": 1}

    def __init__(self, kind):
        self.kind = kind
        super().__init__("sgd", self.KIND[kind])

    def initialize_model(self, P, Q, Qb, num_nnz, set_gpu=True):
        self._check_vdim(P, Q)
        if Qb.shape != (Q.shape[0], 1):
            raise ValueError("Qb must be [%d, 1], got %s" % (Q.shape[0], Qb.shape))
        self._keep = [P, Q, Qb]
        _cabi.check(self._lib.bfl_sgd_initialize_model(self._h, _host(P, np.float32, 2, "P"), P.shape[0],
                                                       _host(Q, np.float32, 2, "Q"), Q.shape[0],
                                                       _host(Qb, np.float32, 2, "Qb"), int(num_nnz)),
                    "initialize_model")

    def set_cumulative_table(self, sampling_table, size):
        _cabi.check(self._lib.bfl_sgd_set_cumulative_table(self._h, _host(sampling_table, np.int64, 1, "cum"),
                                                           int(size)), "set_cumulative_table")

    def set_placeholder(self, indptr, batch_size):
        _cabi.check(self._lib.bfl_sgd_set_placeholder(self._h, _host(indptr, np.int64, 1, "indptr"),
                                                      int(batch_size)), "set_placeholder")

    def launch_workers(self):
        _cabi.check(self._lib.bfl_sgd_launch_workers(self._h), "launch_workers")

    def add_jobs(self, start_x, next_x, indptr, keys):
        _cabi.check(self._lib.bfl_sgd_add_jobs(self._h, int(start_x), int(next_x),
                                               _host(indptr, np.int64, 1, "indptr"),
                                               _host(keys, np.int32, 1, "keys")), "add_jobs")

    def update_parameters(self):
        _cabi.check(self._lib.bfl_sgd_update_parameters(self._h), "update_parameters")

    def wait_until_done(self):
        _cabi.check(self._lib.bfl_sgd_wait_until_done(self._h), "wait_until_done")

    def synchronize(self, device_to_host):
        _cabi.check(self._lib.bfl_sgd_synchronize(self._h, int(bool(device_to_host))), "synchronize")

    def compute_loss(self, users, positives, negatives):
        out = C.c_double(0.0)
        _cabi.check(self._lib.bfl_sgd_compute_loss(self._h, int(users.shape[0]), _host(users, np.int32, 1, "users"),
                                                   _host(positives, np.int32, 1, "positives"),
                                                   _host(negatives, np.int32, 1, "negatives"), C.byref(out)),
                    "compute_loss")
        return out.value

    def join(self):
        out = C.c_double(0.0)
        _cabi.check(self._lib.bfl_sgd_join(self._h, C.byref(out)), "join")
        return out.value

    # --- device-resident path ---------------------------------------------------------------
    def bind_factors(self, P, Q, Qb, num_total_samples):
        """P, Q: torch float32 CUDA tensors [rows, vdim] (padding columns zero), Qb: Q.shape[0] floats; updated in
        place."""
        self._check_vdim(P, Q)
        if Qb.numel() != Q.shape[0]:
            raise ValueError("Qb must hold %d elements (one per row of Q), got %s" % (Q.shape[0], tuple(Qb.shape)))
        self._keep = [P, Q, Qb]
        _cabi.check(self._lib.bfl_sgd_bind_factors_device(self._h, _dev(P, "float32", "P"), P.shape[0],
                                                          _dev(Q, "float32", "Q"), Q.shape[0],
                                                          _dev(Qb, "float32", "Qb"), int(num_total_samples)),
                    "bind_factors")

    def bind_csr(self, indptr, keys):
        self._keep += [indptr, keys]
        _cabi.check(self._lib.bfl_sgd_bind_csr_device(self._h, _dev(indptr, "int64", "indptr"),
                                                      _dev(keys, "int32", "keys"), indptr.shape[0], keys.shape[0]),
                    "bind_csr")

    def add_jobs_device(self, row_begin, row_end, stream=None):
        _cabi.check(self._lib.bfl_sgd_add_jobs_device(self._h, int(row_begin), int(row_end), _stream_ptr(stream)),
                    "add_jobs_device")

    def update_parameters_device(self, stream=None):
        _cabi.check(self._lib.bfl_sgd_update_parameters_device(self._h, _stream_ptr(stream)),
                    "update_parameters_device")

    def sample_device(self, row_begin, row_end, users, pos, neg, stream=None):
        _cabi.check(self._lib.bfl_sgd_sample_device(self._h, int(row_begin), int(row_end),
                                                    _dev(users, "int32", "users"), _dev(pos, "int32", "pos"),
                                                    _dev(neg, "int32", "neg"), _stream_ptr(stream)), "sample_device")

    def apply_triples_device(self, users, pos, neg, lr, stream=None):
        _cabi.check(self._lib.bfl_sgd_apply_triples_device(self._h, _dev(users, "int32", "users"),
                                                           _dev(pos, "int32", "pos"), _dev(neg, "int32", "neg"),
                                                           users.shape[0], float(lr), _stream_ptr(stream)),
                    "apply_triples_device")

    def grad_tensor(self, which, shape):
        ptr = self._lib.bfl_sgd_grad_device(self._h, int(which))
        if not ptr:
            return None
        return _device_view(ptr, (int(np.prod(shape)),), "<f4").view(*shape)

    def count_tensor(self, which, rows):
        """int32[rows] sample counters of per_coordinate_normalize (0: P rows, 1: Q rows); None if not allocated."""
        ptr = self._lib.bfl_sgd_count_device(self._h, int(which))
        if not ptr:
            return None
        return _device_view(ptr, (int(rows),), "<i4")

    def set_trace(self, trials, negs):
        self._keep += [trials, negs]
        _cabi.check(self._lib.bfl_sgd_set_trace_device(self._h, _dev(trials, "int32", "trials"),
                                                       _dev(negs, "int32", "negs")), "set_trace")

    def epoch(self):
        return self._lib.bfl_sgd_epoch(self._h)

    def current_lr(self):
        return self._lib.bfl_sgd_current_lr(self._h)

    def read_stats(self):
        loss, n = C.c_double(0.0), C.c_int64(0)
        _cabi.check(self._lib.bfl_sgd_read_stats(self._h, C.byref(loss), C.byref(n)), "read_stats")
        return loss.value, n.value

    def reduce_items_device(self, stream=None):
        """Deterministic mode: adds the item sums of the samples recorded since the last call to the Q / Qb gradient
        accumulators and the WARP loss terms to the running loss.  update_parameters does it first; call it to read
        (or all-reduce) an epoch's accumulators before the optimizer step."""
        _cabi.check(self._lib.bfl_sgd_reduce_items_device(self._h, _stream_ptr(stream)), "reduce_items_device")

    @staticmethod
    def segment_len():
        """Samples / item entries per segment of the deterministic user and item sums."""
        return _cabi.lib().bfl_sgd_segment_len()

    def fold_in_items_device(self, P, Q, Qb, train_indptr, train_keys, cum, indptr, users, X, Xb, epochs, trace=None,
                             stream=None):
        """Item fold-in (bfl_sgd_fold_in_items_device): `epochs` epochs of training's item side on the rows X [n, vdim]
        and biases Xb [n] (start values in, results out) with P, Q [rows, vdim] and Qb [Q rows] frozen.  train_indptr /
        train_keys: the training data's rowwise CSR (int64 END offsets, int32 items); cum: the int64 popularity table or
        None for uniform negatives; indptr / users: the new rows' END offsets and int32 user ids.  trace: None or
        (negs, trials) int32 tensors [epochs, nnz * samples per positive] / [epochs, nnz] (trials None for BPR).  All
        torch CUDA tensors."""
        self._check_vdim(P, X)
        if Q.shape[1] != P.shape[1] or Qb.numel() != Q.shape[0] or Xb.numel() != X.shape[0]:
            raise ValueError("Q must be [rows, %d] with one Qb entry per row, and Xb one entry per row of X"
                             % P.shape[1])
        if indptr.shape[0] != X.shape[0]:
            raise ValueError("indptr must hold one END offset per row of X (%d), got %d" % (X.shape[0], indptr.shape[0]))
        negs, trials = trace if trace is not None else (None, None)
        _cabi.check(self._lib.bfl_sgd_fold_in_items_device(
            self._h, _dev(P, "float32", "P"), P.shape[0], _dev(Q, "float32", "Q"), _dev(Qb, "float32", "Qb"),
            Q.shape[0], _dev(train_indptr, "int64", "train_indptr"), _dev(train_keys, "int32", "train_keys"),
            None if cum is None else _dev(cum, "int64", "cum"), _dev(indptr, "int64", "indptr"),
            _dev(users, "int32", "users"), X.shape[0], users.shape[0], _dev(X, "float32", "X"),
            _dev(Xb, "float32", "Xb"), int(epochs), None if negs is None else _dev(negs, "int32", "negs"),
            None if trials is None else _dev(trials, "int32", "trials"), _stream_ptr(stream)),
            "bfl_sgd_fold_in_items_device")


class CuPLSI(_Holder):
    """pLSI backend (CyPLSI, buffalo/algo/_plsi.pyx:13-57).  Holder methods take the [rows, d] host arrays of
    buffalo/algo/plsi.py:107-111; the device-resident path takes [rows, vdim] torch CUDA tensors."""

    def __init__(self):
        super().__init__("plsi")

    def _factors(self, P, Q):
        pP, pQ = _host(P, np.float32, 2, "P"), _host(Q, np.float32, 2, "Q")
        if P.shape[1] != self._d or Q.shape[1] != self._d:
            raise ValueError("factor matrices must have d=%d columns" % self._d)
        self._keep = [P, Q]  # native side retains the pointers (plsi.cc:46-47)
        return pP, pQ

    def initialize_model(self, P, Q):
        """Fills P [users, d] and Q [items, d] in place with the normalised random start (plsi.cc:44-70)."""
        pP, pQ = self._factors(P, Q)
        _cabi.check(self._lib.bfl_plsi_initialize_model(self._h, pP, P.shape[0], pQ, Q.shape[0]), "initialize_model")

    def set_model(self, P, Q):
        """Retains P and Q and uploads their current values (inherited or user-replaced factors)."""
        pP, pQ = self._factors(P, Q)
        _cabi.check(self._lib.bfl_plsi_set_model(self._h, pP, P.shape[0], pQ, Q.shape[0]), "set_model")

    def reset(self):
        _cabi.check(self._lib.bfl_plsi_reset(self._h), "reset")

    def partial_update(self, start_x, next_x, indptr, keys, vals):
        loss = C.c_double(0.0)
        _cabi.check(self._lib.bfl_plsi_partial_update(self._h, int(start_x), int(next_x),
                                                      _host(indptr, np.int64, 1, "indptr"),
                                                      _host(keys, np.int32, 1, "keys"),
                                                      _host(vals, np.float32, 1, "vals"), C.byref(loss)),
                    "partial_update")
        return loss.value

    def partial_update_items(self, start_x, next_x, indptr, keys, vals):
        """Deterministic mode: the item pass over one colwise chunk (items [start_x, next_x)), before the rowwise
        chunks of the same iteration.  Same conventions as partial_update."""
        _cabi.check(self._lib.bfl_plsi_partial_update_items(self._h, int(start_x), int(next_x),
                                                            _host(indptr, np.int64, 1, "indptr"),
                                                            _host(keys, np.int32, 1, "keys"),
                                                            _host(vals, np.float32, 1, "vals")),
                    "partial_update_items")

    def item_segment_len(self):
        """Entries per segment of a long item row in the deterministic item pass."""
        return self._lib.bfl_plsi_item_segment_len()

    def normalize(self, alpha1, alpha2):
        _cabi.check(self._lib.bfl_plsi_normalize(self._h, float(alpha1), float(alpha2)), "normalize")

    def swap(self):
        _cabi.check(self._lib.bfl_plsi_swap(self._h), "swap")

    def release(self):
        _cabi.check(self._lib.bfl_plsi_release(self._h), "release")
        self._keep = []

    # --- device-resident path ---------------------------------------------------------------
    def bind_factors(self, P, Q):
        """P, Q: torch float32 CUDA tensors [rows, vdim] (padding columns zero), updated in place."""
        self._check_vdim(P, Q)
        self._keep = [P, Q]
        _cabi.check(self._lib.bfl_plsi_bind_factors_device(self._h, _dev(P, "float32", "P"), P.shape[0],
                                                           _dev(Q, "float32", "Q"), Q.shape[0]), "bind_factors")

    def bind_csr(self, indptr, keys, vals):
        """Rowwise CSR: indptr int64[rows] END offsets, keys int32[nnz], vals float32[nnz] torch CUDA tensors."""
        self._keep += [indptr, keys, vals]
        _cabi.check(self._lib.bfl_plsi_bind_csr_device(self._h, _dev(indptr, "int64", "indptr"),
                                                       _dev(keys, "int32", "keys"), _dev(vals, "float32", "vals"),
                                                       indptr.shape[0], keys.shape[0]), "bind_csr")

    def bind_colwise_csr(self, indptr, keys, vals):
        """Deterministic mode: the colwise CSR (indptr int64[items] END offsets, keys int32[nnz] user rows,
        vals float32[nnz]) as torch CUDA tensors, bound after the factors."""
        self._keep += [indptr, keys, vals]
        _cabi.check(self._lib.bfl_plsi_bind_colwise_csr_device(self._h, _dev(indptr, "int64", "indptr"),
                                                               _dev(keys, "int32", "keys"),
                                                               _dev(vals, "float32", "vals"),
                                                               indptr.shape[0], keys.shape[0]), "bind_colwise_csr")

    def update_items_device(self, item_begin, item_end, stream=None):
        """Deterministic mode: the item pass over items [item_begin, item_end), before update_device."""
        _cabi.check(self._lib.bfl_plsi_update_items_device(self._h, int(item_begin), int(item_end),
                                                           _stream_ptr(stream)), "update_items_device")

    def update_device(self, row_begin, row_end, loss=None, stream=None):
        """loss: optional torch float64 CUDA tensor[1] receiving (+=) -sum v log(norm)."""
        lp = _dev(loss, "float64", "loss") if loss is not None else None
        _cabi.check(self._lib.bfl_plsi_update_device(self._h, int(row_begin), int(row_end), lp, _stream_ptr(stream)),
                    "update_device")

    def normalize_device(self, alpha1, alpha2, stream=None):
        _cabi.check(self._lib.bfl_plsi_normalize_device(self._h, float(alpha1), float(alpha2), _stream_ptr(stream)),
                    "normalize_device")

    def swap_device(self, stream=None):
        _cabi.check(self._lib.bfl_plsi_swap_device(self._h, _stream_ptr(stream)), "swap_device")

    def fold_in_device(self, Q, indptr, keys, vals, X, iters, alpha1, stream=None):
        """Folding-in (bfl_plsi_fold_in_device): `iters` EM iterations on the rows of X [rows, vdim] (start rows in,
        results out) against the fixed item factors Q [Q_rows, vdim], for the history CSR indptr int64[rows] END
        offsets, keys int32, vals float32.  All torch CUDA tensors; keys must lie in [0, Q_rows) (not checked here)."""
        vdim = self.get_vdim()
        if Q.ndim != 2 or X.ndim != 2 or Q.shape[1] != vdim or X.shape[1] != vdim:
            raise ValueError("Q and X must be [rows, vdim=%d] (got %s, %s)" % (vdim, tuple(Q.shape), tuple(X.shape)))
        if indptr.shape[0] != X.shape[0]:
            raise ValueError("indptr must hold one END offset per row of X")
        nnz = keys.shape[0]
        _cabi.check(self._lib.bfl_plsi_fold_in_device(
            self._h, _dev(Q, "float32", "Q"), Q.shape[0], _dev(indptr, "int64", "indptr"), _dev(keys, "int32", "keys"),
            _dev(vals, "float32", "vals"), X.shape[0], nnz, _dev(X, "float32", "X"), int(iters), float(alpha1),
            _stream_ptr(stream)), "bfl_plsi_fold_in_device")


def device_available():
    """True when the CUDA library is loadable and a GPU is visible (used by host-side helpers that have a device
    implementation; the training backends never consult this: they fail loudly without a GPU)."""
    try:
        import torch
        return bool(torch.cuda.is_available()) and os.path.isfile(_cabi.LIB_PATH)
    except Exception:
        return False


def require_device():
    """Raises the library's BackendError ("... no CPU fallback") unless an sm_90 GPU is current."""
    _cabi.check(_cabi.lib().bfl_require_device(), "bfl_require_device")


def topk_host(queries, items, item_bias, k):
    """k best item indices per query row for scores = queries @ items.T (+ item_bias), best first, computed on the
    device (bfl_topk_host).  queries [nq, d], items [I, d] float32 host arrays; returns int32 [nq, k]."""
    q = np.ascontiguousarray(queries, dtype=np.float32)
    it = np.ascontiguousarray(items, dtype=np.float32)
    if q.ndim == 1:
        q = q.reshape(1, -1)
    d = min(q.shape[1], it.shape[1])
    k = int(min(k, it.shape[0]))
    out = np.empty((q.shape[0], k), dtype=np.int32)
    b = None if item_bias is None else np.ascontiguousarray(np.asarray(item_bias, dtype=np.float32).reshape(-1))
    _cabi.check(_cabi.lib().bfl_topk_host(q.ctypes.data, q.shape[0], q.shape[1], it.ctypes.data, it.shape[0],
                                          it.shape[1], None if b is None else b.ctypes.data, int(d), k,
                                          out.ctypes.data, None), "bfl_topk_host")
    return out


def topk_device(queries, items, item_bias, k, stream=None):
    """Device tensors in, device tensors out: (idx int32 [nq, k], val float32 [nq, k])."""
    import torch
    nq, n_items = queries.shape[0], items.shape[0]
    k = int(min(k, n_items))
    idx = torch.empty((nq, k), dtype=torch.int32, device=queries.device)
    val = torch.empty((nq, k), dtype=torch.float32, device=queries.device)
    _cabi.check(_cabi.lib().bfl_topk_device(_dev(queries, "float32", "queries"), nq, queries.stride(0),
                                            _dev(items, "float32", "items"), n_items, items.stride(0),
                                            None if item_bias is None else _dev(item_bias, "float32", "bias"),
                                            int(min(queries.shape[1], items.shape[1])), k, idx.data_ptr(), val.data_ptr(),
                                            _stream_ptr(stream)), "bfl_topk_device")
    return idx, val


SERVE_KMAX = 4096
MMR_MMAX = 256        # candidates per row of the MMR re-ranking (its Gram triangle lives in shared memory)


class Serve(_Holder):
    """Batch top-k handle (csrc/serve.cu, bfl_serve_*): the item and query factors stay on the device between calls.
    Host arrays are uploaded once by set_items / set_queries; bind_items / bind_queries borrow torch CUDA tensors."""

    def __init__(self):
        super(Serve, self).__init__("serve")
        self.num_items = self.num_queries = 0
        self._d = None
        self._bound = {}                            # device tensors the native side holds pointers to

    def _destroy(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._fn("destroy")(h)
        self._bound = {}

    close = __del__ = _destroy

    @staticmethod
    def _matrix(a, name):
        _host(a, np.float32, 2, name)
        return a.ctypes.data, a.shape[0], a.shape[1]

    def _items_changed(self, rows, d):
        # the native side drops the pool and the queries with the old items
        self.num_items, self._d, self.num_queries = rows, d, 0
        self._bound = {}

    def set_items(self, items, item_bias=None, d=None):
        """items float32 [I, ld] host array (C-contiguous), the first d columns are used; item_bias float32 [I].
        Clears the pool and the queries."""
        ptr, rows, ld = self._matrix(items, "items")
        d = ld if d is None else int(d)
        if rows == 0 or not 0 < d <= ld:
            raise ValueError("items must have rows and 0 < d <= its width")
        b = None
        if item_bias is not None:
            b = np.ascontiguousarray(np.asarray(item_bias, dtype=np.float32).reshape(-1))
            if b.shape[0] != rows:
                raise ValueError("item_bias must have one value per item")
        self._items_changed(0, None)
        _cabi.check(self._fn("set_items")(self._h, ptr, rows, ld, d, None if b is None else b.ctypes.data), "set_items")
        self._items_changed(rows, d)

    def set_queries(self, queries):
        """queries float32 [N, ld] host array; the array given to set_items shares its resident copy."""
        ptr, rows, ld = self._matrix(queries, "queries")
        if self._d is None:
            raise ValueError("set the items before the queries")
        if rows == 0 or ld < self._d:
            raise ValueError("queries must have rows and at least d columns")
        _cabi.check(self._fn("set_queries")(self._h, ptr, rows, ld), "set_queries")
        self._bound.pop("queries", None)
        self.num_queries = rows

    def bind_items(self, items, item_bias=None, d=None):
        """Borrows torch CUDA tensors (kept alive by this object).  Clears the pool and the queries."""
        ptr = _dev(items, "float32", "items")
        d = items.shape[1] if d is None else int(d)
        b = None if item_bias is None else _dev(item_bias, "float32", "item_bias")
        self._items_changed(0, None)
        _cabi.check(self._fn("bind_items_device")(self._h, ptr, items.shape[0], items.stride(0), d, b), "bind_items")
        self._items_changed(items.shape[0], d)
        self._bound["items"] = (items, item_bias)

    def bind_queries(self, queries):
        _cabi.check(self._fn("bind_queries_device")(self._h, _dev(queries, "float32", "queries"), queries.shape[0],
                                                    queries.stride(0)), "bind_queries")
        self._bound["queries"] = queries
        self.num_queries = queries.shape[0]

    def unbind_queries(self):
        """Drops this object's hold on the tensor given to bind_queries, so it can be freed; the handle has no queries
        until the next set_queries / bind_queries."""
        self._bound.pop("queries", None)
        self.num_queries = 0

    def set_pool(self, pool):
        """pool: int32 indices into the items (None removes it).  An empty pool is an error."""
        if pool is None:
            _cabi.check(self._fn("set_pool")(self._h, None, 0), "set_pool")
            return
        p = np.ascontiguousarray(pool, dtype=np.int32).reshape(-1)
        if p.size == 0:
            raise ValueError("pool is empty")
        if p.min() < 0 or p.max() >= self.num_items:
            raise ValueError("pool index out of range")
        _cabi.check(self._fn("set_pool")(self._h, p.ctypes.data, p.size), "set_pool")

    @staticmethod
    def _check_k(k):
        k = int(k)
        if not 1 <= k <= SERVE_KMAX:
            raise ValueError("k must be in [1, %d]" % SERVE_KMAX)
        return k

    def _topk_host(self, name, query_idx, k, want_scores, rows=lambda n: ()):
        """The host-array entries: k and the query indexes checked, then rows(n) (the entry's CSR arguments for n
        queries, checked: arrays or None), then bfl_<name>(handle, queries, n, k, *their pointers, outputs), which
        batches the queries and copies each batch back while the next one runs; not called for no queries."""
        k = self._check_k(k)
        q = np.ascontiguousarray(query_idx, dtype=np.int32).reshape(-1)
        if q.size and (q.min() < 0 or q.max() >= self.num_queries):
            raise ValueError("query index out of range")
        arrays = rows(q.size)
        idx = np.empty((q.size, k), dtype=np.int32)
        val = np.empty((q.size, k), dtype=np.float32) if want_scores else None
        if q.size:
            ptrs = [None if a is None else a.ctypes.data for a in arrays]
            _cabi.check(getattr(self._lib, "bfl_" + name)(self._h, q.ctypes.data, q.size, k, *ptrs, idx.ctypes.data,
                                                          None if val is None else val.ctypes.data), "bfl_" + name)
        return idx, val

    def _host_rows(self, n, indptr, keys, what="seen"):
        """(END offsets, keys) of a host CSR argument checked by _check_seen (keys: one zero when empty)."""
        nnz = self._check_seen(n, indptr, keys, host=True, what=what)
        return indptr, keys if nnz else np.zeros(1, np.int32)

    def topk(self, query_idx, k, want_scores=True):
        """(int32 [n, k] item ids, float32 [n, k] scores or None) for the rows query_idx of the query matrix: best
        first, ties to the smaller id, -1 / 0.0 where fewer than k candidates exist."""
        return self._topk_host("serve_topk", query_idx, k, want_scores)

    def topk_device(self, query_idx, k, stream=None):
        """torch CUDA int32 query_idx [n] -> (int32 [n, k], float32 [n, k]) CUDA tensors, stream-ordered."""
        import torch
        k = self._check_k(k)
        n = query_idx.shape[0]
        idx = torch.empty((n, k), dtype=torch.int32, device=query_idx.device)
        val = torch.empty((n, k), dtype=torch.float32, device=query_idx.device)
        if n:
            _cabi.check(self._fn("topk_device")(self._h, _dev(query_idx, "int32", "query_idx"), n, k, idx.data_ptr(),
                                                val.data_ptr(), _stream_ptr(stream)), "bfl_serve_topk_device")
        return idx, val

    def _check_seen(self, n, seen_indptr, seen_keys, host, what="seen"):
        """Argument checks of the seen rows (or, what="cand", of the candidate lists): END offsets int64 [n],
        non-decreasing from 0, keys int32 in the items."""
        check = _host if host else (lambda a, dt, nd, name: _dev(a, np.dtype(dt).name, name))
        check(seen_indptr, np.int64, 1, what + "_indptr")
        check(seen_keys, np.int32, 1, what + "_keys")
        if seen_indptr.shape[0] != n:
            raise ValueError("%s_indptr must hold one END offset per query (%d), got %d" % (what, n, seen_indptr.shape[0]))
        ptr = seen_indptr if host else seen_indptr.cpu().numpy()
        nnz = int(ptr[-1]) if n else 0
        if n and (ptr[0] < 0 or (np.diff(ptr) < 0).any()):
            raise ValueError("%s_indptr must be non-decreasing END offsets from 0" % what)
        if nnz > seen_keys.shape[0]:
            raise ValueError("%s_indptr ends past the %d %s keys" % (what, seen_keys.shape[0], what))
        if nnz:
            keys = seen_keys[:nnz]
            lo, hi = (int(keys.min()), int(keys.max())) if host else (int(keys.min().item()), int(keys.max().item()))
            if lo < 0 or hi >= self.num_items:
                raise ValueError("%s key out of range [0, %d)" % (what, self.num_items))
        return nnz

    def topk_seen(self, query_idx, k, seen_indptr, seen_keys, want_scores=True):
        """topk with query i's seen items left out: row i of the host CSR (seen_indptr int64 END offsets [n], seen_keys
        int32 item ids in any order, duplicates allowed).  The survivors keep their order and score bits; -1 / 0.0 pad
        when fewer than k candidates remain."""
        return self._topk_host("seen_topk", query_idx, k, want_scores,
                               lambda n: self._host_rows(n, seen_indptr, seen_keys))

    def _device_rows(self, indptr, keys, row, n, what, stream):
        """(END offsets, keys, row map) of a CSR of torch CUDA tensors (int64 END offsets, int32 keys) that n queries
        read: checked by _check_seen (keys: one zero when empty); seen rows not in ascending order sorted first with the
        device radix sort (eval_unsorted_rows, csr_from_triples_device; that check synchronises), candidate lists kept
        in their order; the row map checked by _check_rows."""
        import torch
        dev = indptr.device
        nnz = self._check_seen(indptr.shape[0], indptr, keys, host=False, what=what)
        keys = keys[:nnz] if nnz else torch.zeros(1, dtype=torch.int32, device=dev)
        if what == "seen" and nnz and eval_unsorted_rows(indptr, keys, stream):
            lens = torch.diff(indptr, prepend=indptr.new_zeros(1))
            major = torch.repeat_interleave(torch.arange(indptr.shape[0], dtype=torch.int32, device=dev), lens)
            indptr, keys, _ = csr_from_triples_device(major, keys, torch.ones(nnz, dtype=torch.float32, device=dev),
                                                      indptr.shape[0], self.num_items, stream=stream)
        return indptr, keys, self._check_rows(row, n, indptr.shape[0], what)

    def topk_seen_device(self, query_idx, k, seen_indptr, seen_keys, seen_row=None, stream=None):
        """topk_device with query q's seen items left out: row seen_row[q] (default q) of a CSR of torch CUDA tensors
        (int64 END offsets, int32 keys).  Rows not in ascending order are sorted first with the device radix sort
        (eval_unsorted_rows, csr_from_triples_device); that check synchronises."""
        import torch
        k = self._check_k(k)
        n = query_idx.shape[0]
        dev = query_idx.device
        seen_indptr, keys, seen_row = self._device_rows(seen_indptr, seen_keys, seen_row, n, "seen", stream)
        if seen_row is None:
            seen_row = torch.arange(n, dtype=torch.int32, device=dev)     # bfl_seen_topk_device takes a row map
        idx = torch.empty((n, k), dtype=torch.int32, device=dev)
        val = torch.empty((n, k), dtype=torch.float32, device=dev)
        if n:
            _cabi.check(self._lib.bfl_seen_topk_device(
                self._h, _dev(query_idx, "int32", "query_idx"), n, k, seen_indptr.data_ptr(), keys.data_ptr(),
                _dev(seen_row, "int32", "seen_row"), idx.data_ptr(), val.data_ptr(), _stream_ptr(stream)),
                "bfl_seen_topk_device")
        return idx, val

    def topk_candidates(self, query_idx, k, cand_indptr, cand_keys, seen=None, want_scores=True):
        """topk where query i ranks only its own candidate list, row i of the host CSR (cand_indptr int64 END offsets
        [n], cand_keys int32 item ids in any order, duplicates allowed) instead of the pool: row i is bitwise what topk
        returns for query i alone with set_pool(its list), ties to the earlier list position.  seen: None or
        (seen_indptr, seen_keys) as topk_seen takes them.  An empty list, or fewer than k candidates left, pads with
        -1 / 0.0."""
        return self._topk_host("cand_topk", query_idx, k, want_scores, lambda n: self._host_rows(
            n, cand_indptr, cand_keys, "cand") + ((None, None) if seen is None else self._host_rows(n, *seen)))

    def topk_candidates_device(self, query_idx, k, cand_indptr, cand_keys, cand_row=None, seen=None, stream=None):
        """topk_candidates on torch CUDA tensors, stream-ordered: query q ranks row cand_row[q] (default q) of the
        candidate CSR (int64 END offsets, int32 keys); seen: None or (seen_indptr, seen_keys[, seen_row]) as
        topk_seen_device takes them (rows not in ascending order are sorted first).  Synchronises once per internal
        batch."""
        import torch
        k = self._check_k(k)
        n = query_idx.shape[0]
        dev = query_idx.device
        cand_indptr, ckeys, cand_row = self._device_rows(cand_indptr, cand_keys, cand_row, n, "cand", stream)
        sptr = skeys = srow = None
        if seen is not None:
            sptr, skeys, srow = self._device_rows(seen[0], seen[1], seen[2] if len(seen) > 2 else None, n, "seen",
                                                  stream)
        idx = torch.empty((n, k), dtype=torch.int32, device=dev)
        val = torch.empty((n, k), dtype=torch.float32, device=dev)
        if n:
            _cabi.check(self._lib.bfl_cand_topk_device(
                self._h, _dev(query_idx, "int32", "query_idx"), n, k, cand_indptr.data_ptr(), ckeys.data_ptr(),
                None if cand_row is None else cand_row.data_ptr(), None if sptr is None else sptr.data_ptr(),
                None if skeys is None else skeys.data_ptr(), None if srow is None else srow.data_ptr(),
                idx.data_ptr(), val.data_ptr(), _stream_ptr(stream)), "bfl_cand_topk_device")
        return idx, val

    def rerank_mmr_device(self, cand_idx, cand_val, k, diversify, stream=None):
        """MMR re-ranking (bfl_mmr_rerank_device) of torch CUDA candidate lists against the handle's items: cand_idx
        int32 [n, m] item ids (-1 pads), cand_val float32 [n, m] their scores, 1 <= k <= m <= MMR_MMAX, diversify in
        [0, 1] -> (int32 [n, k], float32 [n, k]) CUDA tensors, stream-ordered.  The id range check synchronises."""
        import torch
        _dev(cand_idx, "int32", "cand_idx")
        _dev(cand_val, "float32", "cand_val")
        if cand_idx.dim() != 2 or cand_val.shape != cand_idx.shape:
            raise ValueError("cand_idx and cand_val must be [n, m] tensors of one shape")
        n, m = cand_idx.shape
        k = int(k)
        if not 1 <= k <= m <= MMR_MMAX:
            raise ValueError("need 1 <= k <= m <= %d, got k=%d, m=%d" % (MMR_MMAX, k, m))
        if not 0.0 <= float(diversify) <= 1.0:
            raise ValueError("diversify must be in [0, 1], got %r" % (diversify,))
        if self._d is None:
            raise ValueError("set the items before reranking")
        if n and cand_idx.numel():
            lo, hi = torch.aminmax(cand_idx)
            if int(lo.item()) < -1 or int(hi.item()) >= self.num_items:
                raise ValueError("cand_idx holds an id outside [-1, %d)" % self.num_items)
        idx = torch.empty((n, k), dtype=torch.int32, device=cand_idx.device)
        val = torch.empty((n, k), dtype=torch.float32, device=cand_idx.device)
        _cabi.check(self._lib.bfl_mmr_rerank_device(self._h, cand_idx.data_ptr(), cand_val.data_ptr(), n, m, k,
                                                    float(diversify), idx.data_ptr(), val.data_ptr(),
                                                    _stream_ptr(stream)), "bfl_mmr_rerank_device")
        return idx, val

    @staticmethod
    def _check_rows(row, n, rows, what):
        """row: None (query q reads row q: the CSR needs n rows) or int32 CUDA [n] row numbers inside the CSR."""
        if row is None:
            if rows != n:
                raise ValueError("without %s_row the %s CSR needs one row per query" % (what, what))
            return None
        _dev(row, "int32", what + "_row")
        if row.shape[0] != n:
            raise ValueError("%s_row must name one row per query" % what)
        if n and (int(row.min().item()) < 0 or int(row.max().item()) >= rows):
            raise ValueError("%s_row names a row outside the %s CSR" % (what, what))
        return row

    def _set_cand_budget(self, entries):
        """Test hook: list entries per internal batch of topk_candidates (0: the default)."""
        _cabi.check(self._lib.bfl_cand_set_budget(self._h, int(entries)), "bfl_cand_set_budget")


def csr_from_triples_device(major, minor, vals, num_major, num_minor, sort_minor=True, stream=None):
    """(indptr_end int64, key int32, val float32) torch CUDA tensors of one orientation from int32 major / minor and
    float32 vals CUDA tensors, through the device radix sort (bfl_csr_from_triples_device)."""
    import torch
    n, dev = int(major.shape[0]), major.device
    indptr = torch.empty(int(num_major), dtype=torch.int64, device=dev)
    key = torch.empty(max(n, 1), dtype=torch.int32, device=dev)
    val = torch.empty(max(n, 1), dtype=torch.float32, device=dev)
    _cabi.check(_cabi.lib().bfl_csr_from_triples_device(
        _dev(major, "int32", "major") if n else None, _dev(minor, "int32", "minor") if n else None,
        _dev(vals, "float32", "vals") if n else None, n, int(num_major), int(max(num_minor, 1)), int(bool(sort_minor)),
        indptr.data_ptr(), key.data_ptr(), val.data_ptr(), _stream_ptr(stream)), "bfl_csr_from_triples_device")
    return indptr, key[:n], val[:n]


def category_table_slots(topk):
    """Slots of a row's (category, count) table in category_walk_device's state: a power of two >= max(32, 2 topk)."""
    return 1 << max(5, (2 * int(topk) - 1).bit_length())


def category_walk_device(cand_idx, cand_val, rows, categories, caps, topk, state, out_idx, out_val, stream=None):
    """One round of the per-category cap walk (bfl_category_walk_device) on torch CUDA tensors: candidate row r (int32
    cand_idx / float32 cand_val [n, m], best first, -1 skipped) continues the walk of state / output row rows[r] (int32
    [n], or None: row r).  categories int32 [num_items] in [-1, C); caps an int (one cap for every category) or int32
    [C]; state int32 [R, 1 + 2 category_table_slots(topk)] zero-filled before the first round; out_idx / out_val [R,
    topk] filled with -1 / 0.0 before it.  Stream-ordered."""
    n, m = cand_idx.shape
    slots = category_table_slots(topk)
    if cand_val.shape != cand_idx.shape or state.shape[1] != 1 + 2 * slots or out_idx.shape[1] != topk \
            or out_val.shape != out_idx.shape or state.shape[0] != out_idx.shape[0]:
        raise ValueError("category walk: inconsistent shapes")
    if rows is not None and rows.shape[0] != n:
        raise ValueError("category walk: rows must name one row per candidate row")
    scalar = isinstance(caps, (int, np.integer))
    _cabi.check(_cabi.lib().bfl_category_walk_device(
        _dev(cand_idx, "int32", "cand_idx"), _dev(cand_val, "float32", "cand_val"), n, m,
        None if rows is None else _dev(rows, "int32", "rows"), _dev(categories, "int32", "categories"),
        None if scalar else _dev(caps, "int32", "caps"), int(caps) if scalar else 0, int(topk), slots,
        _dev(state, "int32", "state"), _dev(out_idx, "int32", "out_idx"), _dev(out_val, "float32", "out_val"),
        _stream_ptr(stream)), "bfl_category_walk_device")


def eval_unsorted_rows(indptr, keys, stream=None):
    """Number of rows of a device CSR (END offsets) whose keys are not non-decreasing; synchronises."""
    import torch
    count = torch.zeros(1, dtype=torch.int64, device=indptr.device)
    _cabi.check(_cabi.lib().bfl_eval_unsorted_rows_device(_dev(indptr, "int64", "indptr"), _dev(keys, "int32", "keys"),
                                                          indptr.shape[0], count.data_ptr(), _stream_ptr(stream)),
                "bfl_eval_unsorted_rows_device")
    return int(count.item())


def eval_topk_masked(queries, items, item_bias, k, seen_indptr, seen_keys, seen_row, stream=None):
    """int32 [nq, k] device tensor: per query, the k best items (scores of bfl_topk_device) outside seen row
    seen_row[q] of the device CSR (seen_indptr END offsets, sorted seen_keys); -1 pads."""
    import torch
    nq = queries.shape[0]
    idx = torch.empty((nq, int(k)), dtype=torch.int32, device=queries.device)
    _cabi.check(_cabi.lib().bfl_eval_topk_masked_device(
        _dev(queries, "float32", "queries"), nq, queries.stride(0), _dev(items, "float32", "items"), items.shape[0],
        items.stride(0), None if item_bias is None else _dev(item_bias, "float32", "bias"),
        int(min(queries.shape[1], items.shape[1])), int(k), _dev(seen_indptr, "int64", "seen_indptr"),
        _dev(seen_keys, "int32", "seen_keys"), _dev(seen_row, "int32", "seen_row"), idx.data_ptr(), _stream_ptr(stream)),
        "bfl_eval_topk_masked_device")
    return idx


def eval_ranking_terms(ranked, users, seen_indptr, seen_row, gt_indptr, gt_keys, gains, ideal, num_items, terms,
                       stream=None):
    """Fills the float64 [nq, 6] device tensor `terms` with the per-row ranking terms of bfl_eval_ranking_terms_device."""
    nq, k = ranked.shape
    if terms.shape != (nq, 6):
        raise ValueError("terms must be [%d, 6], got %s" % (nq, tuple(terms.shape)))
    _cabi.check(_cabi.lib().bfl_eval_ranking_terms_device(
        _dev(ranked, "int32", "ranked"), nq, k, _dev(users, "int32", "users"), _dev(seen_indptr, "int64", "seen_indptr"),
        _dev(seen_row, "int32", "seen_row"), _dev(gt_indptr, "int64", "gt_indptr"), _dev(gt_keys, "int32", "gt_keys"),
        _dev(gains, "float64", "gains"), _dev(ideal, "float64", "ideal"), int(num_items), _dev(terms, "float64", "terms"),
        _stream_ptr(stream)), "bfl_eval_ranking_terms_device")


EVAL_SCORE_MODES = {"dot": 0, "dot_bias": 1, "l2": 2}


def eval_score_terms(P, Q, Qb, mode, rows, cols, vals, stream=None):
    """float64 [n, 2] device tensor of (err^2, |err|) per held-out triple (bfl_eval_score_terms_device); P, Q rows of
    the same width, mode one of EVAL_SCORE_MODES."""
    import torch
    if P.shape[1] != Q.shape[1]:
        raise ValueError("P and Q must have the same width (got %d, %d)" % (P.shape[1], Q.shape[1]))
    n = rows.shape[0]
    terms = torch.empty((n, 2), dtype=torch.float64, device=P.device)
    _cabi.check(_cabi.lib().bfl_eval_score_terms_device(
        _dev(P, "float32", "P"), _dev(Q, "float32", "Q"), None if Qb is None else _dev(Qb, "float32", "Qb"), P.shape[1],
        EVAL_SCORE_MODES[mode], _dev(rows, "int32", "rows"), _dev(cols, "int32", "cols"), _dev(vals, "float32", "vals"), n,
        terms.data_ptr(), _stream_ptr(stream)), "bfl_eval_score_terms_device")
    return terms


def eval_sum(terms, stream=None):
    """Column sums (float64 numpy array) of a float64 [n, width <= 8] device tensor, in a fixed order."""
    import torch
    out = torch.empty(terms.shape[1], dtype=torch.float64, device=terms.device)
    _cabi.check(_cabi.lib().bfl_eval_sum_device(_dev(terms, "float64", "terms") if terms.shape[0] else None,
                                                terms.shape[0], terms.shape[1], out.data_ptr(), _stream_ptr(stream)),
                "bfl_eval_sum_device")
    return out.cpu().numpy()


EVAL_ILD_KMAX = 256


def eval_cutoff_terms(ranked, truth_indptr, truth_keys, truth_row, cutoffs, gains, ideal, terms, stream=None):
    """Writes rows of the float64 [n_cut, rows, 8] device tensor `terms` (its row q for ranked row q; pass a view such as
    terms[:, s:s + n]) with bfl_eval_cutoff_terms_device's columns 0-7 for the int32 [n, k] ranked lists.  cutoffs: int32
    device tensor, ascending and distinct, each in [1, k]; truth_row: int32 device tensor or None (row q)."""
    n, k = ranked.shape
    if terms.dim() != 3 or terms.shape[0] != cutoffs.shape[0] or terms.shape[1] != n or terms.shape[2] != 8 \
            or terms.stride(1) != 8 or terms.stride(2) != 1:
        raise ValueError("terms must be a [%d, %d, 8] view with contiguous rows, got %s"
                         % (cutoffs.shape[0], n, tuple(terms.shape)))
    _cabi.check(_cabi.lib().bfl_eval_cutoff_terms_device(
        _dev(ranked, "int32", "ranked"), n, k, _dev(truth_indptr, "int64", "truth_indptr"),
        _dev(truth_keys, "int32", "truth_keys"), None if truth_row is None else _dev(truth_row, "int32", "truth_row"),
        _dev(cutoffs, "int32", "cutoffs"), cutoffs.shape[0], _dev(gains, "float64", "gains"),
        _dev(ideal, "float64", "ideal"), terms.data_ptr(), terms.stride(0), _stream_ptr(stream)),
        "bfl_eval_cutoff_terms_device")


def eval_ild(ranked, kmax, items, cutoffs, terms, stream=None):
    """Columns 6-7 of eval_cutoff_terms' `terms` view: intra-list diversity over the rows of the contiguous float32
    [n_items, d] device tensor `items`; kmax = the largest cutoff (<= EVAL_ILD_KMAX)."""
    n, k = ranked.shape
    if terms.dim() != 3 or terms.shape[:2] != (cutoffs.shape[0], n) or terms.stride(1) != 8 or terms.stride(2) != 1:
        raise ValueError("terms must be a [%d, %d, 8] view with contiguous rows" % (cutoffs.shape[0], n))
    if items.dim() != 2:
        raise ValueError("items must be a [n_items, d] tensor")
    _cabi.check(_cabi.lib().bfl_eval_ild_device(
        _dev(ranked, "int32", "ranked"), n, k, int(kmax), _dev(items, "float32", "items"), items.shape[1],
        items.shape[1], _dev(cutoffs, "int32", "cutoffs"), cutoffs.shape[0], terms.data_ptr(), terms.stride(0),
        _stream_ptr(stream)), "bfl_eval_ild_device")


def eval_coverage_mark(ranked, bucket, first, stream=None):
    """first[item] = min(first[item], bucket[p]) over the entries at positions p < len(bucket) of the int32 [n, k] lists."""
    n, k = ranked.shape
    _cabi.check(_cabi.lib().bfl_eval_coverage_mark_device(
        _dev(ranked, "int32", "ranked"), n, k, _dev(bucket, "int32", "bucket"), bucket.shape[0],
        _dev(first, "int32", "first"), _stream_ptr(stream)), "bfl_eval_coverage_mark_device")


def eval_coverage_count(first, n_cut, stream=None):
    """int64 numpy [n_cut]: the number of items whose `first` entry is c, for each c < n_cut."""
    import torch
    count = torch.empty(int(n_cut), dtype=torch.int64, device=first.device)
    _cabi.check(_cabi.lib().bfl_eval_coverage_count_device(_dev(first, "int32", "first"), first.shape[0], int(n_cut),
                                                           count.data_ptr(), _stream_ptr(stream)),
                "bfl_eval_coverage_count_device")
    return count.cpu().numpy()


def csr_from_triples_host(major, minor, vals, num_major, num_minor, sort_minor=True):
    """(indptr_end int64, key int32, val float32) of one orientation through the hand-written device radix sort
    (csrc/ingest.cu: bfl_csr_from_triples_host)."""
    mj = np.ascontiguousarray(major, dtype=np.int32)
    mn = np.ascontiguousarray(minor, dtype=np.int32)
    v = np.ascontiguousarray(vals, dtype=np.float32)
    n = len(mj)
    indptr = np.empty(int(num_major), dtype=np.int64)
    key = np.empty(max(n, 1), dtype=np.int32)
    val = np.empty(max(n, 1), dtype=np.float32)
    _cabi.check(_cabi.lib().bfl_csr_from_triples_host(mj.ctypes.data, mn.ctypes.data, v.ctypes.data, n, int(num_major),
                                                      int(max(num_minor, 1)), int(bool(sort_minor)), indptr.ctypes.data,
                                                      key.ctypes.data, val.ctypes.data), "bfl_csr_from_triples_host")
    return indptr, key[:n], val[:n]


class _TextIngest(object):
    """Handle of a device text parser (bfl_<prefix>_*): the text is fed through two pinned staging buffers of
    block_bytes, then the CSR groups are built on the device and copied out.  STAGES names the entries of stats()."""

    STAGES = ()

    def __init__(self, prefix, block_bytes, *create_args):
        self._lib = _cabi.lib()
        self._prefix = prefix
        self._h = self._fn("create")(*create_args)
        if not self._h:
            err = self._lib.bfl_last_error().decode("utf-8", "replace")
            raise _cabi.BackendError("bfl_%s_create failed: %s" % (prefix, err))
        self.block_bytes = int(block_bytes)

    def _fn(self, name):
        return getattr(self._lib, "bfl_%s_%s" % (self._prefix, name))

    def _call(self, name, *args):
        _cabi.check(self._fn(name)(self._h, *args), "bfl_%s_%s" % (self._prefix, name))

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._fn("destroy")(h)

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def staging(self, slot):
        """uint8 view of pinned staging buffer `slot`, free for writing (its previous upload has finished)."""
        p = C.c_void_p()
        self._call("staging", int(slot), C.byref(p))
        return np.ctypeslib.as_array((C.c_uint8 * self.block_bytes).from_address(p.value))

    def feed(self, slot, n, is_last):
        self._call("feed", int(slot), int(n), int(bool(is_last)))

    def build(self, orientation, num_major, nnz):
        """-> (indptr int64[num_major] END offsets, key int32[nnz], val float32[nnz]); 0 = rowwise, 1 = colwise"""
        indptr = np.empty(int(num_major), np.int64)
        key, val = np.empty(max(nnz, 1), np.int32), np.empty(max(nnz, 1), np.float32)
        self._call("build", int(orientation), indptr.ctypes.data, key.ctypes.data, val.ctypes.data)
        return indptr, key[:nnz], val[:nnz]

    def stats(self):
        """-> ({stage: device ms}, peak device bytes of the default memory pool)"""
        ms, peak = (C.c_double * len(self.STAGES))(), C.c_int64(0)
        self._call("stats", ms, C.byref(peak))
        return dict(zip(self.STAGES, list(ms))), peak.value


class MMIngest(_TextIngest):
    """Handle of the device MatrixMarket parser (csrc/mm_ingest.cu, bfl_mm_ingest_*): stream the text after the header
    through two pinned staging buffers, then split and build both CSR orientations on the device."""

    STAGES = ("h2d", "parse", "patch", "split", "csr_rowwise", "csr_colwise", "d2h")

    def __init__(self, num_rows, num_cols, nnz_hint, block_bytes, header_lines, slow_cap):
        super().__init__("mm_ingest", block_bytes, int(num_rows), int(num_cols), int(nnz_hint), int(block_bytes),
                         int(header_lines), int(slow_cap))

    def finish(self):
        """-> dict(nnz, tokmask, reject_line, range_line, n_slow)"""
        v = [C.c_int64(0), C.c_int32(0), C.c_int64(0), C.c_int64(0), C.c_int64(0)]
        self._call("finish", *[C.byref(x) for x in v])
        return dict(zip(("nnz", "tokmask", "reject_line", "range_line", "n_slow"), [x.value for x in v]))

    def slow_tokens(self, n):
        """-> (ordinal int64, offset from the first fed byte int64, length int32) of n slow value tokens"""
        o, off, ln = np.empty(n, np.int64), np.empty(n, np.int64), np.empty(n, np.int32)
        self._call("slow_tokens", int(n), o.ctypes.data, off.ctypes.data, ln.ctypes.data)
        return o, off, ln

    def patch_values(self, ordinal, vals):
        o = np.ascontiguousarray(ordinal, dtype=np.int64)
        v = np.ascontiguousarray(vals, dtype=np.float32)
        self._call("patch_values", o.ctypes.data, v.ctypes.data, len(o))

    def split(self, sample_idx):
        """-> (row int32, col int32, val float32) of the sampled data-line ordinals (strictly increasing)"""
        idx = np.ascontiguousarray(sample_idx, dtype=np.int64)
        n = len(idx)
        r, c, v = np.empty(n, np.int32), np.empty(n, np.int32), np.empty(n, np.float32)
        self._call("split", idx.ctypes.data, n, r.ctypes.data, c.ctypes.data, v.ctypes.data)
        return r, c, v


class StreamIngest(_TextIngest):
    """Handle of the device Stream parser (csrc/stream_ingest.cu, bfl_stream_ingest_*): stream the text through two
    pinned staging buffers, intern the item tokens on the device, then split and build the CSR groups there."""

    STAGES = ("h2d", "parse", "intern", "number", "split", "csr_rowwise", "csr_colwise", "d2h")

    def __init__(self, block_bytes, whitespace, hash_bits=64):
        ascii_ws = sum(1 << c for c in whitespace if c < 64)
        usp = np.ascontiguousarray([c for c in whitespace if c >= 0x80], dtype=np.int32)
        super().__init__("stream_ingest", block_bytes, int(block_bytes), ascii_ws, usp.ctypes.data, len(usp),
                         int(hash_bits))

    def load_iid(self, names):
        """names: list of bytes (UTF-8 item names, in id order)"""
        offs = np.zeros(len(names) + 1, np.int64)
        np.cumsum([len(x) for x in names], out=offs[1:])
        buf = np.frombuffer(b"".join(names) or b"\0", np.uint8)
        self._call("load_iid", buf.ctypes.data, offs.ctypes.data, len(names))

    def finish(self):
        """-> dict(tokens, lines, items, decline, decline_line)"""
        v = [C.c_int64(0), C.c_int64(0), C.c_int32(0), C.c_int32(0), C.c_int64(0)]
        self._call("finish", *[C.byref(x) for x in v])
        return dict(zip(("tokens", "lines", "items", "decline", "decline_line"), [x.value for x in v]))

    def names(self, n):
        """-> (offset int64, length int32) of the first occurrence of each of the n items"""
        off, ln = np.empty(max(n, 1), np.int64), np.empty(max(n, 1), np.int32)
        self._call("names", off.ctypes.data, ln.ctypes.data)
        return off[:n], ln[:n]

    def split(self, num_users, method, newest_n, sample_idx, as_matrix):
        """method: 0 none, 1 newest, 2 sample -> (n_train, (row int32, col int32, val float32) of the vali triples)"""
        idx = np.ascontiguousarray(sample_idx, dtype=np.int64)
        nv, nt = C.c_int64(0), C.c_int64(0)
        self._call("split", int(num_users), int(method), int(newest_n), idx.ctypes.data, len(idx), int(bool(as_matrix)),
                   C.byref(nv), C.byref(nt))
        n = nv.value
        r, c, v = np.empty(max(n, 1), np.int32), np.empty(max(n, 1), np.int32), np.empty(max(n, 1), np.float32)
        self._call("vali", r.ctypes.data, c.ctypes.data, v.ctypes.data)
        return nt.value, (r[:n], c[:n], v[:n])


def device_free_bytes():
    """Free device memory of the current device (cudaMemGetInfo)."""
    import torch
    return int(torch.cuda.mem_get_info()[0])


def popularity_table_host(keys, n_items, power):
    """int64 cumulative table of count(item)**power (bpr.py:99-111) built on the device."""
    k = np.ascontiguousarray(keys, dtype=np.int32)
    cum = np.empty(int(n_items), dtype=np.int64)
    _cabi.check(_cabi.lib().bfl_popularity_table_host(k.ctypes.data, len(k), int(n_items), int(power), cum.ctypes.data),
                "bfl_popularity_table_host")
    return cum

IVF_MAX_LISTS = 65536
IVF_DMAX = 256


class IVF(object):
    """Inverted-file index (csrc/ivf.cu, bfl_ivf_*, DESIGN.md 4.12): the rows clustered by spherical k-means into nlist
    lists; search scores each query against the rows of its nprobe best lists only, with the scores and ranking of
    Serve.topk, so nprobe = nlist gives Serve.topk's result bit for bit.  GPU only: build and search raise the
    library's "no CPU fallback" error without one."""

    def __init__(self):
        self._lib = _cabi.lib()
        self._h = self._lib.bfl_ivf_create()
        if not self._h:
            raise MemoryError("bfl_ivf_create")
        self.nlist = 0
        self.num_rows = 0
        self.has_bias = False

    def close(self):
        h, self._h = getattr(self, "_h", None), None
        if h:
            self._lib.bfl_ivf_destroy(h)

    __del__ = close

    def _attach(self):
        _cabi.check(self._lib.bfl_ivf_attach(self._h), "bfl_ivf_attach")

    def build(self, rows, bias=None, nlist=1024, iters=10, seed=0):
        """rows float32 [n, d] host array (C-contiguous), bias float32 [n] or None.  Replaces any earlier index."""
        _host(rows, np.float32, 2, "rows")
        n, d = rows.shape
        nlist, iters = int(nlist), int(iters)
        if not 1 <= nlist <= min(n, IVF_MAX_LISTS):
            raise ValueError("nlist must be in [1, min(rows, %d)] = [1, %d]" % (IVF_MAX_LISTS, min(n, IVF_MAX_LISTS)))
        if iters < 1:
            raise ValueError("iters must be at least 1")
        if not 0 < d <= IVF_DMAX:
            raise ValueError("the index holds rows of 1 to %d floats, got %d" % (IVF_DMAX, d))
        if bias is not None:
            bias = np.ascontiguousarray(np.asarray(bias, dtype=np.float32).reshape(-1))
            if bias.shape[0] != n:
                raise ValueError("bias must have one value per row")
        self._attach()
        import torch
        dr = torch.from_numpy(rows).cuda()
        db = None if bias is None else torch.from_numpy(bias).cuda()
        torch.cuda.synchronize()
        self.nlist = self.num_rows = 0
        _cabi.check(self._lib.bfl_ivf_build_device(self._h, dr.data_ptr(), n, d, d, None if db is None else db.data_ptr(),
                                                   nlist, iters, int(seed) & (2 ** 64 - 1)), "bfl_ivf_build_device")
        self.nlist, self.num_rows, self.d, self.has_bias = nlist, n, d, bias is not None

    def _check_nprobe(self, nprobe):
        if isinstance(nprobe, bool) or not isinstance(nprobe, (int, np.integer)):
            raise ValueError("nprobe must be an integer")
        nprobe = int(nprobe)
        if not 1 <= nprobe <= self.nlist:
            raise ValueError("nprobe must be in [1, nlist=%d]" % self.nlist)
        if nprobe > SERVE_KMAX and nprobe != self.nlist:
            raise ValueError("nprobe above %d must be nlist=%d" % (SERVE_KMAX, self.nlist))
        return nprobe

    def search_device(self, queries, nprobe, k, use_bias=False, stream=None):
        """queries: torch float32 CUDA tensor [n, >= d] -> (int32 [n, k] row ids, float32 [n, k] scores) CUDA tensors."""
        import torch
        nprobe, k = self._check_nprobe(nprobe), Serve._check_k(k)
        n = queries.shape[0]
        idx = torch.empty((n, k), dtype=torch.int32, device=queries.device)
        val = torch.empty((n, k), dtype=torch.float32, device=queries.device)
        if n:
            _cabi.check(self._lib.bfl_ivf_search_device(self._h, _dev(queries, "float32", "queries"), n,
                                                        queries.stride(0), nprobe, k, int(bool(use_bias)),
                                                        idx.data_ptr(), val.data_ptr(), _stream_ptr(stream)),
                        "bfl_ivf_search_device")
        return idx, val

    def search(self, queries, nprobe, k, use_bias=False):
        """queries float32 [n, >= d] host array -> (int32 [n, k], float32 [n, k]) host arrays: best first, ties to the
        smaller row id, -1 / 0.0 where the probed lists hold fewer than k rows."""
        _host(queries, np.float32, 2, "queries")
        nprobe, k = self._check_nprobe(nprobe), Serve._check_k(k)
        self._attach()
        if queries.shape[0] == 0:
            return np.zeros((0, k), np.int32), np.zeros((0, k), np.float32)
        import torch
        idx, val = self.search_device(torch.from_numpy(queries).cuda(), nprobe, k, use_bias)
        return idx.cpu().numpy(), val.cpu().numpy()

    def _set_batch_rows(self, rows):
        """Queries per internal batch at most (0: automatic); lets tests cross batch edges at small sizes."""
        _cabi.check(self._lib.bfl_ivf_set_batch_rows(self._h, int(rows)), "bfl_ivf_set_batch_rows")

    def _read(self, what):
        n, nl, ld, d = C.c_int64(0), C.c_int(0), C.c_int(0), C.c_int(0)
        _cabi.check(self._lib.bfl_ivf_info(self._h, C.byref(n), C.byref(nl), C.byref(ld), C.byref(d)), "bfl_ivf_info")
        out = {"centroids": np.empty((nl.value, ld.value), np.float32), "offsets": np.empty(nl.value, np.int64),
               "ids": np.empty(n.value, np.int32)}[what]
        args = [out.ctypes.data if w == what else None for w in ("centroids", "offsets", "ids")]
        _cabi.check(self._lib.bfl_ivf_read(self._h, *args), "bfl_ivf_read")
        return out[:, :d.value] if what == "centroids" else out

    def centroids(self):
        """float32 [nlist, d]: the unit centroids."""
        return self._read("centroids")

    def offsets(self):
        """int64 [nlist]: END offsets of the lists into ids()."""
        return self._read("offsets")

    def ids(self):
        """int32 [n]: the row ids of every list, list after list, ascending within a list."""
        return self._read("ids")

    def nbytes(self):
        """Device bytes of the index: centroids, offsets, ids, list-major rows and bias, chunk counts."""
        return (self.nlist * self.d * 4 + self.nlist * 8 + self.num_rows * 4 + self.num_rows * self.d * 4
                + (self.num_rows * 4 if self.has_bias else 0) + self.nlist * 4)

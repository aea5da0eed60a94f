"""Folding-in (DESIGN.md 4.10): the host side that ALS.fold_in, PLSI.fold_in and ALS.explain (4.11) share.

A fold-in computes user rows from their histories with the model's item factors held fixed.  This module turns the
caller's histories and start rows into checked host arrays (before any device work), keeps the model's item factors on
the device, padded to the holder's row pitch and uploaded again only when their bits change, and moves one call's
histories to the device as one CSR.  The solves themselves are the models' (als.py, plsi.py)."""
import json

import numpy as np
import scipy.sparse


def history_csr(algo, histories, num_items):
    """(END offsets int64 [n], keys int32, vals float32) host arrays of the histories:
      * a scipy sparse (n, num_items) matrix, read after tocsr() / sort_indices() (on a copy: the caller's matrix is not
        changed), so each row's entries are in ascending item order; values in the units of the training data;
      * or a list of n lists of item ids, mapped through the model's item-id map; unknown ids are dropped, every entry
        has the value 1.0 and each row is put in ascending item order.
    Raises ValueError on a wrong column count, a key outside [0, num_items) or another input type."""
    if scipy.sparse.issparse(histories):
        if histories.ndim != 2 or histories.shape[1] != num_items:
            raise ValueError("histories must be an (n, %d) matrix, got %s" % (num_items, histories.shape))
        m = histories.tocsr(copy=True)
        m.sort_indices()
        nnz = int(m.indptr[-1])
        keys = np.asarray(m.indices[:nnz])
        if keys.size and (int(keys.min()) < 0 or int(keys.max()) >= num_items):
            raise ValueError("histories hold an item outside [0, %d)" % num_items)
        return (np.ascontiguousarray(m.indptr[1:], dtype=np.int64), np.ascontiguousarray(keys, dtype=np.int32),
                np.ascontiguousarray(m.data[:nnz], dtype=np.float32))
    if not isinstance(histories, (list, tuple)):
        raise ValueError("histories must be a scipy sparse matrix or a list of lists of item ids, got %s"
                         % type(histories).__name__)
    rows = []
    for h in histories:
        if not isinstance(h, (list, tuple, np.ndarray)):
            raise ValueError("every history must be a list of item ids, got %s" % type(h).__name__)
        idx = algo.get_index(list(h), group="item") if len(h) else []
        rows.append(np.sort(np.array([i for i in idx if i is not None], dtype=np.int64), kind="stable"))
    lens = np.array([len(r) for r in rows], dtype=np.int64)
    keys = np.concatenate(rows).astype(np.int32) if rows else np.zeros(0, np.int32)
    return np.cumsum(lens).astype(np.int64), keys, np.ones(len(keys), dtype=np.float32)


def target_matrix(algo, items, n, num_items, kmax):
    """int32 (n, k) item indexes, -1 for no target, of explanation targets given as
      * an (n, k) integer array of item indexes in [-1, num_items) (the shape ParALS.topk_recommendation returns),
      * or n lists of item ids, mapped through the model's item-id map; unknown ids become -1 and the rows are padded
        with -1 to the longest.
    Raises ValueError on a wrong shape, an index out of range, k > kmax or another input type."""
    if isinstance(items, np.ndarray):
        if items.ndim != 2 or items.shape[0] != n or not np.issubdtype(items.dtype, np.integer):
            raise ValueError("items must be an (%d, k) integer array, got %s %s" % (n, items.dtype, items.shape))
        if items.size and (int(items.min()) < -1 or int(items.max()) >= num_items):
            raise ValueError("items hold an index outside [-1, %d)" % num_items)
        T = np.ascontiguousarray(items, dtype=np.int32)
    elif isinstance(items, (list, tuple)):
        if len(items) != n:
            raise ValueError("items must hold one list per history row (%d), got %d" % (n, len(items)))
        k = 0
        for it in items:
            if not isinstance(it, (list, tuple, np.ndarray)):
                raise ValueError("every row of items must be a list of item ids, got %s" % type(it).__name__)
            k = max(k, len(it))
        T = np.full((n, k), -1, dtype=np.int32)
        for r, it in enumerate(items):
            idx = algo.get_index(list(it), group="item") if len(it) else []
            T[r, :len(idx)] = [-1 if i is None else i for i in idx]
    else:
        raise ValueError("items must be an (n, k) integer array or a list of lists of item ids, got %s"
                         % type(items).__name__)
    if T.shape[1] > kmax:
        raise ValueError("at most %d targets per row, got %d" % (kmax, T.shape[1]))
    return T


def start_rows(init, n, d, fill):
    """float32 (n, d) start rows: `fill` everywhere when init is None, else init (ValueError unless its shape is (n, d))."""
    if init is None:
        return np.full((n, d), fill, dtype=np.float32)
    X = np.asarray(init, dtype=np.float32)
    if X.shape != (n, d):
        raise ValueError("init must be (%d, %d), got %s" % (n, d, X.shape))
    return X


def positive_int(value, name):
    if isinstance(value, bool) or not isinstance(value, (int, np.integer)) or value < 1:
        raise ValueError("%s must be an integer >= 1, got %r" % (name, value))
    return int(value)


class ItemState(object):
    """A model's fold-in state on the device: a backend holder of its own, made from the model's options, and the item
    factors Q padded to the holder's row pitch (padding columns zero).  `key` is the checksum of Q's bits (the rule of
    Parallel._fingerprint) and the options; refresh() uploads Q again, and marks derived data such as the ALS Gram
    stale, when either changed: normalize(), a second train() or an in-place edit."""

    def __init__(self):
        self.key = self.okey = self.holder = self.Q = None
        self.derived_key = None          # key the holder's derived item data (the ALS Gram) was computed for

    @staticmethod
    def make_holder(make, opt):
        holder = make()
        if not holder.init(dict(opt)):
            raise ValueError("fold_in: the model's options were refused: %s" % getattr(holder, "last_error", ""))
        return holder

    def refresh(self, make, opt, Q):
        """make: the holder class; returns the holder.  Without a GPU, creating the holder raises the backend's
        "no CPU fallback" error."""
        from buffalo_b200.parallel.base import Parallel
        okey = json.dumps(opt, sort_keys=True, default=str)
        if self.holder is None or self.okey != okey:
            self.holder, self.okey, self.key, self.derived_key, self.Q = self.make_holder(make, opt), okey, None, None, None
        key = Parallel._fingerprint(np.ascontiguousarray(Q, dtype=np.float32))
        if self.key != key:
            import torch
            vdim, d = self.holder.get_vdim(), int(opt["d"])
            self.Q, self.key = None, None
            T = torch.zeros((Q.shape[0], vdim), dtype=torch.float32, device=device())
            T[:, :d] = torch.from_numpy(np.ascontiguousarray(Q[:, :d], dtype=np.float32)).to(T.device)
            self.Q, self.key = T, key
        return self.holder


def begin(model, make, histories, init, fill):
    """The common start of a model's fold-in: the checked host input (histories, start rows filled with `fill` when
    init is None), then the model's ItemState refreshed for its current Q with a holder from `make`, and the call's
    device arrays.  Returns (state, holder, (indptr, keys, vals, X) as to_device gives them)."""
    indptr, keys, vals = history_csr(model, histories, model.Q.shape[0])
    X0 = start_rows(init, len(indptr), model.opt.d, fill)
    st, h = item_state(model, make)
    return st, h, to_device(indptr, keys, vals, X0, h.get_vdim())


def item_state(model, make):
    """(the model's ItemState, its holder), refreshed for the model's current Q and options."""
    if getattr(model, "_fold_state", None) is None:
        model._fold_state = ItemState()
    st = model._fold_state
    return st, st.refresh(make, model.opt, model.Q)


def device():
    import torch
    return torch.device("cuda", torch.cuda.current_device())


def to_device(indptr, keys, vals, X0, vdim):
    """(indptr, keys, vals, X) torch CUDA tensors; keys / vals have at least one element, X is [n, vdim] with the start
    rows in its first d columns and zero padding."""
    import torch
    X = torch.zeros((X0.shape[0], vdim), dtype=torch.float32, device=device())
    X[:, :X0.shape[1]] = torch.from_numpy(np.ascontiguousarray(X0)).to(X.device)
    return csr_to_device(indptr, keys, vals) + (X,)


def csr_to_device(indptr, keys, vals):
    """(indptr, keys, vals) torch CUDA tensors; keys / vals have at least one element."""
    import torch
    dev = device()
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    if not len(keys):
        keys, vals = np.zeros(1, np.int32), np.zeros(1, np.float32)
    return t(indptr), t(keys), t(vals)

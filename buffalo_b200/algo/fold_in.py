"""Folding-in (DESIGN.md 4.10, 4.16): the host side that ALS.fold_in, PLSI.fold_in, ALS.explain (4.11),
ALS.posterior_sample (4.17) and the item fold-ins (ALS / BPRMF / WARP .fold_in_items) share.

A user fold-in computes user rows from their histories with the model's item factors held fixed; an item fold-in
computes item rows from the users who interacted with them, with the user factors held fixed.  This module turns the
caller's histories and start rows into checked host arrays (before any device work), keeps the fixed side's factors on
the device, padded to the holder's row pitch and uploaded again only when their bits change, and moves one call's
histories to the device as one CSR.  The solves themselves are the models' (als.py, plsi.py, bpr.py)."""
import json

import numpy as np
import scipy.sparse


def history_csr(algo, histories, num_items, group="item"):
    """(END offsets int64 [n], keys int32, vals float32) host arrays of the histories; `group` is what the columns are
    ("item" for user fold-in, "user" for item fold-in, where num_items is the number of users):
      * a scipy sparse (n, num_items) matrix, read after tocsr() / sort_indices() (on a copy: the caller's matrix is not
        changed), so each row's entries are in ascending column order; values in the units of the training data;
      * or a list of n lists of ids, mapped through the model's id map of `group`; unknown ids are dropped, every entry
        has the value 1.0 and each row is put in ascending column order.
    Raises ValueError on a wrong column count, a key outside [0, num_items) or another input type."""
    if scipy.sparse.issparse(histories):
        if histories.ndim != 2 or histories.shape[1] != num_items:
            raise ValueError("histories must be an (n, %d) matrix, got %s" % (num_items, histories.shape))
        m = histories.tocsr(copy=True)
        m.sort_indices()
        nnz = int(m.indptr[-1])
        keys = np.asarray(m.indices[:nnz])
        if keys.size and (int(keys.min()) < 0 or int(keys.max()) >= num_items):
            raise ValueError("histories hold a%s %s outside [0, %d)" % ("n" if group == "item" else "", group, num_items))
        return (np.ascontiguousarray(m.indptr[1:], dtype=np.int64), np.ascontiguousarray(keys, dtype=np.int32),
                np.ascontiguousarray(m.data[:nnz], dtype=np.float32))
    if not isinstance(histories, (list, tuple)):
        raise ValueError("histories must be a scipy sparse matrix or a list of lists of %s ids, got %s"
                         % (group, type(histories).__name__))
    rows = []
    for h in histories:
        if not isinstance(h, (list, tuple, np.ndarray)):
            raise ValueError("every history must be a list of %s ids, got %s" % (group, type(h).__name__))
        idx = algo.get_index(list(h), group=group) if len(h) else []
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


def posterior_args(scale, seed, scale_name="scale", seed_name="seed"):
    """(float32-rounded scale, seed) of a posterior draw: scale a finite real >= 0, seed an integer in [0, 2^32)."""
    if isinstance(scale, bool) or not isinstance(scale, (int, float, np.integer, np.floating)) \
            or not 0 <= scale <= float(np.finfo(np.float32).max):
        raise ValueError("%s must be a finite real number >= 0, got %r" % (scale_name, scale))
    if isinstance(seed, bool) or not isinstance(seed, (int, np.integer)) or not 0 <= seed < 2 ** 32:
        raise ValueError("%s must be an integer in [0, 2^32), got %r" % (seed_name, seed))
    return float(np.float32(scale)), int(seed)


def draw_key_array(draw_keys, n):
    """int64 [n] draw keys: arange(n) when None, else n distinct non-negative integers (ValueError otherwise)."""
    if draw_keys is None:
        return np.arange(n, dtype=np.int64)
    K = np.asarray(draw_keys)
    if K.shape != (n,) or (K.size and not np.issubdtype(K.dtype, np.integer)):
        raise ValueError("draw_keys must be %d integers, got %s %s" % (n, K.dtype, K.shape))
    K = K.astype(np.int64)
    if K.size and (int(K.min()) < 0 or len(np.unique(K)) != n):
        raise ValueError("draw_keys must be distinct non-negative integers")
    return K


class ItemState(object):
    """A model's fold-in state on the device for one fixed side: a backend holder of its own, made from the model's
    options, and that side's factors F padded to the holder's row pitch (padding columns zero) -- Q for user fold-in, P
    for item fold-in (resident_state).  `key` is the checksum of F's bits (the rule of Parallel._fingerprint) and the
    options; refresh() uploads F again, and marks derived data such as the ALS Gram stale, when either changed:
    normalize(), a second train() or an in-place edit.  F costs rows * vdim * 4 bytes of device memory for as long as
    the model lives (P at 10M users and d = 128: 5 GB)."""

    def __init__(self):
        self.key = self.okey = self.holder = self.F = None
        self.derived_key = None          # key the holder's derived data (the ALS Gram) was computed for
        self.extra = {}                  # name -> (key, device arrays) kept between calls: cached()

    @staticmethod
    def make_holder(make, opt):
        holder = make()
        if not holder.init(dict(opt)):
            raise ValueError("fold_in: the model's options were refused: %s" % getattr(holder, "last_error", ""))
        return holder

    def refresh(self, make, opt, F):
        """make: the holder class; returns the holder.  Without a GPU, creating the holder raises the backend's
        "no CPU fallback" error."""
        okey = json.dumps(opt, sort_keys=True, default=str)
        if self.holder is None or self.okey != okey:
            self.holder, self.okey, self.key, self.derived_key, self.F = self.make_holder(make, opt), okey, None, None, None
            self.extra = {}
        key = fingerprint(F)
        if self.key != key:
            self.F, self.key = None, None
            self.F, self.key = padded(F, self.holder.get_vdim(), int(opt["d"])), key
        return self.holder

    def cached(self, name, key, build):
        """The device arrays build() returns, kept under `name` until a call brings another `key` (or the options
        change)."""
        old = self.extra.pop(name, None)
        if old is not None and old[0] == key:
            self.extra[name] = old
            return old[1]
        value = build()
        self.extra[name] = (key, value)
        return value


def fingerprint(A):
    """Checksum of the bits of A as float32 / its own dtype (the rule of Parallel._fingerprint)."""
    from buffalo_b200.parallel.base import Parallel
    A = np.asarray(A)
    A = np.ascontiguousarray(A, dtype=np.float32) if A.dtype.kind == "f" else np.ascontiguousarray(A)
    return Parallel._fingerprint(A.reshape(A.shape[0], -1) if A.ndim else A.reshape(1, 1))


def padded(F, vdim, d):
    """torch CUDA float32 [rows, vdim]: F's first d columns, zero padding."""
    import torch
    T = torch.zeros((F.shape[0], vdim), dtype=torch.float32, device=device())
    T[:, :d] = torch.from_numpy(np.ascontiguousarray(F[:, :d], dtype=np.float32)).to(T.device)
    return T


def begin(model, make, histories, init, fill, side="Q"):
    """The common start of a model's fold-in: the checked host input (histories, start rows filled with `fill` when
    init is None), then the model's state for the fixed `side` ("Q": user fold-in, "P": item fold-in) refreshed with a
    holder from `make`, and the call's device arrays.  Returns (state, holder, (indptr, keys, vals, X) as to_device
    gives them)."""
    indptr, keys, vals = history_csr(model, histories, *columns(model, side))
    X0 = start_rows(init, len(indptr), model.opt.d, fill)
    st, h = resident_state(model, make, side)
    return st, h, to_device(indptr, keys, vals, X0, h.get_vdim())


def columns(model, side):
    """(column count, id group) of the histories of a fold-in against the fixed `side`."""
    return (model.Q.shape[0], "item") if side == "Q" else (model.P.shape[0], "user")


def resident_state(model, make, side="Q"):
    """(the model's ItemState for the fixed `side`, its holder), refreshed for the model's current factors of that side
    and its options.  The two sides keep separate states: their holders hold different Grams."""
    attr = "_fold_state" if side == "Q" else "_fold_state_items"
    if getattr(model, attr, None) is None:
        setattr(model, attr, ItemState())
    st = getattr(model, attr)
    return st, st.refresh(make, model.opt, model.Q if side == "Q" else model.P)


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

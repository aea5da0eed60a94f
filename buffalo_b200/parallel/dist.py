"""Row-sharded multi-GPU driver for ALS (SURVEY.md 8e): one process per GPU, contiguous user / item row ranges
per rank, full factor replicas everywhere, ONE exchange step per half-epoch -- an in-place all-gather of the
freshly updated factor shard over NCCL (NVLink / NVSwitch).  The same class drives the gloo CPU tests
(tests/test_dist_cpu.py) with a CPU row-update function, so the sharding / exchange logic is covered without GPUs.
"""
import numpy as np


def row_shard(total, rank, world):
    """Equal contiguous pieces (the in-place all-gather needs equal counts); the last pieces may be empty."""
    per = (total + world - 1) // world
    lo = min(rank * per, total)
    return lo, min(lo + per, total), per


def nnz_shard(indptr_end, rank, world):
    """Contiguous row range of `rank` when rows are split so that every rank gets (nearly) the same number of
    nonzeros: boundary k is the first row whose end offset reaches k * nnz / world (SURVEY 8e: prefix-sum split of
    indptr).  `indptr_end` = exclusive end offsets (NumPy array or torch tensor).  Needs an exchange that accepts
    unequal shard sizes (the fused p2p exchange does; the in-place all-gather does not)."""
    n = int(indptr_end.shape[0])
    if n == 0:
        return 0, 0, None
    nnz = int(indptr_end[-1])

    def boundary(k):
        if k <= 0:
            return 0
        if k >= world:
            return n
        target = (nnz * k + world - 1) // world
        if hasattr(indptr_end, "cpu"):   # torch tensor (possibly on the device)
            import torch
            t = torch.tensor([target], dtype=indptr_end.dtype, device=indptr_end.device)
            return int(torch.searchsorted(indptr_end, t, right=False).item()) + 1 if target > 0 else 0
        return int(np.searchsorted(indptr_end, target, side="left")) + 1 if target > 0 else 0
    lo, hi = min(boundary(rank), n), min(boundary(rank + 1), n)
    return lo, max(lo, hi), None


_opened = {}   # IPC handle bytes -> mapped base address (a handle may be opened once per process)
_exportable = {}   # data_ptr -> owner object keeping the cudaMalloc buffer alive


class _DevBuffer(object):
    """A plain cudaMalloc buffer owned by the C library (its IPC handle refers to exactly this buffer), exposed to
    torch through __cuda_array_interface__."""

    def __init__(self, shape):
        from buffalo_b200 import _cabi
        self.shape = tuple(int(x) for x in shape)
        n = 1
        for x in self.shape:
            n *= x
        self._lib = _cabi.lib()
        self.ptr = self._lib.bfl_dev_alloc(n * 4)
        if not self.ptr:
            raise _cabi.BackendError("bfl_dev_alloc: " + self._lib.bfl_last_error().decode())
        self.__cuda_array_interface__ = {"shape": self.shape, "typestr": "<f4", "data": (self.ptr, False), "version": 2}

    def __del__(self):
        if getattr(self, "ptr", None):
            self._lib.bfl_dev_free(self.ptr)
            self.ptr = None


def exportable_like(t):
    """Copy of the float32 CUDA tensor `t` in an IPC-exportable buffer (torch's caching allocator sub-allocates and
    tags its handles; a dedicated cudaMalloc keeps the exchange independent of torch internals)."""
    import torch
    buf = _DevBuffer(t.shape)
    out = torch.as_tensor(buf, device=t.device)
    out.copy_(t)
    _exportable[out.data_ptr()] = buf
    return out


def open_peer_replicas(t, rank, world, dist):
    """CUDA-IPC exchange of one replica: returns the device addresses, valid in THIS process with the current
    device as accessor, of the other ranks' copies of `t` (same node, peer access over NVLink).  `t` must come
    from exportable_like()."""
    import ctypes as C

    from buffalo_b200 import _cabi
    assert t.data_ptr() in _exportable, "replicas of the fused exchange must be allocated with exportable_like()"
    lib = _cabi.lib()
    mine = C.create_string_buffer(64)
    _cabi.check(lib.bfl_ipc_export(t.data_ptr(), mine), "bfl_ipc_export")
    gathered = [None] * world
    dist.all_gather_object(gathered, mine.raw)
    ptrs = []
    for r, h in enumerate(gathered):
        if r == rank:
            continue
        if h not in _opened:
            base = lib.bfl_ipc_open(C.create_string_buffer(h, 64))
            if not base:
                raise _cabi.BackendError("bfl_ipc_open: " + lib.bfl_last_error().decode())
            _opened[h] = base
        ptrs.append(_opened[h])
    return ptrs


class ShardedALS(object):
    """precompute(axis), update(axis, row_begin, row_end): callables bound to this rank's backend;
    P, Q: this rank's full replicas (torch tensors, updated in place by `update`).

    exchange="allgather": one in-place NCCL all-gather of the updated shard after each half-epoch.
    exchange="p2p": fused -- the solve kernel stores every finished row into the peers' replicas itself
    (backend.set_peer_replicas), so the transfer overlaps the solve row by row over NVLink; the only collective
    left is a one-element all-reduce used as a stream-ordered barrier between half-epochs."""

    def __init__(self, precompute, update, P, Q, rank=0, world=1, dist=None, exchange="allgather", backend=None,
                 indptrs=None):
        """indptrs = (rowwise end offsets, colwise end offsets): with the p2p exchange the rows are then split by
        nonzeros instead of by count (skewed matrices: equal row counts can mean very unequal work)."""
        self.precompute, self.update, self.P, self.Q = precompute, update, P, Q
        self.rank, self.world, self.dist = rank, world, dist
        self.mode = exchange if world > 1 else "none"
        if self.mode == "p2p" and indptrs is not None:
            self.ranges = [nnz_shard(indptrs[0], rank, world), nnz_shard(indptrs[1], rank, world)]
        else:
            self.ranges = [row_shard(P.shape[0], rank, world), row_shard(Q.shape[0], rank, world)]
        if self.mode == "allgather":
            for F in (P, Q):
                assert F.shape[0] % world == 0, "row counts must be divisible by the world size (pad the matrix)"
        # Gram of the opposite factor: every rank sums over its OWN row range and the d x d partials are all-reduced
        # (instead of every rank re-reading the whole replica) when the backend offers the range form
        self.backend = backend
        self.sharded_gram = world > 1 and backend is not None and hasattr(backend, "precompute_rows_device")
        if self.mode == "p2p":
            import torch
            self._flag = torch.zeros(1, device=P.device)
            self._peers = [open_peer_replicas(P, rank, world, dist), open_peer_replicas(Q, rank, world, dist)]
            backend.set_peer_replicas(0, self._peers[0])
            backend.set_peer_replicas(1, self._peers[1])
            dist.barrier()

    def exchange(self, axis):
        if self.mode == "none":
            return
        if self.mode == "p2p":
            # every rank's stores were issued by the kernels already queued on its stream; a stream-ordered
            # collective after them is a barrier for the NEXT half-epoch's reads
            self.dist.all_reduce(self._flag)
            return
        F = self.P if axis == 0 else self.Q
        lo, hi, _ = self.ranges[axis]
        self.dist.all_gather_into_tensor(F, F[lo:hi])

    def half_epoch(self, axis, on_update=None):
        lo, hi, _ = self.ranges[axis]
        if self.sharded_gram:
            olo, ohi, _ = self.ranges[1 - axis]     # the rows of the opposite factor this rank solved last
            self.backend.precompute_rows_device(axis, olo, ohi)
            self.dist.all_reduce(self.backend.gram_tensor())
        else:
            self.precompute(axis)
        if on_update:
            on_update(axis, "begin")
        self.update(axis, lo, hi)
        if on_update:
            on_update(axis, "end")
        self.exchange(axis)

    def iteration(self, on_update=None):
        self.half_epoch(0, on_update)
        self.half_epoch(1, on_update)


class ShardedSGD(object):
    """Row-sharded BPRMF / WARP epoch (SURVEY 8e): every rank owns a contiguous, nnz-balanced user range of the
    rowwise CSR and holds full replicas of P, Q (and Qb).

    * gradient-accumulating configurations (WARP always; BPR with adagrad / adam; bpr.cc:138-156, warp.cc:156-158):
      P and Q are read-only inside an epoch and the gradient sums are additive over users, so the ranks all-reduce
      the accumulators (and the per-row sample counters) and then apply the SAME optimizer step
      (`update_parameters`) -- the replicas stay identical and the result equals the single-GPU epoch up to fp32
      summation order.  Negative sampling is keyed by the global positive index, so the draws do not depend on the
      number of ranks.  The reference does not zero the accumulators after the step (algo.cc:382-465): only rank 0
      carries that leftover into the next epoch, so the all-reduce counts it once.
    * plain-SGD BPR (Hogwild, bpr.cc:157-171): each rank applies its users' updates to its replicas; after the
      epoch the item-side deltas are summed over ranks (Q = Q_start + sum of deltas: bounded staleness of one
      epoch) and each user range is broadcast from its owner.

    `accumulate(lo, hi)` runs the local part of the epoch, `apply()` the optimizer step; `grads` is the list of
    tensors to all-reduce in accumulate mode (float or int), `P, Q, Qb` the replicas."""

    def __init__(self, accumulate, apply, P, Q, Qb, indptr_end, rank=0, world=1, dist=None, grads=None):
        self.accumulate, self.apply = accumulate, apply
        self.P, self.Q, self.Qb = P, Q, Qb
        self.rank, self.world, self.dist = rank, world, dist
        self.grads = [g for g in (grads or []) if g is not None]
        self.mode = "accumulate" if self.grads else "sgd"
        self.bounds = [nnz_shard(indptr_end, r, world)[0] for r in range(world)] + [int(indptr_end.shape[0])]
        self.lo, self.hi = self.bounds[rank], self.bounds[rank + 1]

    def local_positives(self, indptr_end):
        if self.hi <= self.lo:
            return 0
        return int(indptr_end[self.hi - 1]) - (int(indptr_end[self.lo - 1]) if self.lo else 0)

    def epoch(self):
        if self.world == 1:
            self.accumulate(self.lo, self.hi)
            self.apply()
            return
        if self.mode == "accumulate":
            if self.rank != 0:
                for g in self.grads:
                    if g.is_floating_point():
                        g.zero_()
            self.accumulate(self.lo, self.hi)
            for g in self.grads:
                self.dist.all_reduce(g)
            self.apply()
            return
        # plain-SGD BPR: only the item side is shared.  Every rank reads and writes ONLY its own users' rows of P
        # during training, so P is not exchanged per epoch at all (finalize() gathers the user ranges once, at the
        # end); the item deltas of the epoch are summed over the ranks in place:
        #   Q <- Q - Q_start (local delta), all-reduce, Q <- Q_start + sum of deltas, Q_start <- Q
        if getattr(self, "_q_start", None) is None:
            raise RuntimeError("ShardedSGD sgd mode: call begin() once before the first epoch")
        self.accumulate(self.lo, self.hi)
        self.Q.sub_(self._q_start)
        self.dist.all_reduce(self.Q)
        self.Q.add_(self._q_start)
        self._q_start.copy_(self.Q)
        if self.Qb is not None:
            self.Qb.sub_(self._b_start)
            self.dist.all_reduce(self.Qb)
            self.Qb.add_(self._b_start)
            self._b_start.copy_(self.Qb)
        self.apply()

    def begin(self):
        """sgd mode, world > 1: snapshot of the item side the epoch deltas are taken against."""
        if self.world > 1 and self.mode == "sgd":
            self._q_start = self.Q.clone()
            self._b_start = self.Qb.clone() if self.Qb is not None else None

    def finalize(self):
        """sgd mode, world > 1: every user range is broadcast from its owner (once, after the last epoch; callers that
        evaluate between epochs call it before they read rows of P they do not own)."""
        if self.world > 1 and self.mode == "sgd":
            for r in range(self.world):
                lo, hi = self.bounds[r], self.bounds[r + 1]
                if hi > lo:
                    self.dist.broadcast(self.P[lo:hi], src=r)

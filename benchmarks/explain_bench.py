"""ALS explanations (DESIGN.md 4.11): ALS.explain on generated histories, against the host NumPy loop it replaces.

`--users` histories (default 131072) of Pareto lengths (shape 2, mean about 50, capped at 5000) with values 1..5, each
with k = 10 random target items and topm = 5, are explained against models of 100k and 1M items at d = 20, 128 and
256 (random signed item factors of scale 0.1).  The "long" case is `--long-users` histories (default 2048) of exactly
5000 entries each at 1M items, the tail of the Pareto lengths alone.  Per case:
  - call_s     : host clock around ALS.explain (scipy read of the histories, Q checksum, upload, kernel, copy back; it
                 returns host arrays, so the clock ends after a synchronise), Gram cached from a warm-up call;
  - kernel_s   : bfl_als_explain_device alone on resident tensors (CUDA events);
  - rows/s     : histories / seconds, for both;
  - the FLOP and byte model below over kernel_s (an effective rate: item rows gathered twice per target tile mostly hit
    L2, and they count as if read from HBM);
  - host_s     : the per-user NumPy loop (build A_r and b_r, one d x d solve with k right-hand sides, contributions,
                 merge, top-m; fp32) on `--host-sample` rows, scaled to all rows (marked host_extrapolated).
The median of `--repeats` timed calls after one warm-up call is printed.  One JSON line per case; the card's name and
power limit are read in the same process.

Model per row of n entries, D = d, k targets, T = ceil(k / 16) target tiles:
  FLOP  = n D^2 + 2 n D                 (A_r lower triangle and b_r)
        + D^3 / 3                       (Cholesky)
        + k (2 D^2 + 2 D + 2 n D)       (two triangular solves, the score, one dot per history entry)
  bytes = (1 + T) n (8 + 4 D)           (keys, values and gathered item rows: once for A_r, once per target tile)
        + 2 D (D + 1)                   (lower half of the Gram)
        + k (8 + 4 D + 8 topm)          (targets, target rows, scores, keys and contributions)

    python benchmarks/explain_bench.py
    python benchmarks/explain_bench.py --items 100000 --users 16384 --ds 20 --repeats 2      # quick look
"""
import argparse
import json
import subprocess
import sys
import time

import numpy as np
import scipy.sparse

sys.path.insert(0, __file__.rsplit("/benchmarks/", 1)[0])

K, TOPM, TILE = 10, 5, 16


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return None, "unknown"


def histories(n, num_items, seed, length=None):
    rng = np.random.default_rng(seed)
    if length is None:
        lengths = np.minimum(np.ceil((rng.pareto(2.0, n) + 1.0) * 25.0), 5000).astype(np.int64)
    else:
        lengths = np.full(n, length, np.int64)
    keys = rng.integers(0, num_items, int(lengths.sum()), dtype=np.int32)
    vals = rng.integers(1, 6, len(keys)).astype(np.float32)
    indptr = np.concatenate([[0], np.cumsum(lengths)])
    return scipy.sparse.csr_matrix((vals, keys, indptr), shape=(n, num_items))


def model(d, Q):
    from buffalo_b200.algo.als import ALS
    from buffalo_b200.algo.options import ALSOption
    o = ALSOption().get_default_option()
    o.update(d=d)
    m = ALS(o)
    m.P, m.Q = np.zeros((1, d), np.float32), Q
    return m


def flop_byte_model(lengths, d, k, topm):
    n = lengths.astype(np.float64)
    tiles = -(-k // TILE)
    flop = (n * d * d + 2 * n * d + d ** 3 / 3.0 + k * (2 * d * d + 2 * d + 2 * n * d)).sum()
    nbytes = ((1 + tiles) * n * (8 + 4 * d) + 2 * d * (d + 1) + k * (8 + 4 * d + 8 * topm)).sum()
    return float(flop), float(nbytes)


def host_loop(Q, G, H, targets, rows, alpha, reg, topm):
    """The per-user NumPy loop: one d x d solve with k right-hand sides per row."""
    d = Q.shape[1]
    eye = reg * np.eye(d, dtype=np.float32)
    for r in rows:
        lo, hi = H.indptr[r], H.indptr[r + 1]
        keys, v = H.indices[lo:hi], H.data[lo:hi]
        q = Q[keys]
        A = G + (q * (alpha * v)[:, None]).T @ q + eye
        b = ((1.0 + alpha * v)[:, None] * q).sum(axis=0)
        U = np.linalg.solve(A, Q[targets[r]].T)                     # [d, k]
        scores = b @ U
        c = (q @ U) * (1.0 + alpha * v)[:, None]                    # [n, k]
        items, start = np.unique(keys, return_index=True)
        merged = np.add.reduceat(c, start, axis=0)                  # keys are sorted: duplicates adjacent
        order = np.lexsort((np.broadcast_to(items[:, None], merged.shape), -merged), axis=0)[:topm]
        _ = scores, items[order], np.take_along_axis(merged, order, axis=0)


def run_case(a, base, case, H, num_items, d, Q):
    import torch
    from buffalo_b200.algo import fold_in
    rng = np.random.default_rng(7)
    n = H.shape[0]
    targets = rng.integers(0, num_items, (n, K)).astype(np.int32)
    m = model(d, Q)
    m.explain(H, targets, topm=TOPM)                                  # warm-up: uploads Q, computes its Gram
    ts = []
    for _ in range(a.repeats):
        t0 = time.perf_counter()
        m.explain(H, targets, topm=TOPM)
        ts.append(time.perf_counter() - t0)
    call_s = float(np.median(ts))

    st = m._fold_state
    h = st.holder
    indptr, keys, vals = fold_in.history_csr(m, H, num_items)
    ind_t, keys_t, vals_t = fold_in.csr_to_device(indptr, keys, vals)
    tg = torch.from_numpy(targets).cuda()
    m._bind_fold_items(st, h, torch.zeros((1, h.get_vdim()), dtype=torch.float32, device="cuda"))
    h.explain_device(ind_t, keys_t, vals_t, tg, TOPM)
    ks = []
    for _ in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        h.explain_device(ind_t, keys_t, vals_t, tg, TOPM)
        e1.record()
        e1.synchronize()
        ks.append(e0.elapsed_time(e1) / 1e3)
    kernel_s = float(np.median(ks))
    h._keep = []
    lengths = np.diff(H.indptr)
    flop, nbytes = flop_byte_model(lengths, d, K, TOPM)

    sample = np.sort(rng.choice(n, min(a.host_sample, n), replace=False))
    Hs = H.tocsr(copy=True)
    Hs.sort_indices()
    G = (Q.T @ Q).astype(np.float32)
    t0 = time.perf_counter()
    host_loop(Q, G, Hs, targets, sample, float(m.opt.alpha), float(m.opt.reg_u), TOPM)
    host_s = (time.perf_counter() - t0) * n / len(sample)
    print(json.dumps(dict(base, case=case, items=num_items, d=d, users=n, nnz=int(H.nnz), k=K, topm=TOPM,
                          max_len=int(lengths.max()), call_s=round(call_s, 4), call_rows_per_s=round(n / call_s),
                          kernel_s=round(kernel_s, 5), kernel_rows_per_s=round(n / kernel_s),
                          model_GFLOP=round(flop / 1e9, 2), model_GB=round(nbytes / 1e9, 3),
                          kernel_TFLOPps=round(flop / kernel_s / 1e12, 2), kernel_model_GBps=round(nbytes / kernel_s / 1e9, 1),
                          host_s=round(host_s, 2), host_extrapolated=True, host_sample=len(sample),
                          speedup_call_vs_host=round(host_s / call_s, 1))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=131072)
    ap.add_argument("--long-users", type=int, default=2048)
    ap.add_argument("--items", default="100000,1000000")
    ap.add_argument("--ds", default="20,128,256")
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--host-sample", type=int, default=256)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "explain_bench needs a GPU"
    name, limit = card()
    base = dict(gpu=name, power_limit=limit)
    ds = [int(x) for x in a.ds.split(",")]
    items = [int(x) for x in a.items.split(",")]
    for num_items in items:
        H = histories(a.users, num_items, 1)
        for d in ds:
            Q = (np.random.default_rng(2).standard_normal((num_items, d), dtype=np.float32) * 0.1).astype(np.float32)
            run_case(a, base, "pareto", H, num_items, d, Q)
            del Q
        torch.cuda.empty_cache()
    if a.long_users:
        num_items = items[-1]
        H = histories(a.long_users, num_items, 3, length=5000)
        for d in ds:
            Q = (np.random.default_rng(2).standard_normal((num_items, d), dtype=np.float32) * 0.1).astype(np.float32)
            run_case(a, base, "long", H, num_items, d, Q)
            del Q


if __name__ == "__main__":
    main()

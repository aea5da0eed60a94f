"""Exploration (DESIGN.md 4.17): ALS.posterior_sample and ParALS.topk_recommendation(explore=sigma) on generated
histories.

`--users` histories (default 131072) of Pareto lengths (shape 2, mean about 50, capped at 5000) with values 1..5 are
the training rows of `--users` users of models of 100k and 1M items at d = 20, 128 and 256 (random signed factors of
scale 0.1).  Per case:
  - kernel_s   : bfl_als_posterior_sample_device alone on resident tensors (CUDA events), in place on the mean rows;
  - call_s     : host clock around ALS.posterior_sample (scipy read of the histories, Q checksum, uploads, kernel, copy
                 back; it returns host arrays, so the clock ends after a synchronise), Gram cached from a warm-up call;
  - rows/s     : histories / seconds, for both;
  - the FLOP model below over kernel_s;
  - topk_plain_s / topk_explore_s : ParALS.topk_recommendation(users, 10) without and with explore = 1.0 (a new
                 explore_seed per call), the two alternated in one process; the difference is the sampling of the
                 users' rows inside the call (training rows gathered on the host, uploaded, sampled, bound as queries).
The median of `--repeats` timed calls after one warm-up call is printed.  One JSON line per case; the card's name and
power limit are read in the same process.

FLOP model per row of n entries, D = d:
  n D^2      (A_r lower triangle: D (D + 1) / 2 multiply-adds per entry)
  + D^3 / 3  (Cholesky)
  + D^2      (back substitution)
The Box-Muller draws (D / 4 Philox calls, D logf / sincospif) are not counted.

    python benchmarks/explore_bench.py
    python benchmarks/explore_bench.py --items 100000 --users 16384 --ds 20 --repeats 2      # quick look
"""
import argparse
import json
import os
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from benchmarks.explain_bench import card, histories, model  # noqa: E402

SIGMA = 1.0


def flop_model(lengths, d):
    n = lengths.astype(np.float64)
    return float((n * d * d + d ** 3 / 3.0 + d * d).sum())


class _Data(object):
    """The part of a database that ParALS reads for explore: the "rowwise" group."""

    def __init__(self, H):
        self.groups = {"rowwise": {"indptr": H.indptr[1:].astype(np.int64), "key": H.indices.astype(np.int32),
                                   "val": H.data.astype(np.float32)}}

    def get_group(self, name):
        return self.groups[name]


def run_case(a, base, H, num_items, d, Q):
    import torch
    from buffalo_b200.algo import fold_in
    from buffalo_b200.parallel.base import ParALS
    n = H.shape[0]
    rng = np.random.default_rng(7)
    m = model(d, Q)
    m.P = (rng.standard_normal((n, d), dtype=np.float32) * 0.1).astype(np.float32)
    m.posterior_sample(H, m.P, SIGMA, 0)                             # warm-up: uploads Q, computes its Gram
    ts = []
    for r in range(a.repeats):
        t0 = time.perf_counter()
        m.posterior_sample(H, m.P, SIGMA, r + 1)
        ts.append(time.perf_counter() - t0)
    call_s = float(np.median(ts))

    st = m._fold_state
    h = st.holder
    indptr, keys, vals = fold_in.history_csr(m, H, num_items)
    ind_t, keys_t, vals_t, tM = fold_in.to_device(indptr, keys, vals, m.P, h.get_vdim())
    tK = torch.arange(n, dtype=torch.int64, device=tM.device)
    m._bind_fold_items(st, h, torch.zeros((1, h.get_vdim()), dtype=torch.float32, device="cuda"))
    h.posterior_sample_device(ind_t, keys_t, vals_t, tM, tK, 0, SIGMA, out=tM)
    ks = []
    for r in range(a.repeats):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        h.posterior_sample_device(ind_t, keys_t, vals_t, tM, tK, r + 1, SIGMA, out=tM)
        e1.record()
        e1.synchronize()
        ks.append(e0.elapsed_time(e1) / 1e3)
    kernel_s = float(np.median(ks))
    h._keep = []
    del ind_t, keys_t, vals_t, tM, tK
    lengths = np.diff(H.indptr)
    flop = flop_model(lengths, d)

    m.data = _Data(H)
    par = ParALS(m)
    users = np.arange(n, dtype=np.int32)
    par.topk_recommendation(users, 10)                                # warm-up of both
    par.topk_recommendation(users, 10, explore=SIGMA, explore_seed=0)
    plain, explore = [], []
    for r in range(a.repeats):
        t0 = time.perf_counter()
        par.topk_recommendation(users, 10)
        plain.append(time.perf_counter() - t0)
        t0 = time.perf_counter()
        par.topk_recommendation(users, 10, explore=SIGMA, explore_seed=r + 1)
        explore.append(time.perf_counter() - t0)
    plain_s, explore_s = float(np.median(plain)), float(np.median(explore))
    print(json.dumps(dict(base, items=num_items, d=d, users=n, nnz=int(H.nnz), max_len=int(lengths.max()),
                          kernel_s=round(kernel_s, 5), kernel_rows_per_s=round(n / kernel_s),
                          call_s=round(call_s, 4), call_rows_per_s=round(n / call_s),
                          model_GFLOP=round(flop / 1e9, 2), kernel_TFLOPps=round(flop / kernel_s / 1e12, 2),
                          topk_plain_s=round(plain_s, 4), topk_explore_s=round(explore_s, 4),
                          topk_explore_over_plain=round(explore_s / plain_s, 2))), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=131072)
    ap.add_argument("--items", default="100000,1000000")
    ap.add_argument("--ds", default="20,128,256")
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "explore_bench needs a GPU"
    name, limit = card()
    base = dict(gpu=name, power_limit=limit)
    ds = [int(x) for x in a.ds.split(",")]
    for num_items in [int(x) for x in a.items.split(",")]:
        H = histories(a.users, num_items, 1)
        H.sort_indices()
        for d in ds:
            Q = (np.random.default_rng(2).standard_normal((num_items, d), dtype=np.float32) * 0.1).astype(np.float32)
            run_case(a, base, H, num_items, d, Q)
            del Q
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

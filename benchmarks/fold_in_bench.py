"""Fold-in (DESIGN.md 4.10): ALS.fold_in, PLSI.fold_in and ParALS.fold_in_recommendation on generated histories.

`--users` histories (default 131072) of Pareto lengths (shape 2, mean about 50, capped at 5000) with values 1..5 are
folded into a model of 100k and of 1M items (random factors; only the item factors matter):
  - als      : ALS.fold_in (d = 20 manual_cg, d = 128 iALS++), one sweep, host clock around the call (it returns a host
               array, so the clock covers the history upload, the solve and the copy back).  "cached": the Gram and the
               padded Q are resident from an earlier call (what every call after the first pays); "recomputed": the
               state's checksum and the Gram's are dropped first, so the call uploads Q and computes its Gram again
               (what a call after train() or normalize() pays).  users/s = users / seconds.  q_checksum_s: the host
               checksum of Q (Parallel._fingerprint) alone, which every call computes.
  - plsi     : PLSI.fold_in with iters = 10 (host clock, cached Q), and plsi_fold_in_kernel alone on resident tensors
               (CUDA events).  Byte model per call: iters * (8 B of key + value and 4 * vdim B of item row per entry)
               + 8 * vdim B per row (read start row, write result); GB/s = model bytes / kernel seconds (item rows that
               hit L2 count as if read from HBM, so this is an effective rate, not a measured DRAM rate).
  - serve    : ParALS.fold_in_recommendation (k = 10, exclude_seen) against fold_in followed by the host-array path
               topk_recommendation(exclude_seen=...) runs (Parallel._rank: folded rows and seen CSR uploaded from the
               host, bfl_seen_topk), both with a resident item handle; host clock; keys compared.
The median of `--repeats` timed calls after one warm-up call is printed.  One JSON line per case; the card's name and
power limit are read in the same process.

    python benchmarks/fold_in_bench.py
    python benchmarks/fold_in_bench.py --items 100000 --users 16384 --repeats 2      # quick look
"""
import argparse
import json
import subprocess
import sys
import time

import numpy as np
import scipy.sparse

sys.path.insert(0, __file__.rsplit("/benchmarks/", 1)[0])


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return None, "unknown"


def histories(n, num_items, seed):
    rng = np.random.default_rng(seed)
    lengths = np.minimum(np.ceil((rng.pareto(2.0, n) + 1.0) * 25.0), 5000).astype(np.int64)
    keys = rng.integers(0, num_items, int(lengths.sum()), dtype=np.int32)
    vals = rng.integers(1, 6, len(keys)).astype(np.float32)
    indptr = np.concatenate([[0], np.cumsum(lengths)])
    return scipy.sparse.csr_matrix((vals, keys, indptr), shape=(n, num_items))


def timed(fn, repeats):
    fn()
    ts = []
    for _ in range(repeats):
        t0 = time.perf_counter()
        out = fn()
        ts.append(time.perf_counter() - t0)
    return out, float(np.median(ts))


def make_model(kind, d, Q):
    if kind == "als":
        from buffalo_b200.algo.als import ALS
        from buffalo_b200.algo.options import ALSOption
        o = ALSOption().get_default_option()
        o.update(d=d, optimizer="manual_cg" if d < 128 else "ialspp")
        m = ALS(o)
    else:
        from buffalo_b200.algo.options import PLSIOption
        from buffalo_b200.algo.plsi import PLSI
        o = PLSIOption().get_default_option()
        o.update(d=d, num_iters=10)
        m = PLSI(o)
    m.P, m.Q = np.zeros((1, d), np.float32), Q
    return m


def item_factors(kind, num_items, d, seed):
    rng = np.random.default_rng(seed)
    if kind == "als":
        return (rng.standard_normal((num_items, d), dtype=np.float32) * 0.1).astype(np.float32)
    Q = rng.random((num_items, d), dtype=np.float32) + 0.05
    return (Q / Q.sum(axis=0, keepdims=True)).astype(np.float32)


def plsi_kernel_seconds(m, H, iters, repeats):
    import torch
    from buffalo_b200.algo import fold_in
    indptr, keys, vals = fold_in.history_csr(m, H, m.Q.shape[0])
    st = m._fold_state
    vdim = st.holder.get_vdim()
    X0 = fold_in.start_rows(None, len(indptr), m.opt.d, 1.0 / m.opt.d)
    ind_t, keys_t, vals_t, tX = fold_in.to_device(indptr, keys, vals, X0, vdim)
    run = lambda: st.holder.fold_in_device(st.F, ind_t, keys_t, vals_t, tX, iters, m.opt.alpha1)
    run()
    best = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        run()
        b.record()
        b.synchronize()
        best.append(a.elapsed_time(b) / 1e3)
    nnz, n = len(keys), len(indptr)
    model_bytes = iters * nnz * (8 + 4 * vdim) + 8 * vdim * n
    sec = float(np.median(best))
    return sec, model_bytes


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=131072)
    ap.add_argument("--items", default="100000,1000000")
    ap.add_argument("--repeats", type=int, default=3)
    a = ap.parse_args()
    import torch
    from buffalo_b200.parallel.base import Parallel
    assert torch.cuda.is_available(), "fold_in_bench needs a GPU"
    name, limit = card()
    base = dict(gpu=name, power_limit=limit, users=a.users)
    for num_items in [int(x) for x in a.items.split(",")]:
        H = histories(a.users, num_items, 1)
        nnz = int(H.nnz)
        for d in (20, 128):
            Q = item_factors("als", num_items, d, 2)
            m = make_model("als", d, Q)
            _, t_cached = timed(lambda: m.fold_in(H), a.repeats)

            def recomputed():
                st = m._fold_state
                st.key = st.derived_key = None          # as after a change of Q: upload Q, compute the Gram
                return m.fold_in(H)
            _, t_recomputed = timed(recomputed, a.repeats)
            _, t_checksum = timed(lambda: Parallel._fingerprint(Q), a.repeats)
            print(json.dumps(dict(base, case="als", items=num_items, d=d, nnz=nnz, cached_s=round(t_cached, 4),
                                  cached_users_per_s=round(a.users / t_cached), recomputed_s=round(t_recomputed, 4),
                                  recomputed_users_per_s=round(a.users / t_recomputed),
                                  q_checksum_s=round(t_checksum, 4))), flush=True)
            if d == 128 or num_items == 100000:
                from buffalo_b200.parallel.base import ParALS
                par = ParALS(m)
                (k1, _), t_dev = timed(lambda: par.fold_in_recommendation(H, topk=10), a.repeats)
                from buffalo_b200.algo import fold_in as F
                indptr, keys, _ = F.history_csr(m, H, num_items)

                def host_path():
                    X = m.fold_in(H)
                    return par._rank(np.arange(a.users, dtype=np.int32), X, m.Q, None, 10, seen=(indptr, keys))
                (k2, _), t_host = timed(host_path, a.repeats)
                print(json.dumps(dict(base, case="serve", items=num_items, d=d, k=10, device_path_s=round(t_dev, 4),
                                      host_round_trip_s=round(t_host, 4), same_keys=bool(np.array_equal(k1, k2)))),
                      flush=True)
            del m, Q
        for d in (20, 128):
            Q = item_factors("plsi", num_items, d, 3)
            m = make_model("plsi", d, Q)
            _, t_call = timed(lambda: m.fold_in(H, iters=10), a.repeats)
            sec, model_bytes = plsi_kernel_seconds(m, H, 10, a.repeats)
            print(json.dumps(dict(base, case="plsi", items=num_items, d=d, iters=10, nnz=nnz, call_s=round(t_call, 4),
                                  users_per_s=round(a.users / t_call), kernel_s=round(sec, 5),
                                  kernel_model_GBps=round(model_bytes / sec / 1e9, 1))), flush=True)
            del m, Q
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

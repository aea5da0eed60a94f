#!/usr/bin/env python
"""IVF index against exact serving (DESIGN.md 4.12): build time, search time (device events and end to end),
queries/s, rows scanned per query (mean / max: list imbalance), recall@10 against exact Serve.topk timed in the same
process and alternated with it, index memory, and the card name and power limit read in the same run.

Two factor sets: a clustered Gaussian mixture (what trained factors look like) and isotropic Gaussian rows (the worst
case: no cluster structure, so the lists carry little information about a query's best items).

  python benchmarks/ivf_bench.py                    # 131072 queries, 100k and 1M items, d = 20 and 128
  python benchmarks/ivf_bench.py --items 100000 --d 20 --queries 16384 --nlist 1024 --nprobe 8 32
Prints one JSON line per configuration."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests.ivf_ref import gaussian_mixture  # noqa: E402


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def timed(fn, reps):
    """(end-to-end seconds, device-event seconds) of the best of reps calls, and the last result."""
    import torch
    best_e2e = best_dev = float("inf")
    out = None
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        a.record()
        out = fn()
        b.record()
        torch.cuda.synchronize()
        best_e2e = min(best_e2e, time.perf_counter() - t0)
        best_dev = min(best_dev, a.elapsed_time(b) / 1e3)
    return best_e2e, best_dev, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--items", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--d", type=int, nargs="+", default=[20, 128])
    ap.add_argument("--queries", type=int, default=131072)
    ap.add_argument("--nlist", type=int, nargs="+", default=[1024, 4096])
    ap.add_argument("--nprobe", type=int, nargs="+", default=[8, 16, 32, 64, 128])
    ap.add_argument("--sets", nargs="+", default=["clustered", "isotropic"])
    ap.add_argument("--reps", type=int, default=2)
    args = ap.parse_args()
    import torch
    from buffalo_b200 import backend
    assert torch.cuda.is_available(), "ivf_bench needs a GPU"
    gpu = card()
    for fset in args.sets:
        for n in args.items:
            for d in args.d:
                if fset == "clustered":
                    items = gaussian_mixture(n, d, 2048, seed=1)
                    users = gaussian_mixture(args.queries, d, 2048, seed=2)
                else:
                    rng = np.random.default_rng(1)
                    items = rng.standard_normal((n, d)).astype(np.float32)
                    users = rng.standard_normal((args.queries, d)).astype(np.float32)
                qidx = np.arange(args.queries, dtype=np.int32)
                serve = backend.Serve()
                serve.set_items(items)
                serve.set_queries(users)
                dq = torch.from_numpy(users).cuda()
                for nlist in args.nlist:
                    ivf = backend.IVF()
                    t0 = time.perf_counter()
                    ivf.build(items, None, nlist, 10, seed=0)
                    build_s = time.perf_counter() - t0
                    lens = np.diff(ivf.offsets(), prepend=0)
                    cent = np.ascontiguousarray(ivf.centroids())
                    for nprobe in [p for p in args.nprobe if p <= nlist]:
                        ivf.search_device(dq[:1024], nprobe, 10)       # warm-up of this shape
                        serve.topk(qidx[:1024], 10)
                        ex_e2e = ex_dev = iv_e2e = iv_dev = float("inf")
                        for _ in range(args.reps):                      # alternated: exact, then IVF
                            e, dv, (want, _) = timed(lambda: serve.topk(qidx, 10), 1)
                            ex_e2e, ex_dev = min(ex_e2e, e), min(ex_dev, dv)
                            e, dv, got = timed(lambda: ivf.search_device(dq, nprobe, 10), 1)
                            iv_e2e, iv_dev = min(iv_e2e, e), min(iv_dev, dv)
                        got = got[0].cpu().numpy()
                        recall = float(np.mean([len(np.intersect1d(g, w)) / 10.0 for g, w in zip(got, want)]))
                        # rows scanned per query: the sizes of its nprobe lists (the coarse step as the index runs it)
                        cs = backend.Serve()
                        cs.set_items(cent)
                        cs.set_queries(users)
                        probed, _ = cs.topk(qidx, nprobe, want_scores=False)
                        cs.close()
                        scanned = lens[probed].sum(1)
                        print(json.dumps({
                            "set": fset, "items": n, "d": d, "queries": args.queries, "nlist": nlist,
                            "nprobe": nprobe, "build_s": round(build_s, 3),
                            "ivf_search_s_events": round(iv_dev, 4), "ivf_search_s_e2e": round(iv_e2e, 4),
                            "ivf_qps": round(args.queries / iv_e2e), "exact_s_events": round(ex_dev, 4),
                            "exact_s_e2e": round(ex_e2e, 4), "exact_qps": round(args.queries / ex_e2e),
                            "speedup_e2e": round(ex_e2e / iv_e2e, 2), "recall_at_10": round(recall, 4),
                            "rows_scanned_mean": round(float(scanned.mean())), "rows_scanned_max": int(scanned.max()),
                            "list_len_max": int(lens.max()), "empty_lists": int((lens == 0).sum()),
                            "index_mb": round(ivf.nbytes() / 2 ** 20, 1), "gpu": gpu}), flush=True)
                    ivf.close()
                serve.close()


if __name__ == "__main__":
    main()

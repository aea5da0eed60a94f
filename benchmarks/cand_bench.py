#!/usr/bin/env python
"""Per-user candidate pools (DESIGN.md 4.13): ParALS.topk_recommendation(pool=<sparse matrix>) for 131072 users.

For each configuration: the device time of Serve.topk_candidates_device with the lists already on the device (CUDA
events on the call's stream), the end-to-end time of the public call (host row gather, checksum, query upload, list
upload, kernels, copy back), candidates/s, the byte model (gathered item rows sum(|C|) * 4 * ld, plus the lists and the
seen keys) over the 3.35 TB/s data-sheet rate, and two baselines timed on a sample of users and scaled: one
topk_recommendation(pool=list) call per user (its keys checked equal on the sample) and the NumPy per-row loop.
The card name and power limit are read in the same run.

  python benchmarks/cand_bench.py                         # 100k and 1M items, d = 20 and 128, 100 / 1000 / 10000
  python benchmarks/cand_bench.py --items 100000 --d 20 --lens 100 pareto
Prints one JSON line per configuration."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np
import scipy.sparse

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

HBM_BYTES_PER_S = 3.35e12                           # H100 SXM data sheet


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


def model(U, I, d, seed):
    from tests.test_ivf_cpu import cpu_model
    m = cpu_model("als", U=2, I=2, d=d)
    rng = np.random.default_rng(seed)
    m.P = rng.standard_normal((U, d)).astype(np.float32)
    m.Q = rng.standard_normal((I, d)).astype(np.float32)
    m._idmanager.userids = ["u%d" % i for i in range(U)]
    m._idmanager.itemids = ["i%d" % i for i in range(I)]
    return m


def pool_matrix(U, I, lens, seed):
    rng = np.random.default_rng(seed)
    if lens == "pareto":                            # mean near 1000, a long tail capped at 100k
        n = np.minimum((rng.pareto(1.2, size=U) + 1) * 170, 100000).astype(np.int64)
    else:
        n = np.full(U, int(lens), np.int64)
    ptr = np.concatenate([[0], np.cumsum(n)]).astype(np.int64)
    idx = rng.integers(0, I, size=int(ptr[-1])).astype(np.int32)
    return scipy.sparse.csr_matrix((np.ones(idx.size, np.float32), idx, ptr), shape=(U, I))


def best(fn, reps):
    import torch
    t, out = float("inf"), None
    for _ in range(reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        t = min(t, time.perf_counter() - t0)
    return t, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=131072)
    ap.add_argument("--items", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--d", type=int, nargs="+", default=[20, 128])
    ap.add_argument("--lens", nargs="+", default=["100", "1000", "10000", "pareto"])
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--sample", type=int, default=64)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "cand_bench needs a GPU"
    from buffalo_b200.parallel.base import ParALS, cand_topn
    from buffalo_b200.evaluate.device import _gather_rows
    name = card()
    U, k = args.users, args.k
    for I in args.items:
        for d in args.d:
            par = ParALS(model(U, I, d, 1))
            users = np.arange(U, dtype=np.int32)
            for lens in args.lens:
                M = pool_matrix(U, I, lens, 2)
                S = pool_matrix(U, I, 20, 3)              # 20 seen items per user
                for seen in (False, True):
                    excl = S if seen else False
                    par.topk_recommendation(users[:1024], topk=k, pool=M, exclude_seen=excl)   # warm-up
                    e2e, (_, keys, _) = best(lambda: par.topk_recommendation(users, topk=k, pool=M, exclude_seen=excl),
                                             args.reps)
                    # device time: the lists and the seen rows on the device, the queries resident
                    h = par._serve
                    h.set_queries(np.ascontiguousarray(par.algo.P))
                    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
                    cptr, ckeys = t(np.asarray(M.indptr[1:], np.int64)), t(M.indices.astype(np.int32))
                    sarg = (t(np.asarray(S.indptr[1:], np.int64)), t(S.indices.astype(np.int32))) if seen else None
                    q = t(users)
                    h.topk_candidates_device(q, k, cptr, ckeys, seen=sarg)
                    dev = float("inf")
                    for _ in range(args.reps):
                        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        a.record()
                        idx, _ = h.topk_candidates_device(q, k, cptr, ckeys, seen=sarg)
                        b.record()
                        torch.cuda.synchronize()
                        dev = min(dev, a.elapsed_time(b) / 1e3)
                    assert np.array_equal(idx.cpu().numpy(), keys)
                    ncand = int(M.indptr[-1])
                    nbytes = ncand * 4 * d + ncand * 4 + U * 8 + (int(S.indptr[-1]) * 4 + U * 8 if seen else 0)
                    # baselines on a sample, scaled to all users
                    rng = np.random.default_rng(4)
                    sample = rng.choice(U, size=args.sample, replace=False).astype(np.int32)
                    rows = [M.indices[M.indptr[u]:M.indptr[u + 1]].astype(np.int32) for u in sample]

                    def per_user():
                        out = []
                        for u, row in zip(sample, rows):
                            out.append(par.topk_recommendation(np.array([u], np.int32), topk=k, pool=row,
                                                               exclude_seen=excl)[1][0] if row.size else np.full(k, -1))
                        return np.array(out)
                    t_user, ku = best(per_user, 1)
                    assert np.array_equal(ku, keys[sample])
                    cands = _gather_rows(np.asarray(M.indptr[1:], np.int64), M.indices, sample)
                    sr = _gather_rows(np.asarray(S.indptr[1:], np.int64), S.indices, sample) if seen else ()
                    t0 = time.perf_counter()
                    cand_topn(sample, par.algo.P, par.algo.Q, None, k, *cands, *sr)
                    t_np = time.perf_counter() - t0
                    print(json.dumps(dict(
                        card=name, users=U, items=I, d=d, k=k, lens=lens, exclude_seen=seen, candidates=ncand,
                        device_s=round(dev, 5), end_to_end_s=round(e2e, 4),
                        candidates_per_s_device=float("%.4g" % (ncand / dev)),
                        candidates_per_s_e2e=float("%.4g" % (ncand / e2e)),
                        model_bytes=nbytes, model_s_at_datasheet=float("%.4g" % (nbytes / HBM_BYTES_PER_S)),
                        per_user_calls_s_scaled=round(t_user / args.sample * U, 2),
                        numpy_loop_s_scaled=round(t_np / args.sample * U, 2))), flush=True)


if __name__ == "__main__":
    main()

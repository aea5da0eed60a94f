#!/usr/bin/env python
"""MMR re-ranking (DESIGN.md 4.15): ParALS.topk_recommendation(diversify=w) for 131072 users.

For each configuration (items, d, M candidates per user, weight w; k = 10):
  - rerank_ms: the device time of bfl_mmr_rerank_device alone on candidates already on the device (CUDA events, best
    of --reps);
  - stage_kM_ms / stage_k10_ms: the candidate stage (Serve.topk_device over all items) at k = M and at k = 10;
  - plain_s / diverse_s: the public call without and with diversify, end to end, alternated in one process (best of
    --reps each);
  - ild10_plain / ild10_diverse: ild@10 of both lists from evaluate_lists(item_factors=Q);
  - the cost model per row: M (M + 1) / 2 * d FMAs for the Gram triangle plus k * M fp64 objective updates, and
    M * vdim * 4 bytes of gathered item rows plus 8 M bytes of candidates in and 8 k bytes out; the rates these give
    over rerank_ms, against the 67 TFLOP/s FP32 and 3.35 TB/s of the H100 SXM data sheet;
  - numpy_extrapolated_s: parallel.base.mmr_numpy on a 256-user sample of the same candidates, scaled to all users.
The card name and power limit are read in the same run.

  python benchmarks/rerank_bench.py                       # 100k and 1M items, d = 20 and 128, M = 50 / 100 / 256
  python benchmarks/rerank_bench.py --items 100000 --d 20 --m 50 --w 0.3
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
FP32_FLOP_PER_S = 67e12


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
    return m


def events(fn, reps):
    """Best CUDA-event time of fn() in ms over reps calls after one warm-up."""
    import torch
    fn()
    best = float("inf")
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def wall(fn):
    import torch
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return time.perf_counter() - t0, out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=131072)
    ap.add_argument("--items", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--d", type=int, nargs="+", default=[20, 128])
    ap.add_argument("--m", type=int, nargs="+", default=[50, 100, 256])
    ap.add_argument("--w", type=float, nargs="+", default=[0.1, 0.3, 0.5])
    ap.add_argument("--k", type=int, default=10)
    ap.add_argument("--sample", type=int, default=256)
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "rerank_bench needs a GPU"
    from buffalo_b200 import _cabi
    from buffalo_b200.evaluate import evaluate_lists
    from buffalo_b200.parallel.base import ParALS, mmr_numpy
    name = card()
    U, k = args.users, args.k
    users = np.arange(U, dtype=np.int32)
    rng = np.random.default_rng(3)
    test = scipy.sparse.csr_matrix((np.ones(U, np.float32), rng.integers(0, min(args.items), size=U), np.arange(U + 1)),
                                   shape=(U, min(args.items)))
    for I in args.items:
        test.resize((U, I))
        for d in args.d:
            par = ParALS(model(U, I, d, 1))
            Q = par.algo.Q
            par.topk_recommendation(users[:1024], topk=k)                       # warm-up: items resident
            h = par._serve
            h.set_queries(np.ascontiguousarray(par.algo.P))
            q = torch.from_numpy(users).cuda()
            stage_k = events(lambda: h.topk_device(q, k), args.reps)
            for M in args.m:
                stage_m = events(lambda: h.topk_device(q, M), args.reps)
                ci, cv = h.topk_device(q, M)
                oi = torch.empty((U, k), dtype=torch.int32, device="cuda")
                ov = torch.empty((U, k), dtype=torch.float32, device="cuda")
                sample = np.sort(rng.choice(U, size=args.sample, replace=False))
                ci_s, cv_s = ci.cpu().numpy()[sample], cv.cpu().numpy()[sample]
                for w in args.w:
                    w32 = float(np.float32(w))

                    def kernel():
                        _cabi.check(h._lib.bfl_mmr_rerank_device(h._h, ci.data_ptr(), cv.data_ptr(), U, M, k, w32,
                                                                 oi.data_ptr(), ov.data_ptr(),
                                                                 torch.cuda.current_stream().cuda_stream), "rerank")
                    rerank = events(kernel, args.reps)
                    plain_s = diverse_s = float("inf")
                    for _ in range(args.reps):                                   # alternated in one process
                        t, (_, plain, _) = wall(lambda: par.topk_recommendation(users, topk=k))
                        plain_s = min(plain_s, t)
                        t, (_, div, _) = wall(lambda: par.topk_recommendation(users, topk=k, diversify=w,
                                                                              diversify_candidates=M))
                        diverse_s = min(diverse_s, t)
                    assert np.array_equal(div, oi.cpu().numpy())
                    ild_p = evaluate_lists(plain, test, cutoffs=(k,), item_factors=Q)["ild@%d" % k]
                    ild_d = evaluate_lists(div, test, cutoffs=(k,), item_factors=Q)["ild@%d" % k]
                    t0 = time.perf_counter()
                    kn, _ = mmr_numpy(ci_s, cv_s, Q, k, w32)
                    t_np = time.perf_counter() - t0
                    vdim = Q.shape[1]
                    flop = U * (M * (M + 1) * d)                                 # 2 FLOPs per Gram FMA
                    obj = U * k * M
                    nbytes = U * (M * vdim * 4 + 8 * M + 8 * k)
                    print(json.dumps(dict(
                        card=name, users=U, items=I, d=d, k=k, M=M, w=w,
                        rerank_ms=round(rerank, 3), stage_kM_ms=round(stage_m, 3), stage_k10_ms=round(stage_k, 3),
                        plain_s=round(plain_s, 4), diverse_s=round(diverse_s, 4),
                        ild10_plain=round(ild_p, 5), ild10_diverse=round(ild_d, 5),
                        model_gram_flop=flop, model_obj_updates=obj, model_bytes=nbytes,
                        gram_tflop_per_s=round(flop / rerank / 1e9, 2),
                        gram_share_of_fp32_datasheet=round(flop / rerank * 1e3 / FP32_FLOP_PER_S, 4),
                        bytes_tb_per_s=round(nbytes / rerank / 1e9, 3),
                        bytes_share_of_hbm_datasheet=round(nbytes / rerank * 1e3 / HBM_BYTES_PER_S, 4),
                        numpy_sample_keys_equal_share=float(np.mean(kn == oi.cpu().numpy()[sample])),
                        numpy_extrapolated_s=round(t_np / args.sample * U, 2))), flush=True)
            par._serve.close()
            par._serve = None
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

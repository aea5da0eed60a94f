#!/usr/bin/env python
"""Item fold-in throughput (DESIGN.md 4.16): ALS.fold_in_items and BPRMF / WARP .fold_in_items on 131072 new items with
a mean of 50 users each, against 1M and 10M users, at d = 20 and 128.

  python benchmarks/item_fold_in_bench.py [--users 1000000 10000000] [--dims 20 128] [--items 131072] [--out DIR]

Per configuration it prints end-to-end seconds of a call (host clock around the call, which ends with the copy of the
rows to the host) and items/s, and the summed device time of the call (kernels and copies) from torch.profiler in a
separate run.
ALS is timed with the Gram cached (P already resident: the steady state of repeated calls) and uncached (P uploaded and
its Gram computed in the call); BPRMF with sgd and adagrad, WARP with adagrad, each for epochs = 1 and num_iters = 10.
The trained catalogue has 1M items and each user 10 training items (the negatives' seen check).  Factors are random:
the work per positive does not depend on their values.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import subprocess
import sys
import time
import types

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


class Data(object):
    def __init__(self, U, I, per_user, rng):
        keys = np.sort(rng.integers(0, I, (U, per_user), dtype=np.int32), axis=1)
        self.header = {"num_users": U, "num_items": I, "num_nnz": U * per_user}
        self.rowwise = {"indptr": np.arange(1, U + 1, dtype=np.int64) * per_user, "key": keys.reshape(-1),
                        "val": np.ones(U * per_user, np.float32)}
        self.opt = types.SimpleNamespace(data=types.SimpleNamespace(batch_mb=64))

    def get_header(self):
        return self.header

    def get_group(self, name):
        return self.rowwise


def card():
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True, check=True).stdout.strip().splitlines()
    return out[0]


def histories(n, U, mean, rng):
    import scipy.sparse
    lengths = rng.poisson(mean, n).astype(np.int64)
    cols = rng.integers(0, U, int(lengths.sum()))
    rows = np.repeat(np.arange(n), lengths)
    H = scipy.sparse.csr_matrix((np.ones(len(cols), np.float32), (rows, cols)), shape=(n, U))
    H.sum_duplicates()
    H.data[:] = 1.0
    return H


def device_ms(fn):
    import torch
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        fn()
        torch.cuda.synchronize()
    return sum(e.device_time_total for e in prof.key_averages()) / 1e3


def timed(fn, reps=3):
    import torch
    fn()
    torch.cuda.synchronize()
    best = float("inf")
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        best = min(best, time.perf_counter() - t0)
    return best


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, nargs="+", default=[1000000, 10000000])
    ap.add_argument("--dims", type=int, nargs="+", default=[20, 128])
    ap.add_argument("--items", type=int, default=131072)
    ap.add_argument("--catalogue", type=int, default=1000000)
    ap.add_argument("--mean-users", type=float, default=50.0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    from buffalo_b200.algo.als import ALS
    from buffalo_b200.algo.bpr import BPRMF
    from buffalo_b200.algo.options import ALSOption, BPRMFOption, WARPOption
    from buffalo_b200.algo.warp import WARP
    gpu = card()
    print("card:", gpu)
    rng = np.random.default_rng(0)
    results = []
    for U in a.users:
        data = Data(U, a.catalogue, 10, rng)
        H = histories(a.items, U, a.mean_users, rng)
        for d in a.dims:
            P = (rng.standard_normal((U, d), dtype=np.float32) * 0.1)
            Q = (rng.standard_normal((a.catalogue, d), dtype=np.float32) * 0.1)
            configs = [("als", "gram cached", ALS, ALSOption, dict(optimizer="manual_cg"), None),
                       ("als", "gram uncached", ALS, ALSOption, dict(optimizer="manual_cg"), None)]
            for epochs in (1, 10):
                configs += [("bpr", "sgd", BPRMF, BPRMFOption, dict(optimizer="sgd"), epochs),
                            ("bpr", "adagrad", BPRMF, BPRMFOption, dict(optimizer="adagrad"), epochs),
                            ("warp", "adagrad", WARP, WARPOption, dict(optimizer="adagrad"), epochs)]
            for kind, label, cls, opt_cls, extra, epochs in configs:
                o = opt_cls().get_default_option()
                o.update(dict(d=d, num_iters=10, random_seed=1, compute_loss_on_training=False), **extra)
                m = cls(o)
                m.P, m.Q = P, Q
                if kind != "als":
                    m.Qb = np.zeros((a.catalogue, 1), np.float32)
                    m.data = data
                    call = lambda: m.fold_in_items(H, epochs=epochs)
                elif label == "gram uncached":
                    def call():
                        m._fold_state_items = None      # as after a change of P: upload P, compute its Gram
                        m.fold_in_items(H)
                else:
                    call = lambda: m.fold_in_items(H)
                sec = timed(call)
                kms = device_ms(call)
                r = dict(model=kind, variant=label, epochs=epochs, users=U, d=d, items=a.items, nnz=int(H.nnz),
                         seconds=round(sec, 4), items_per_s=round(a.items / sec), device_ms=round(kms, 2), card=gpu)
                print(json.dumps(r), flush=True)
                results.append(r)
                del m
                torch.cuda.empty_cache()
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "item_fold_in_bench.json"), "w") as f:
            json.dump(results, f, indent=1)


if __name__ == "__main__":
    main()

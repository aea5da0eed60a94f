"""Offline evaluation (Evaluable.evaluate, csrc/offline_eval.cu) on a generated Zipf CSR: 1M users x 100k items, d = 128,
cutoffs 10 / 20 / 50 / 100, exclude_seen=True, with and without diversity.

Every user holds out a Zipf-length set of items.  Per configuration one warm-up call, then --steps timed calls: the
end-to-end time (host clock around a call that ends in a synchronise), the device milliseconds per stage (CUDA events:
upload, topk, terms, ild, coverage, sum), rows/s and the peak torch device memory of the call (the library's own
stream-ordered scratch is not in it).  The NumPy reference (tests/eval_offline_ref.py, after a float64 NumPy ranking
that leaves the training items out) is timed on --host-sample users and scaled to all users, marked
"numpy_extrapolated".  The card name and power limit are read in the same run.  One JSON line per configuration.

    python benchmarks/offline_eval_bench.py --users 1000000 --items 100000 --d 128
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
    out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                         stdout=subprocess.PIPE, text=True).stdout.strip().splitlines()
    return out[0] if out else "unknown"


class Model(object):
    """The part of a trained model Evaluable.evaluate reads: factors, the training rows and the device-ranking hook."""

    def __init__(self, P, Q, data):
        self.P, self.Q, self.data = P, Q, data

    def _device_eval_model(self):
        from buffalo_b200.evaluate.device import EvalModel
        return EvalModel(self.P, self.Q, None, None, False)


def numpy_reference(P, Q, indptr, keys, T, rows, cutoffs, diversity):
    """Seconds of the fp64 NumPy path on `rows`: scores, training items left out, top max(cutoffs), reference metrics."""
    from tests import eval_offline_ref as ref
    K = max(cutoffs)
    t0 = time.perf_counter()
    s = P[rows].astype(np.float64) @ Q.astype(np.float64).T
    for i, u in enumerate(rows):
        s[i, keys[(indptr[u - 1] if u else 0):indptr[u]]] = -np.inf
    ranked = np.argsort(-s, axis=1, kind="stable")[:, :K]
    ref.evaluate(ranked, T[rows], cutoffs, Q if diversity else None)
    return time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--cutoffs", default="10,20,50,100")
    ap.add_argument("--mean-len", type=int, default=20)
    ap.add_argument("--max-len", type=int, default=5000)
    ap.add_argument("--steps", type=int, default=2)
    ap.add_argument("--host-sample", type=int, default=200)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "offline_eval_bench.py measures the device path: it needs a GPU"
    from benchmarks.eval_bench import ArrayData, zipf_csr
    cutoffs = [int(x) for x in a.cutoffs.split(",")]
    t0 = time.perf_counter()
    indptr, keys, vrow, vcol, vval = zipf_csr(a.users, a.items, a.mean_len, a.max_len, a.seed)
    data = ArrayData(a.users, a.items, indptr, keys, vrow, vcol, vval)
    rng = np.random.default_rng(a.seed + 1)
    P = (rng.normal(size=(a.users, a.d)) * 0.1).astype(np.float32)
    Q = (rng.normal(size=(a.items, a.d)) * 0.1).astype(np.float32)
    lens = np.minimum(rng.zipf(2.0, size=a.users), 200)
    T = scipy.sparse.csr_matrix((np.ones(int(lens.sum())), (np.repeat(np.arange(a.users), lens),
                                                            rng.integers(0, a.items, int(lens.sum())))),
                                shape=(a.users, a.items))
    model = Model(P, Q, data)
    gen_s = time.perf_counter() - t0
    from buffalo_b200.evaluate import offline
    base = dict(card=card(), users=a.users, items=a.items, train_nnz=int(len(keys)), test_nnz=int(T.nnz), d=a.d,
                cutoffs=cutoffs, exclude_seen=True, gen_s=round(gen_s, 2), steps=a.steps)
    sample = np.random.default_rng(a.seed + 2).choice(a.users, min(a.host_sample, a.users), replace=False)
    for diversity in (False, True):
        offline.evaluate_model(model, T, cutoffs, True, diversity)                 # warm-up of every shape
        torch.cuda.synchronize()
        times, stages_all = [], []
        for _ in range(a.steps):
            torch.cuda.reset_peak_memory_stats()
            stages = {}
            t0 = time.perf_counter()
            res = offline.evaluate_model(model, T, cutoffs, True, diversity, stages=stages)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
            stages_all.append(stages)
        peak = torch.cuda.max_memory_allocated()
        best = int(np.argmin(times))
        host_s = numpy_reference(P, Q, indptr, keys, T, sample, cutoffs, diversity)
        host_full = host_s * res["users"] / len(sample)
        out = dict(base, diversity=diversity, rows=res["users"], e2e_s=[round(t, 4) for t in times],
                   rows_per_s=round(res["users"] / times[best], 1),
                   device_stage_ms={k: round(v, 3) for k, v in stages_all[best].items()},
                   peak_torch_bytes=int(peak), numpy_s=round(host_full, 1), numpy_extrapolated=True,
                   numpy_sample=int(len(sample)), speedup=round(host_full / times[best], 1),
                   metrics={k: v for k, v in res.items() if k != "users"})
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

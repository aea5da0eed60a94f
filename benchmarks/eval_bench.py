"""Validation metrics: host path (Evaluable's Python loop over bfl_topk_host / NumPy scoring) against the device path
(csrc/evaluate.cu through buffalo_b200.evaluate.device) on a generated Zipf CSR.

Every user holds out one item (like a Stream "newest" split), so every user is a validation user.  For each
eval_samples size the device path is timed end to end (host clock around work that ends in a synchronise) and per
stage (CUDA events); the host path is timed on a sample of --host-sample users (its per-user Python sets included) and
extrapolated linearly to the full size, which the output marks with "host_extrapolated".  On the sample both paths
must give the same metrics (1e-12).  One JSON line per size.

    python benchmarks/eval_bench.py --users 1000000 --items 100000 --d 128 --topk 10
"""
import argparse
import json
import sys
import time

import numpy as np

sys.path.insert(0, __file__.rsplit("/benchmarks/", 1)[0])


def zipf_csr(U, I, mean_len, max_len, seed):
    rng = np.random.default_rng(seed)
    lens = np.minimum(rng.zipf(1.8, size=U) * max(1, mean_len // 3), max_len).astype(np.int64)
    pop = 1.0 / np.arange(1, I + 1) ** 0.8
    pop /= pop.sum()
    raw = rng.choice(I, size=int(lens.sum()), p=pop).astype(np.int32)
    owner = np.repeat(np.arange(U, dtype=np.int64), lens)
    key = np.unique(owner * I + raw)                 # sorted, distinct (user, item)
    rows, keys = key // I, (key % I).astype(np.int32)
    indptr = np.cumsum(np.bincount(rows, minlength=U)).astype(np.int64)
    vcol = rng.integers(0, I, size=U).astype(np.int32)
    return indptr, keys, np.arange(U, dtype=np.int32), vcol, np.ones(U, np.float32)


class ArrayData(object):
    def __init__(self, U, I, indptr, keys, vrow, vcol, vval):
        self.header = {"num_users": U, "num_items": I, "num_nnz": len(keys)}
        self.groups = {"rowwise": {"indptr": indptr, "key": keys}, "vali": {"row": vrow, "col": vcol, "val": vval}}

    def get_header(self):
        return self.header

    def get_group(self, name):
        return self.groups[name]

    def has_group(self, name):
        return name in self.groups


def host_ranking(data, P, Q, topk, rows_drawn, eval_samples, seed):
    """Evaluable._evaluate_ranking_metrics on the drawn rows, with the per-user sets built for them only."""
    from buffalo_b200.algo.base import Algo
    from buffalo_b200.algo.options import ALSOption
    from buffalo_b200.evaluate import Evaluable
    from buffalo_b200.misc import aux

    class Host(Algo, Evaluable):
        def normalize(self, group="item"):
            pass

        def _get_feature(self, index, group="item"):
            return None

        def _get_topk_recommendation(self, rows, topk, pool=None):
            return zip(rows, Algo._get_topk_recommendation(self, P[rows], Q, None, None, pool, topk, 1))
    t0 = time.perf_counter()
    indptr, keys = data.groups["rowwise"]["indptr"], data.groups["rowwise"]["key"]
    vrow, vcol = data.groups["vali"]["row"], data.groups["vali"]["col"]
    lens = np.diff(indptr, prepend=0)
    seen = {int(u): set(keys[indptr[u] - lens[u]:indptr[u]].tolist()) for u in rows_drawn}
    gt = {int(u): set() for u in rows_drawn}
    for r, c in zip(vrow[rows_drawn], vcol[rows_drawn]):     # one held-out item per user, row u at position u
        gt[int(r)].add(int(c))
    build_s = time.perf_counter() - t0
    h = Host()
    h.opt = ALSOption().get_default_option()
    h.opt.validation = aux.Option({"topk": topk, "eval_samples": eval_samples})
    h.data = data
    data.vali_data = {"vali_rows": np.arange(len(indptr)), "vali_gt": gt, "validation_seen": seen,
                      "validation_max_seen_size": int(lens.max())}
    np.random.seed(seed)
    t0 = time.perf_counter()
    res = h._evaluate_ranking_metrics()
    return res, build_s + time.perf_counter() - t0


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=1_000_000)
    ap.add_argument("--items", type=int, default=100_000)
    ap.add_argument("--d", type=int, default=128)
    ap.add_argument("--topk", type=int, default=10)
    ap.add_argument("--mean-len", type=int, default=20)
    ap.add_argument("--max-len", type=int, default=5000)
    ap.add_argument("--samples", default="1000,10000,100000,0", help="eval_samples sizes; 0 = all users")
    ap.add_argument("--host-sample", type=int, default=1000)
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "eval_bench.py measures the device path: it needs a GPU"
    from buffalo_b200.evaluate import device
    props = torch.cuda.get_device_properties(0)
    t0 = time.perf_counter()
    indptr, keys, vrow, vcol, vval = zipf_csr(a.users, a.items, a.mean_len, a.max_len, a.seed)
    data = ArrayData(a.users, a.items, indptr, keys, vrow, vcol, vval)
    rng = np.random.default_rng(a.seed + 1)
    P = (rng.normal(size=(a.users, a.d)) * 0.1).astype(np.float32)
    Q = (rng.normal(size=(a.items, a.d)) * 0.1).astype(np.float32)
    model = device.EvalModel(P, Q, None, None, False)
    gen_s = time.perf_counter() - t0
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    device.Evaluation(data, model)            # builds the per-Data state (held-out CSR, seen rows)
    torch.cuda.synchronize()
    state_s = time.perf_counter() - t0
    base = dict(gpu=props.name, users=a.users, items=a.items, nnz=int(len(keys)), d=a.d, topk=a.topk,
                max_seen=int(np.diff(indptr, prepend=0).max()), gen_s=round(gen_s, 2), state_build_s=round(state_s, 3))
    for n in [int(x) for x in a.samples.split(",")]:
        n_eval = a.users if n == 0 else min(n, a.users)
        torch.cuda.reset_peak_memory_stats()
        ev = device.Evaluation(data, model)
        stages = {}
        np.random.seed(a.seed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        ev.ranking(a.topk, n, stages=stages)       # warm-up of the shapes, then the timed call
        torch.cuda.synchronize()
        stages = {}
        np.random.seed(a.seed)
        t0 = time.perf_counter()
        dev = ev.ranking(a.topk, n, stages=stages)
        torch.cuda.synchronize()
        dev_s = time.perf_counter() - t0
        peak = torch.cuda.max_memory_allocated()
        # host on a sample: the same draw, then the first host_sample rows of it
        hs = min(a.host_sample, n_eval)
        np.random.seed(a.seed + 7)
        drawn = np.random.choice(np.arange(a.users), size=hs, replace=False)
        host_res, host_s = host_ranking(data, P, Q, a.topk, drawn, hs, a.seed + 7)
        np.random.seed(a.seed + 7)
        dev_sample = device.Evaluation(data, model).ranking(a.topk, hs)
        diff = float(max(abs(host_res[k] - dev_sample[k]) for k in host_res))
        host_full = host_s * n_eval / hs
        out = dict(base, eval_users=n_eval, device_s=round(dev_s, 4), device_stage_ms={k: round(v, 3) for k, v in stages.items()},
                   device_users_per_s=round(n_eval / dev_s, 1), peak_torch_bytes=int(peak),
                   host_s=round(host_full, 3), host_extrapolated=bool(hs < n_eval), host_sample=hs,
                   host_users_per_s=round(hs / host_s, 1), speedup=round(host_full / dev_s, 1),
                   sample_max_abs_diff=diff, sample_equal=bool(diff <= 1e-12), metrics=dev)
        print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()

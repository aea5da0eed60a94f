#!/usr/bin/env python
"""Per-category caps (DESIGN.md 4.18): ParALS.topk_recommendation(categories=..., category_cap=c) for 131072 users.

Item factors carry a popularity direction (column 0 lognormal, every user's weight on it positive), so the users' top
items overlap as they do in practice.  Category layouts:
  - uniform: every item in one of 1000 categories, uniformly;
  - zipf: 1000 categories of Zipf(1.1) sizes, the largest categories on the most popular items;
  - adversarial: the 4000 most popular items in one category, the rest uniform over 999 others, so a capped row walks
    past thousands of items and needs several rounds.
For each configuration (items, d, topk, cap, layout):
  - stage_ms: the first candidate stage (Serve.topk_device at depth M0 for all users), CUDA events, best of --reps;
  - walk_ms: bfl_category_walk_device over those candidates, CUDA events, best of --reps;
  - rounds: the largest number of walk rounds a row took, and the users still short after the first round;
  - plain_s / capped_s: the public call without and with the caps, end to end, alternated in one process (best of
    --reps each).
The card name and power limit are read in the same run.

  python benchmarks/category_bench.py                          # 100k and 1M items, d = 20 / 128, the default grid
  python benchmarks/category_bench.py --items 100000 --d 20 --topk 10 --cap 1 --layout uniform
Prints one JSON line per configuration."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))


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
    m.P[:, 0] = np.abs(m.P[:, 0]) + 1.0
    m.Q[:, 0] = rng.lognormal(0.0, 1.0, I).astype(np.float32)
    return m


def layout(name, Q, seed):
    rng = np.random.default_rng(seed)
    I = Q.shape[0]
    by_pop = np.argsort(-Q[:, 0], kind="stable")
    cats = np.empty(I, np.int64)
    if name == "uniform":
        cats[:] = rng.integers(0, 1000, I)
    elif name == "zipf":
        sizes = 1.0 / np.arange(1, 1001) ** 1.1
        sizes = np.maximum(1, np.floor(sizes / sizes.sum() * I)).astype(np.int64)
        sizes[0] += I - sizes.sum()
        cats[by_pop] = np.repeat(np.arange(1000), sizes)[:I]
    else:
        cats[:] = rng.integers(1, 1000, I)
        cats[by_pop[:4000]] = 0
    return cats


def events(fn, reps):
    import torch
    fn()
    best = float("inf")
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        b.synchronize()
        best = min(best, a.elapsed_time(b))
    return best


def run(U, I, d, topk, cap, lay, reps, seed=1):
    import torch
    from buffalo_b200 import backend
    from buffalo_b200.parallel import base
    m = model(U, I, d, seed)
    cats = layout(lay, m.Q, seed)
    par = base.ParALS(m)
    users = np.arange(U, dtype=np.int32)
    par.topk_recommendation(users, topk)                      # uploads the items
    h = par._serve
    M0 = base._category_depth(topk)
    q = torch.arange(U, dtype=torch.int32, device="cuda")
    box = {}

    def stage():
        box["c"] = h.topk_device(q, M0)
    stage_ms = events(stage, reps)
    ci, cv = box["c"]
    slots = backend.category_table_slots(topk)
    tc = torch.from_numpy(cats.astype(np.int32)).cuda()
    state = torch.zeros((U, 1 + 2 * slots), dtype=torch.int32, device="cuda")
    oi = torch.full((U, topk), -1, dtype=torch.int32, device="cuda")
    ov = torch.zeros((U, topk), dtype=torch.float32, device="cuda")

    def walk():
        state.zero_()
        backend.category_walk_device(ci, cv, None, tc, cap, topk, state, oi, ov)
    walk_ms = events(walk, reps)
    del ci, cv, state, oi, ov, box["c"]
    stats = []
    real = base._capped_batches
    base._capped_batches = lambda *a, **k: real(*a, **dict(k, stats=stats))
    try:
        par.topk_recommendation(users, topk, categories=cats, category_cap=cap)
    finally:
        base._capped_batches = real
    rounds = 1 + max(r for r, _, _ in stats)
    short = sum(n for r, n, _ in stats if r == 1)
    plain, capped = [], []
    for _ in range(reps):
        torch.cuda.synchronize()
        t = time.perf_counter()
        par.topk_recommendation(users, topk)
        plain.append(time.perf_counter() - t)
        t = time.perf_counter()
        par.topk_recommendation(users, topk, categories=cats, category_cap=cap)
        capped.append(time.perf_counter() - t)
    torch.cuda.empty_cache()
    return dict(users=U, items=I, d=d, topk=topk, cap=cap, layout=lay, M0=M0, stage_ms=round(stage_ms, 3),
                walk_ms=round(walk_ms, 3), rounds=rounds, rows_after_round1=short, plain_s=round(min(plain), 4),
                capped_s=round(min(capped), 4), ratio=round(min(capped) / min(plain), 3), card=card())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--users", type=int, default=131072)
    ap.add_argument("--items", type=int, nargs="+", default=[100000, 1000000])
    ap.add_argument("--d", type=int, nargs="+", default=[20, 128])
    ap.add_argument("--topk", type=int, nargs="+", default=[10, 50])
    ap.add_argument("--cap", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--layout", nargs="+", default=["uniform", "zipf", "adversarial"])
    ap.add_argument("--reps", type=int, default=3)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "category_bench needs a GPU"
    for I in a.items:
        for d in a.d:
            for topk in a.topk:
                for cap in a.cap:
                    for lay in a.layout:
                        print(json.dumps(run(a.users, I, d, topk, cap, lay, a.reps)), flush=True)


if __name__ == "__main__":
    main()

"""Batch serving top-k (csrc/serve.cu through backend.Serve) against today's bfl_topk_device and the NumPy dot_topn.

For every shape (users x items), width d, k and variant (all items / a 10 % pool with an item bias) the factors are
generated on the device and bound to a handle, then `--queries` user rows are served:
  - device_s : Serve.topk_device, CUDA events around the whole call (score + select + merge kernels, no copies);
  - e2e_s    : Serve.topk with host index and result arrays (batches, pinned staging, copies), host clock;
  - topk_device_s : bfl_topk_device on the first `--compare` of those queries (gathered rows; the pool variant on
    gathered item rows, whose gather is not timed), alternated with the handle on the same queries, CUDA events around
    windows of about 0.4 s of back-to-back calls, and the keys and score bits of the two compared;
  - numpy_s  : dot_topn on `--numpy-sample` queries, scaled linearly to `--queries` (marked "numpy_extrapolated").
GFLOP/s = 2 * queries * candidates * d / device_s.  handle_bytes is the device memory the handle holds after the call
beyond the bound factors (candidate scratch, result buffers, pool).  One JSON line per case; the card's name and power
limit are read in the same process.

    python benchmarks/serve_bench.py --queries 1000000
    python benchmarks/serve_bench.py --small 1,4,16,32,64      # calls of a handful of queries, both kernels
    python benchmarks/serve_bench.py --exclude-seen             # the same calls with each user's seen items left out
"""
import argparse
import json
import subprocess
import sys
import time

import numpy as np

sys.path.insert(0, __file__.rsplit("/benchmarks/", 1)[0])


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                             stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, limit = [x.strip() for x in out.split(",")]
        return name, limit
    except Exception:
        return None, "unknown"


def events(fn, repeats, inner=1):
    """Seconds per call of fn, `repeats` windows of `inner` back-to-back calls each between two CUDA events."""
    import torch
    best = []
    for _ in range(repeats):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        for _ in range(inner):
            out = fn()
        b.record()
        b.synchronize()
        best.append(a.elapsed_time(b) / 1e3 / inner)
    return out, best


def calls_for(seconds_per_call, window=0.4):
    """Back-to-back calls that make a timed window about `window` seconds long."""
    return max(1, int(window / max(seconds_per_call, 1e-6)))


def small_calls(a, name, limit):
    """A handful of queries per call: the handle (32-query CTAs, mostly empty) against bfl_topk_device (4-query CTAs) on
    the gathered rows, alternated, every window about 0.4 s of back-to-back calls."""
    import torch
    from buffalo_b200 import backend
    for I in (100_000, 1_000_000):
        for d in (20, 128):
            g = torch.Generator(device="cuda").manual_seed(a.seed)
            P = torch.randn((4096, d), generator=g, device="cuda") * 0.1
            Q = torch.randn((I, d), generator=g, device="cuda") * 0.1
            h = backend.Serve()
            h.bind_items(Q)
            h.bind_queries(P)
            for n in [int(x) for x in a.small.split(",")]:
                qdev = torch.arange(n, dtype=torch.int32, device="cuda")
                rows = P[:n].contiguous()
                new = lambda: h.topk_device(qdev, 10)
                old = lambda: backend.topk_device(rows, Q, None, 10)
                _, t_new = events(new, 1, 3)
                _, t_old = events(old, 1, 3)
                new_s, old_s = [], []
                for _ in range(a.repeats):
                    (oi, ov), t = events(old, 1, calls_for(t_old[0]))
                    old_s += t
                    (ni, nv), t = events(new, 1, calls_for(t_new[0]))
                    new_s += t
                print(json.dumps(dict(gpu=name, power_limit=limit, small_call=True, items=I, d=d, k=10, queries=n,
                                      serve_ms=round(min(new_s) * 1e3, 4), topk_device_ms=round(min(old_s) * 1e3, 4),
                                      serve_ms_all=[round(x * 1e3, 4) for x in new_s],
                                      topk_device_ms_all=[round(x * 1e3, 4) for x in old_s],
                                      speedup_vs_topk_device=round(min(old_s) / min(new_s), 2),
                                      keys_equal=bool(torch.equal(oi, ni)),
                                      score_bits_equal=bool(torch.equal(ov.view(torch.int32), nv.view(torch.int32))))),
                      flush=True)
            h.close()


def seen_histories(U, I, seed):
    """Sorted, duplicate-free rows of U users: Pareto (Zipf-like) lengths, alpha 1.5 and scale 17 (mean about 51),
    capped at 5000; items uniform over [0, I).  Returns (END offsets int64, keys int32)."""
    rng = np.random.default_rng(seed)
    lens = np.minimum((rng.pareto(1.5, U) + 1) * 17, 5000).astype(np.int64)
    rows = np.repeat(np.arange(U, dtype=np.int64), lens)
    keys = rng.integers(0, I, size=len(rows)).astype(np.int64)
    order = np.lexsort((keys, rows))
    rows, keys = rows[order], keys[order]
    keep = np.ones(len(keys), bool)
    keep[1:] = (rows[1:] != rows[:-1]) | (keys[1:] != keys[:-1])
    rows, keys = rows[keep], keys[keep]
    ptr = np.cumsum(np.bincount(rows, minlength=U)).astype(np.int64)
    return ptr, keys.astype(np.int32)


def exclude_seen_calls(a, name, limit):
    """The filtered call (Serve.topk_seen / topk_seen_device) alternated with the unfiltered one on the same handle,
    `--queries` users x {100k, 1M} items, d = 128, k = 10, every user with a history from seen_histories."""
    import torch
    from buffalo_b200 import _cabi, backend
    d, k = 128, 10
    for I in (100_000, 1_000_000):
        U = a.queries
        g = torch.Generator(device="cuda").manual_seed(a.seed)
        P = torch.randn((U, d), generator=g, device="cuda") * 0.1
        Q = torch.randn((I, d), generator=g, device="cuda") * 0.1
        ptr, keys = seen_histories(U, I, a.seed)
        qidx = np.arange(U, dtype=np.int32)
        qdev, dptr, dkeys = (torch.from_numpy(x).cuda() for x in (qidx, ptr, keys))
        h = backend.Serve()
        h.bind_items(Q)
        h.bind_queries(P)
        plain_dev = lambda: h.topk_device(qdev, k)
        # the C entry point itself: Serve.topk_seen_device adds argument checks and a sortedness check that synchronise
        rows = torch.arange(U, dtype=torch.int32, device="cuda")
        s_idx = torch.empty((U, k), dtype=torch.int32, device="cuda")
        s_val = torch.empty((U, k), dtype=torch.float32, device="cuda")
        seen_dev = lambda: (_cabi.check(_cabi.lib().bfl_seen_topk_device(
            h._h, qdev.data_ptr(), U, k, dptr.data_ptr(), dkeys.data_ptr(), rows.data_ptr(), s_idx.data_ptr(),
            s_val.data_ptr(), backend._stream_ptr(None)), "bfl_seen_topk_device"), (s_idx, s_val))[1]
        for fn in (plain_dev, seen_dev):     # warm-up
            fn()
        h.topk(qidx, k)
        h.topk_seen(qidx, k, ptr, keys)
        torch.cuda.synchronize()
        dev = {"plain": [], "seen": []}
        e2e = {"plain": [], "seen": []}
        for _ in range(a.repeats):
            for arm, fn in (("plain", plain_dev), ("seen", seen_dev)):
                out, t = events(fn, 1)
                dev[arm] += t
            for arm in ("plain", "seen"):
                t0 = time.perf_counter()
                res = h.topk(qidx, k) if arm == "plain" else h.topk_seen(qidx, k, ptr, keys)
                e2e[arm].append(time.perf_counter() - t0)
                if arm == "seen":
                    sk = res[0]
        # no seen item comes back: (user, item) pairs as user * I + item, the seen ones sorted already
        lens = np.diff(ptr, prepend=0)
        seen_pairs = np.repeat(np.arange(U, dtype=np.int64), lens) * I + keys
        got = (np.arange(U, dtype=np.int64)[:, None] * I + sk)[sk >= 0]
        at = np.minimum(np.searchsorted(seen_pairs, got), len(seen_pairs) - 1)
        seen_returned = bool((seen_pairs[at] == got).any())
        di, _ = h.topk_seen_device(qdev, k, dptr, dkeys)
        print(json.dumps(dict(
            gpu=name, power_limit=limit, exclude_seen=True, users=U, items=I, d=d, k=k, seen_keys=int(len(keys)),
            mean_history=round(float(lens.mean()), 1), max_history=int(lens.max()),
            device_plain_s=round(min(dev["plain"]), 4), device_seen_s=round(min(dev["seen"]), 4),
            device_ratio=round(min(dev["seen"]) / min(dev["plain"]), 3),
            e2e_plain_s=round(min(e2e["plain"]), 4), e2e_seen_s=round(min(e2e["seen"]), 4),
            e2e_ratio=round(min(e2e["seen"]) / min(e2e["plain"]), 3),
            device_s_all={x: [round(v, 4) for v in dev[x]] for x in dev},
            e2e_s_all={x: [round(v, 4) for v in e2e[x]] for x in e2e},
            seen_item_returned=seen_returned,
            host_and_device_paths_equal=bool(np.array_equal(sk, di.cpu().numpy())))), flush=True)
        h.close()
        del P, Q, qdev, dptr, dkeys, rows, s_idx, s_val
        torch.cuda.empty_cache()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="1000000x100000,10000000x1000000", help="users x items, comma separated")
    ap.add_argument("--d", default="20,128")
    ap.add_argument("--k", default="10,100")
    ap.add_argument("--queries", type=int, default=1_000_000, help="user rows served per case (streamed in batches)")
    ap.add_argument("--compare", type=int, default=16384, help="queries also run through bfl_topk_device")
    ap.add_argument("--numpy-sample", type=int, default=64)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--small", default="", help="e.g. 1,4,16,32,64: time calls of that many queries instead (see small_calls)")
    ap.add_argument("--exclude-seen", action="store_true",
                    help="time the calls that leave each user's seen items out instead (see exclude_seen_calls)")
    ap.add_argument("--seed", type=int, default=0)
    a = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), "serve_bench.py measures the device path: it needs a GPU"
    from buffalo_b200 import backend
    from buffalo_b200.parallel.base import dot_topn
    name, limit = card()
    name = name or torch.cuda.get_device_properties(0).name
    if a.small:
        small_calls(a, name, limit)
        return
    if a.exclude_seen:
        exclude_seen_calls(a, name, limit)
        return
    for shape in a.shapes.split(","):
        U, I = [int(x) for x in shape.split("x")]
        for d in [int(x) for x in a.d.split(",")]:
            g = torch.Generator(device="cuda").manual_seed(a.seed)
            P = torch.randn((U, d), generator=g, device="cuda") * 0.1
            Q = torch.randn((I, d), generator=g, device="cuda") * 0.1
            Qb = torch.randn((I,), generator=g, device="cuda") * 0.1
            rng = np.random.default_rng(a.seed)
            n = min(a.queries, U)
            qidx = rng.permutation(U)[:n].astype(np.int32)
            qdev = torch.from_numpy(qidx).cuda()
            pool = np.sort(rng.permutation(I)[:I // 10]).astype(np.int32)
            for variant in ("all_items", "pool10_bias"):
                for k in [int(x) for x in a.k.split(",")]:
                    torch.cuda.synchronize()
                    free0 = torch.cuda.mem_get_info()[0]
                    h = backend.Serve()
                    h.bind_items(Q, Qb if variant == "pool10_bias" else None)
                    h.bind_queries(P)
                    if variant == "pool10_bias":
                        h.set_pool(pool)
                    ncand = len(pool) if variant == "pool10_bias" else I
                    nc = min(a.compare, n)
                    # warm-up of every shape the timed windows use
                    h.topk_device(qdev[:nc], k)
                    h.topk(qidx[:nc], k)
                    torch.cuda.synchronize()
                    (di, dv), dev_s = events(lambda: h.topk_device(qdev, k), a.repeats)
                    e2e = []
                    for _ in range(a.repeats):
                        t0 = time.perf_counter()
                        hk, hv = h.topk(qidx, k)
                        e2e.append(time.perf_counter() - t0)
                    same_paths = bool(np.array_equal(hk, di.cpu().numpy()))
                    handle_bytes = free0 - torch.cuda.mem_get_info()[0] - (di.numel() + dv.numel()) * 4
                    del di, dv
                    # today's kernels on the same rows, alternated with the handle
                    rows = P[qdev[:nc].long()].contiguous()
                    cand = Q if variant == "all_items" else Q[torch.from_numpy(pool).cuda().long()].contiguous()
                    cb = None if variant == "all_items" else Qb[torch.from_numpy(pool).cuda().long()].contiguous()
                    _, t_old = events(lambda: backend.topk_device(rows, cand, cb, k), 1)
                    _, t_new = events(lambda: h.topk_device(qdev[:nc], k), 1)
                    old_s, new_s = [], []
                    for _ in range(a.repeats):
                        (oi, ov), t = events(lambda: backend.topk_device(rows, cand, cb, k), 1, calls_for(t_old[0]))
                        old_s += t
                        (ni, nv), t = events(lambda: h.topk_device(qdev[:nc], k), 1, calls_for(t_new[0]))
                        new_s += t
                    oi = oi.cpu().numpy() if variant == "all_items" else pool[oi.cpu().numpy()]
                    keys_equal = bool(np.array_equal(oi, ni.cpu().numpy()))
                    bits_equal = bool(torch.equal(ov.view(torch.int32), nv.view(torch.int32)))
                    del rows, cand, cb, oi, ov, ni, nv
                    h.close()
                    # NumPy on a sample, scaled
                    ns = min(a.numpy_sample, n)
                    Ph, Qh = P[qdev[:ns].long()].cpu().numpy(), Q.cpu().numpy()
                    keys = np.zeros((ns, k), np.int32)
                    vals = np.zeros((ns, k), np.float32)
                    t0 = time.perf_counter()
                    dot_topn(np.arange(ns), Ph, Qh, Qb.cpu().numpy() if variant == "pool10_bias" else None, keys, vals,
                             pool if variant == "pool10_bias" else None, k)
                    np_s = (time.perf_counter() - t0) * n / ns
                    del Ph, Qh
                    flop = 2.0 * n * ncand * d
                    ds, es = min(dev_s), min(e2e)
                    print(json.dumps(dict(
                        gpu=name, power_limit=limit, users=U, items=I, d=d, k=k, variant=variant, queries=n,
                        candidates=ncand, device_s=round(ds, 4), device_s_all=[round(x, 4) for x in dev_s],
                        e2e_s=round(es, 4), e2e_s_all=[round(x, 4) for x in e2e], queries_per_s=round(n / es, 1),
                        device_gflops=round(flop / ds / 1e9, 1), e2e_gflops=round(flop / es / 1e9, 1),
                        compare_queries=nc, topk_device_s=round(min(old_s), 4), serve_same_queries_s=round(min(new_s), 4),
                        speedup_vs_topk_device=round(min(old_s) / min(new_s), 2), keys_equal=keys_equal,
                        score_bits_equal=bits_equal, host_and_device_paths_equal=same_paths,
                        handle_bytes=int(handle_bytes), numpy_s=round(np_s, 1), numpy_extrapolated=bool(ns < n),
                        numpy_sample=ns, speedup_vs_numpy=round(np_s / es, 1))), flush=True)
            del P, Q, Qb
            torch.cuda.empty_cache()


if __name__ == "__main__":
    main()

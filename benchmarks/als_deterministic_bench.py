#!/usr/bin/env python
"""ALS iterations with and without the option `deterministic`, in one process on the device-resident path.

  python benchmarks/als_deterministic_bench.py [--workload c5_d128|c5_small|c2|c2_small|tiny] [--steps 3] [--warmup 1]
                                               [--scratch-mb 0] [--no-profile] [--check-iters 3]

Workloads are bench.py's generators (seeded, built on the device): c2 is the C2-shaped CSR at d = 128 (a few split user
rows); c5_small (d = 256) and c5_d128 (d = 128) have Zipf(1.1) items, so the item pass is dominated by split rows.
Both modes start from the same factors; after the warm-up the timed iterations alternate default, deterministic.  CUDA
events time each pass (Gram + row solves of one axis).  Then one iteration per mode runs under torch.profiler and the
device time of the split-row kernels is summed by kernel name:

  default        memset of the row slots | als_tc_kernel<.., PARTIAL> (atomic adds) | als_explicit_solve_kernel
  deterministic  als_tc_kernel<.., PARTIAL, .., DET> (plain stores) | tc_chunk_reduce_kernel | als_explicit_solve_kernel

Prints one JSON line: ms per iteration and per pass in both modes with the runs, the split-row kernel times, the
scratch model (below) with the number of batches and the peak chunk scratch, whether two deterministic runs of
--check-iters iterations from the same start agree bitwise in P, Q and every iteration's loss, the largest relative factor difference between the modes after the timed
iterations, and the card name and power limit read in the same call.

Scratch and byte model of the split rows of one pass (slot = d*d + 2d + 4 floats; a row of n > 1536 entries has
ceil(n / 2048) chunks):
  default        one slot per row: memset (1 write), each chunk added with atomics (read + write of a slot), the
                 explicit solve reads the row's matrix 3 times (h, diagonal blocks, later blocks)
  deterministic  one slot per chunk and per row of the batch in flight: each chunk stored (1 write), the reduce reads
                 every chunk slot and writes every row slot, the explicit solve as above.  Rows are taken in list order
                 into batches of whole rows whose (chunks + 1) slots fit the budget; a batch takes at least one row.
                 The backend bins rows in an order that is not the row order, so its batch count can differ by a few.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)

SPLIT_MIN, TC_SPLIT = 1536, 2048
AUTO_BUDGET_CAP = 2 << 30


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                             stdout=subprocess.PIPE, stderr=subprocess.PIPE, text=True, timeout=30)
        power = out.stdout.strip() or "unknown"
    except Exception:
        power = "unknown"
    return name, power


def slot_bytes(d):
    return 4 * (d * d + 2 * d + 4)


def split_model(lengths, d, budget_bytes):
    """Scratch and byte model of one pass over rows of the given lengths (see the module docstring)."""
    lengths = np.asarray(lengths, dtype=np.int64)
    long_rows = lengths[lengths > SPLIT_MIN]
    chunks = (long_rows + TC_SPLIT - 1) // TC_SPLIT
    sb = slot_bytes(d)
    batches, peak, used = 0, 0, 0
    for nc in chunks:
        cost = int(nc + 1) * sb
        if used and used + cost > budget_bytes:
            batches, peak, used = batches + 1, max(peak, used), 0
        used += cost
    if used:
        batches, peak = batches + 1, max(peak, used)
    nrows, nchunks = int(len(long_rows)), int(chunks.sum())
    solve = 3 * nrows * sb
    return {"split_rows": nrows, "chunks": nchunks, "slot_bytes": sb, "batches": batches, "peak_scratch_bytes": peak,
            "default_scratch_bytes": nrows * sb,
            "default_bytes": nrows * sb + 2 * nchunks * sb + solve,
            "deterministic_bytes": nchunks * sb + (nchunks + nrows) * sb + solve}


def kernel_class(name):
    """Which split-row stage a profiled device activity belongs to, or None."""
    flat = name.replace("(int)", "").replace("(bool)", "").replace(" ", "")
    if "tc_chunk_reduce_kernel" in flat:
        return "chunk_reduce"
    if "als_explicit_solve_kernel" in flat:
        return "explicit_solve"
    if "als_tc_kernel<" in flat:
        args = flat.split("als_tc_kernel<")[1].split(">")[0].split(",")
        if len(args) > 1 and args[1] in ("true", "1"):
            return "partial"
    return None


class Mode(object):
    def __init__(self, opt, wl, P, Q, deterministic):
        import torch
        from buffalo_b200 import backend
        self.det = deterministic
        self.g = backend.CuALS()
        assert self.g.init(dict(opt, deterministic=True) if deterministic else opt), getattr(self.g, "last_error", "")
        self.P, self.Q = P.clone(), Q.clone()
        self.g.bind_factors(self.P, self.Q)
        self.g.bind_csr(0, wl["r_indptr"], wl["r_keys"], wl["vals"])
        self.g.bind_csr(1, wl["c_indptr"], wl["c_keys"], wl["vals"])
        self.U, self.I = wl["U"], wl["I"]
        self.loss = torch.zeros(2, dtype=torch.float64, device=P.device)
        self.torch = torch

    def iteration(self):
        torch = self.torch
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
        self.loss.zero_()
        ev[0].record()
        for axis, rows in ((0, self.U), (1, self.I)):
            self.g.precompute_device(axis)
            self.g.update_device(axis, 0, rows, self.loss)
            ev[axis + 1].record()
        return ev


def profile_split(mode):
    """Device time (ms) of the split-row stages of one iteration."""
    from torch.profiler import ProfilerActivity, profile
    import torch
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        mode.iteration()
        torch.cuda.synchronize()
    out = {"partial": 0.0, "chunk_reduce": 0.0, "explicit_solve": 0.0, "memset": 0.0}
    for e in prof.events():
        t = getattr(e, "device_time", None)
        if t is None:
            t = getattr(e, "cuda_time", 0.0)
        k = kernel_class(e.name)
        if k:
            out[k] += t / 1e3
        elif "memset" in e.name.lower():
            out["memset"] += t / 1e3
    return out


def main():
    import torch
    import bench
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c5_d128", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--scratch-mb", type=float, default=0.0, help="_b200_det_scratch_mb (0: the backend's default)")
    ap.add_argument("--no-profile", action="store_true")
    ap.add_argument("--check-iters", type=int, default=3, help="iterations of each run of the bitwise check")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark measures the GPU; there is no CPU path"
    w = bench.WORKLOADS[args.workload]
    d = w["d"]
    dev = torch.device("cuda", 0)
    wl = bench.make_workload(w, dev)
    U, I = wl["U"], wl["I"]
    opt = dict(bench.ALS_OPT, d=d, compute_loss_on_training=True)
    if args.scratch_mb:
        opt["_b200_det_scratch_mb"] = args.scratch_mb
    P0, Q0 = bench.init_factors_t(U, d, dev, 1), bench.init_factors_t(I, d, dev, 2)
    free_b, _ = torch.cuda.mem_get_info()
    budget = int(args.scratch_mb * (1 << 20)) if args.scratch_mb else min(free_b // 4, AUTO_BUDGET_CAP)

    def lengths(indptr):
        e = indptr.cpu().numpy()
        return np.diff(np.concatenate([[0], e]))
    model = {"user_pass": split_model(lengths(wl["r_indptr"]), d, budget),
             "item_pass": split_model(lengths(wl["c_indptr"]), d, budget), "budget_bytes": budget}

    # two deterministic runs of --check-iters iterations from the same start, on separate handles
    sig = []
    for _ in range(2):
        m = Mode(opt, wl, P0, Q0, True)
        losses = []
        for _ in range(args.check_iters):
            m.iteration()
            losses.append(m.loss.view(torch.int64).clone())
        torch.cuda.synchronize()
        sig.append((m.P.view(torch.int32).clone(), m.Q.view(torch.int32).clone(), torch.stack(losses)))
        del m
    bitwise = all(bool(torch.equal(a, b)) for a, b in zip(*sig))
    del sig
    torch.cuda.empty_cache()

    modes = [Mode(opt, wl, P0, Q0, False), Mode(opt, wl, P0, Q0, True)]
    del P0, Q0
    for _ in range(args.warmup):
        for m in modes:
            m.iteration()
    torch.cuda.synchronize()
    evs = {id(m): [] for m in modes}
    for _ in range(args.steps):
        for m in modes:
            evs[id(m)].append(m.iteration())
    torch.cuda.synchronize()
    name, power = card()
    res = {}
    for m in modes:
        t = [[e[i].elapsed_time(e[i + 1]) for i in range(2)] for e in evs[id(m)]]
        ms = [sum(x) for x in t]
        res["deterministic" if m.det else "default"] = {
            "ms_per_iteration": sum(ms) / len(ms), "ms_per_iteration_runs": ms,
            "ms_per_pass": {"user": sum(x[0] for x in t) / len(t), "item": sum(x[1] for x in t) / len(t)},
            "loss": [float(v) for v in m.loss.cpu().numpy()]}
    a, b = modes
    diff = max(float(((x - y).abs().max() / y.abs().max()).item()) for x, y in ((a.P, b.P), (a.Q, b.Q)))
    if not args.no_profile:
        for m in modes:
            res["deterministic" if m.det else "default"]["split_row_kernel_ms"] = profile_split(m)
    out = {"workload": w["desc"], "d": d, "users": U, "items": I, "nnz": wl["nnz"], "steps": args.steps,
           "warmup": args.warmup, "card": name, "power_limit": power, "split_row_model": model,
           "deterministic_runs_bitwise_equal": bitwise, "bitwise_check_iterations": args.check_iters, "results": res,
           "deterministic_over_default": res["deterministic"]["ms_per_iteration"] / res["default"]["ms_per_iteration"],
           "max_rel_factor_diff_default_vs_deterministic": diff}
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

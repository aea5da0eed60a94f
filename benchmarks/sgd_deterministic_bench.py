#!/usr/bin/env python
"""BPRMF / WARP epochs with and without the option `deterministic`, in one process on the device-resident path.

  python benchmarks/sgd_deterministic_bench.py [--workload c3|c3_small|c4|c4_small] [--steps 3] [--warmup 1]
                                               [--optimizer adagrad] [--modes both|default|deterministic]

The workloads are those of benchmarks/sgd_bench.py (C3: BPRMF d = 128, 10M x 1M, 500M positives; C4: WARP d = 64,
1M x 100k, 50M positives, reference defaults), trained with an accumulating optimizer (adagrad unless --optimizer says
otherwise; plain SGD has no deterministic mode).  Both modes start from the same factors.  After the warm-up epochs the
timed epochs alternate: one default epoch, then one deterministic epoch.  CUDA events time every pass:

  default        accumulate (add_jobs_device: sample + atomic accumulate) | optimizer (update_parameters_device)
  deterministic  sample + user pass (add_jobs_device) | item pass (reduce_items_device: sort + item sums) | optimizer

Prints one JSON line: ms per epoch and per pass, positives/s, the byte model of each pass (below), the device memory in
use after each pass (cudaMemGetInfo, the most seen), the card name and power limit, and the largest factor difference
between the two modes after the timed epochs (relative to the largest factor).

Byte model per epoch (N samples; rows of 4d bytes; a warp gathers whole rows):
  default accumulate   BPR: per sample P, Q_i, Q_j read and three gradient rows added (atomics: read + write) = 36d + 12
                       WARP: per positive (2 + E[trials]) rows read and three gradient rows added
  sample pass          BPR: 12d read + 36 record and entry bytes written per sample; WARP: (2 + E[trials]) rows + 40
  user pass            per sample the record (12) and two Q rows (8d); per user the gradient row read and written (8d)
  item pass            the stable radix sort of 2N (item, 2s + side, coefficient) entries, 3 digit passes of 24 bytes
                       each plus 40 for keys in and out; then per entry code, coefficient, user (12) and a P row (4d);
                       per item the gradient row read and written (8d)
  optimizer            theta, gradient and state of P and Q streamed (6 rows adagrad, 8 adam) per row
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "benchmarks"))


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


def byte_model(algo, d, nnz, users, items, optimizer, trials):
    n = nnz      # one negative per positive in both workloads
    row = 4 * d
    opt = (users + items) * row * (6 if optimizer == "adagrad" else 8)
    if algo == "bpr":
        default_acc = n * (9 * row + 12)
        sample = n * (3 * row + 36)
    else:
        default_acc = n * ((2 + trials) * row + 6 * row + 4)
        sample = n * ((2 + trials) * row + 40)
    user = n * (12 + 2 * row) + users * 2 * row
    item = 2 * n * (3 * 24 + 40) + 2 * n * (12 + row) + items * 2 * row
    return {"default": {"accumulate": default_acc, "optimizer": opt},
            "deterministic": {"sample_user": sample + user, "item": item, "optimizer": opt}}


class Mode(object):
    def __init__(self, algo, opt, wl, P, Q, Qb, deterministic):
        import torch
        from buffalo_b200 import backend
        self.det = deterministic
        self.g = g = backend.CuSGD(algo)
        assert g.init(dict(opt, deterministic=True) if deterministic else opt), getattr(g, "last_error", "")
        self.P, self.Q, self.Qb = P.clone(), Q.clone(), Qb.clone()
        g.bind_factors(self.P, self.Q, self.Qb, wl["nnz"])
        g.bind_csr(wl["r_indptr_dev"], wl["r_keys"])
        g.launch_workers()
        self.U = wl["U"]
        self.times = []
        self.torch = torch

    def epoch(self, mem):
        torch = self.torch
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(4)]
        ev[0].record()
        self.g.add_jobs_device(0, self.U)
        ev[1].record()
        mem.sample()
        if self.det:
            self.g.reduce_items_device()
        ev[2].record()
        mem.sample()
        self.g.update_parameters_device()
        ev[3].record()
        return ev


class Mem(object):
    def __init__(self):
        import torch
        self.torch = torch
        self.peak = 0

    def sample(self):
        free, total = self.torch.cuda.mem_get_info()
        self.peak = max(self.peak, total - free)


def main():
    import torch
    import bench
    from sgd_bench import SGD_WORKLOADS, sgd_options
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c4_small", choices=sorted(SGD_WORKLOADS))
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--optimizer", default="adagrad", choices=["adagrad", "adam"])
    ap.add_argument("--modes", default="both", choices=["both", "default", "deterministic"])
    args = ap.parse_args()
    w = SGD_WORKLOADS[args.workload]
    algo, d = w["algo"], w["d"]
    dev = torch.device("cuda", 0)
    wl = bench.make_workload(dict(users=w["users"], items=w["items"], nnz=w["nnz"]), dev,
                             seed=2025 if algo == "bpr" else 2026)
    for k in ("c_indptr", "c_keys", "vals"):     # the SGD epoch reads the rowwise keys only
        wl.pop(k, None)
    wl["r_indptr_dev"] = wl["r_indptr"]
    U, I, nnz = wl["U"], wl["I"], wl["nnz"]
    opt = sgd_options(algo, d, args.steps + args.warmup, args.optimizer)
    gen = torch.Generator(device=dev)
    gen.manual_seed(1)
    P = torch.randn(U, d, device=dev, generator=gen) * (1.0 / d ** 2)
    Q = torch.randn(I, d, device=dev, generator=gen) * (1.0 / d ** 2)
    if algo == "bpr":
        P, Q = P.abs_(), Q.abs_()
    Qb = torch.zeros(I, 1, device=dev)
    mem = Mem()
    mem.sample()
    base_mem = mem.peak
    modes = []
    if args.modes in ("both", "default"):
        modes.append(Mode(algo, opt, wl, P, Q, Qb, False))
    if args.modes in ("both", "deterministic"):
        modes.append(Mode(algo, opt, wl, P, Q, Qb, True))
    del P, Q
    for _ in range(args.warmup):
        for m in modes:
            m.epoch(mem)
    torch.cuda.synchronize()
    evs = {id(m): [] for m in modes}
    for _ in range(args.steps):
        for m in modes:
            evs[id(m)].append(m.epoch(mem))
    torch.cuda.synchronize()
    trials = 2.0
    name, power = card()
    bm = byte_model(algo, d, nnz, U, I, opt["optimizer"], trials)
    res = {}
    for m in modes:
        t = [[e[i].elapsed_time(e[i + 1]) for i in range(3)] for e in evs[id(m)]]
        ms = [sum(x) for x in t]
        per = [sum(x[i] for x in t) / len(t) for i in range(3)]
        key = "deterministic" if m.det else "default"
        passes = (["sample_user", "item", "optimizer"] if m.det else ["accumulate", "-", "optimizer"])
        res[key] = {"ms_per_epoch": sum(ms) / len(ms), "ms_per_epoch_runs": ms,
                    "ms_per_pass": {p: v for p, v in zip(passes, per) if p != "-"},
                    "positives_per_s": nnz / (sum(ms) / len(ms) / 1e3),
                    "bytes_per_pass": bm[key],
                    "GBps_per_pass": {p: bm[key][p] / (v / 1e3) / 1e9 for p, v in zip(passes, per) if p != "-" and v > 0}}
    out = {"workload": w["desc"], "algo": algo, "d": d, "users": U, "items": I, "nnz": nnz, "optimizer": opt["optimizer"],
           "steps": args.steps, "warmup": args.warmup, "card": name, "power_limit": power,
           "device_memory_in_use_GB": {"before_holders": base_mem / 1e9, "peak_sampled": mem.peak / 1e9},
           "byte_model_trials_assumed": trials if algo == "warp" else None, "results": res}
    if len(modes) == 2:
        a, b = modes
        diffs = [((x - y).abs() / y.abs().max()) for x, y in ((a.P, b.P), (a.Q, b.Q))]
        out["max_rel_factor_diff_default_vs_deterministic"] = max(float(t.max()) for t in diffs)
        # the reference start abs(N(0, 1/d^2)) leaves most gradients near zero, and the first Adagrad / Adam step
        # g / (|g| + eps) takes their sign, which rounding decides; the share of such elements is the telling figure
        out["share_of_elements_above_1e-3_rel"] = (sum(float((t > 1e-3).sum()) for t in diffs) /
                                                   sum(t.numel() for t in diffs))
        out["deterministic_over_default"] = res["deterministic"]["ms_per_epoch"] / res["default"]["ms_per_epoch"]
    print(json.dumps(out), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

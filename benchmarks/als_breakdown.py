#!/usr/bin/env python
"""Device time per kernel of one ALS iteration, split into the user pass and the item pass.

  python benchmarks/als_breakdown.py [--workload c2] [--warmup 3] [--debug 1,2,12] [--out DIR]

Builds the workload of bench.py (same generator, seeds and options), runs warm-up iterations, then profiles one
iteration with torch.profiler (CUDA activities), one profiler session per half-epoch so that every kernel -- the Gram of
the opposite factor included -- is charged to the pass that launched it.  The traces go to DIR (default: a temporary
directory) as <tag>_<pass>.pt.trace.json; the tables (kernel class, launches, device ms) go to stdout.

--debug repeats the breakdown once per listed BFL_TC_DEBUG value of the tensor-core kernel (timing experiments: the
results of such an iteration are wrong by design, so the factors are re-initialised after every run).
"""
import argparse
import json
import os
import re
import sys
import tempfile
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402

PASSES = ("user", "item")


def kernel_class(name):
    if "gram_partial_kernel" in name or "gram_reduce_kernel" in name:
        return "Gram"
    if "tc_absmax_kernel" in name or "tc_scale_kernel" in name:
        return "absmax / scale"
    m = re.search(r"als_tc_kernel<(\d+), (true|false), (true|false)>", name)
    if m:
        kind = "split-row partial" if m.group(2) == "true" else "fused"
        return "tensor-core %s d=%s%s" % (kind, m.group(1), " (loss)" if m.group(3) == "true" else "")
    if "als_explicit_solve_kernel" in name:
        return "split-row explicit solve"
    m = re.search(r"als_ialspp_team_kernel<([^>]*)>", name)
    if m:
        return "SIMT team <%s>" % m.group(1)
    return re.sub(r"\(.*$", "", name).replace("void ", "")[:80]


def kernel_times(trace_path):
    """{class: [launches, device ms]} from the kernel events of a chrome trace."""
    with open(trace_path) as f:
        ev = json.load(f)["traceEvents"]
    out = defaultdict(lambda: [0, 0.0])
    for e in ev:
        if e.get("cat") == "kernel" and e.get("ph") == "X":
            c = out[kernel_class(e["name"])]
            c[0] += 1
            c[1] += float(e["dur"]) / 1e3
    return out


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--workload", default="c2", choices=sorted(bench.WORKLOADS))
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--debug", default="", help="comma-separated BFL_TC_DEBUG values to repeat the breakdown with")
    ap.add_argument("--out", default=None, help="directory for the traces (default: a temporary directory)")
    args = ap.parse_args()

    import torch
    from torch.profiler import ProfilerActivity, profile
    assert torch.cuda.is_available(), "als_breakdown.py needs a GPU"
    out_dir = args.out or tempfile.mkdtemp(prefix="als_breakdown_")
    os.makedirs(out_dir, exist_ok=True)
    device = torch.device("cuda", 0)
    torch.cuda.set_device(device)
    from buffalo_b200 import backend
    from buffalo_b200.parallel.dist import ShardedALS

    w = bench.WORKLOADS[args.workload]
    d = w["d"]
    wl = bench.make_workload(w, device)
    P = bench.init_factors_t(wl["U"], d, device, 7)
    Q = bench.init_factors_t(wl["I"], d, device, 8)
    obj = backend.CuALS()
    assert obj.init(dict(bench.ALS_OPT, d=d, _b200_kernel_mode=0)), obj.last_error
    obj.bind_factors(P, Q)
    obj.bind_csr(0, wl["r_indptr"], wl["r_keys"], wl["vals"])
    obj.bind_csr(1, wl["c_indptr"], wl["c_keys"], wl["vals"])
    drv = ShardedALS(obj.precompute_device, obj.update_device, P, Q)
    name = torch.cuda.get_device_name(0)
    print("# %s, workload %s: U=%d I=%d nnz=%d d=%d" % (name, args.workload, wl["U"], wl["I"], wl["nnz"], d))

    def run(tag):
        for _ in range(args.warmup):
            drv.iteration()
        torch.cuda.synchronize()
        tables = {}
        for axis, pname in enumerate(PASSES):
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                drv.half_epoch(axis)
                torch.cuda.synchronize()
            path = os.path.join(out_dir, "%s_%s.pt.trace.json" % (tag, pname))
            prof.export_chrome_trace(path)
            tables[pname] = kernel_times(path)
        print("\n## %s" % tag)
        print("| pass | kernel class | launches | device ms |")
        print("|---|---|---|---|")
        for pname in PASSES:
            t = tables[pname]
            for cls, (n, ms) in sorted(t.items(), key=lambda kv: -kv[1][1]):
                print("| %s | %s | %d | %.1f |" % (pname, cls, n, ms))
            print("| %s | **total** | %d | **%.1f** |" % (pname, sum(v[0] for v in t.values()), sum(v[1] for v in t.values())))
        sys.stdout.flush()

    run("default")
    for dbg in [x for x in args.debug.split(",") if x.strip()]:
        os.environ["BFL_TC_DEBUG"] = dbg.strip()
        run("BFL_TC_DEBUG=%s" % dbg.strip())
        os.environ.pop("BFL_TC_DEBUG")
        P.copy_(bench.init_factors_t(wl["U"], d, device, 7))   # a debug iteration leaves wrong factors behind
        Q.copy_(bench.init_factors_t(wl["I"], d, device, 8))
    print("\n# traces: %s" % out_dir)
    return 0


if __name__ == "__main__":
    sys.exit(main())

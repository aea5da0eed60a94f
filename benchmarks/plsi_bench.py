#!/usr/bin/env python
"""Throughput of the pLSI EM iteration on the device-resident path: the C2-shaped synthetic rowwise CSR of bench.py
(10M users x 1M items, 1B nonzeros, clipped-lognormal row degrees) at d = 20 and d = 128.

  python benchmarks/plsi_bench.py [--workload c2|c2_small|c5|c5_small|tiny] [--steps 3] [--warmup 1] [--dims 20,128]
                                  [--deterministic]

CUDA events time the EM pass (bfl_plsi_update_device) and the normalize pass (bfl_plsi_normalize_device +
bfl_plsi_swap_device) separately.  Prints one JSON line with nnz/s per iteration, both kernel times, the algorithmic
byte model below, the HBM share it implies, and the card name and power limit read in the same run.

Byte model of the EM pass, per nonzero: the gathered item row (4d), the key and the value (8); per user row: the P row
read and written (8d) and its end offset (8).  The atomic read-modify-write of the new item row (8d per nonzero) is
reported as its own term: it lands in L2 when the item matrix fits there and in HBM when it does not.  The normalize
pass reads and writes P once and reads the item accumulator twice and writes it once, then copies it into Q.

--deterministic times the deterministic mode: the item pass over the colwise CSR (bfl_plsi_update_items_device) and
the row pass without item accumulation, separately.  Its byte model has no atomic term: each pass moves 4d + 8 bytes
per nonzero (the gathered row of the other side, key, value), plus per major row its own row read and written and its
end offset (8d + 8).  The c5 workloads (Zipf(1.1) items, bench.make_workload_zipf) put millions of entries on the top
items, which the item pass cuts into fixed segments.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "..")
sys.path.insert(0, ROOT)


def em_bytes(d, nnz, users):
    return nnz * (4 * d + 8) + users * (8 * d + 8)


def item_pass_bytes(d, nnz, items):
    return nnz * (4 * d + 8) + items * (8 * d + 8)


def atomic_bytes(d, nnz):
    return nnz * 8 * d


def normalize_bytes(vdim, users, items):
    return users * 8 * vdim + items * 4 * vdim * 3 + items * 8 * vdim


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


def run_dim(wl, d, steps, warmup, deterministic=False):
    import torch
    from buffalo_b200 import backend
    dev = wl["r_indptr"].device
    U, I, nnz = wl["U"], wl["I"], wl["nnz"]
    g = backend.CuPLSI()
    assert g.init(dict(d=d, random_seed=1, deterministic=deterministic))
    vdim = g.get_vdim()
    gen = torch.Generator(device=dev)
    gen.manual_seed(3)
    P = torch.zeros(U, vdim, device=dev)
    Q = torch.zeros(I, vdim, device=dev)
    P[:, :d] = torch.rand(U, d, device=dev, generator=gen) + 1e-3
    Q[:, :d] = torch.rand(I, d, device=dev, generator=gen) + 1e-3
    P /= P.sum(dim=1, keepdim=True)
    Q /= Q.sum(dim=0, keepdim=True).clamp_min(1e-30)
    g.bind_factors(P, Q)
    g.bind_csr(wl["r_indptr"], wl["r_keys"], wl["vals"])
    if deterministic:
        g.bind_colwise_csr(wl["c_indptr"], wl["c_keys"], wl["vals"])    # the values are all 1: one array serves both
    loss = torch.zeros(1, dtype=torch.float64, device=dev)
    ev = [[torch.cuda.Event(enable_timing=True) for _ in range(4)] for _ in range(steps)]
    for i in range(warmup + steps):
        loss.zero_()
        e = ev[i - warmup] if i >= warmup else None
        if e:
            e[0].record()
        if deterministic:
            g.update_items_device(0, I)
        if e:
            e[1].record()
        g.update_device(0, U, loss)
        if e:
            e[2].record()
        g.normalize_device(1.0, 1.0)
        g.swap_device()
        if e:
            e[3].record()
    torch.cuda.synchronize()
    item_ms = sum(e[0].elapsed_time(e[1]) for e in ev) / steps
    em_ms = sum(e[1].elapsed_time(e[2]) for e in ev) / steps
    nrm_ms = sum(e[2].elapsed_time(e[3]) for e in ev) / steps
    finite = bool(torch.isfinite(P).all().item() and torch.isfinite(Q).all().item())
    import bench
    peak, peak_src = bench.measured_peak()
    eb, ab, nb = em_bytes(d, nnz, U), atomic_bytes(d, nnz), normalize_bytes(vdim, U, I)
    if deterministic:
        ib = item_pass_bytes(d, nnz, I)
        out = {"d": d, "vdim": vdim, "mode": "deterministic", "nnz_per_s": nnz / ((item_ms + em_ms + nrm_ms) / 1e3),
               "item_pass_ms": item_ms, "row_pass_ms": em_ms, "normalize_ms": nrm_ms,
               "loss_last": float(loss.item()), "finite": finite,
               "bytes": {"item_pass": ib, "row_pass": eb, "normalize": nb},
               "achieved_gbs": {"item_pass": ib / (item_ms / 1e3) / 1e9, "row_pass": eb / (em_ms / 1e3) / 1e9,
                                "normalize": nb / (nrm_ms / 1e3) / 1e9},
               "hbm_share": {"item_pass": ib / (item_ms / 1e3) / 1e9 / peak, "row_pass": eb / (em_ms / 1e3) / 1e9 / peak},
               "peak_gbs": peak, "peak_source": peak_src}
        del g, P, Q
        torch.cuda.empty_cache()
        return out
    out = {"mode": "default", "d": d, "vdim": vdim, "nnz_per_s": nnz / ((em_ms + nrm_ms) / 1e3), "em_ms": em_ms, "normalize_ms": nrm_ms,
           "em_nnz_per_s": nnz / (em_ms / 1e3), "loss_last": float(loss.item()), "finite": finite,
           "bytes": {"em": eb, "em_atomic_rmw": ab, "normalize": nb},
           "achieved_gbs": {"em": eb / (em_ms / 1e3) / 1e9, "em_with_atomics": (eb + ab) / (em_ms / 1e3) / 1e9,
                            "normalize": nb / (nrm_ms / 1e3) / 1e9},
           "hbm_share": {"em": eb / (em_ms / 1e3) / 1e9 / peak, "em_with_atomics": (eb + ab) / (em_ms / 1e3) / 1e9 / peak,
                         "normalize": nb / (nrm_ms / 1e3) / 1e9 / peak},
           "peak_gbs": peak, "peak_source": peak_src}
    del g, P, Q
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--workload", default="c2", choices=["c2", "c2_small", "c5", "c5_small", "tiny"])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--dims", default="20,128")
    ap.add_argument("--deterministic", action="store_true", help="time the deterministic item pass + row pass")
    args = ap.parse_args()
    import torch
    import bench
    assert torch.cuda.is_available(), "needs a GPU: there is no CPU fallback"
    torch.cuda.set_device(0)
    dev = torch.device("cuda", 0)
    w = bench.WORKLOADS[args.workload]
    wl = bench.make_workload({k: v for k, v in w.items() if k in ("users", "items", "nnz", "zipf")}, dev)
    if not args.deterministic:
        del wl["c_indptr"], wl["c_keys"]            # the default mode reads the rowwise orientation only
    torch.cuda.empty_cache()
    name, power = card()
    res = [run_dim(wl, int(d), args.steps, args.warmup, args.deterministic) for d in args.dims.split(",")]
    clens = torch.diff(wl["c_indptr"], prepend=wl["c_indptr"].new_zeros(1)) if args.deterministic else None
    print(json.dumps({"metric": "pLSI EM iteration nnz/s (device-resident)", "workload": args.workload,
                      "mode": "deterministic" if args.deterministic else "default",
                      "max_item_nnz": int(clens.max().item()) if clens is not None else None,
                      "users": wl["U"], "items": wl["I"], "nnz": wl["nnz"], "steps": args.steps, "warmup": args.warmup,
                      "card": name, "power_limit": power, "results": res}), flush=True)
    return 0


if __name__ == "__main__":
    sys.exit(main())

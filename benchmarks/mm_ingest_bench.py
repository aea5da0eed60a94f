"""MatrixMarket text -> database: the host path (pandas + NumPy) against the device parser (csrc/mm_ingest.cu).

Writes a seeded C2-shaped file (10M users x 1M items by default; clipped-lognormal row degrees, integer values 1..5, or
quarter-step decimals with --decimal) into --out, then runs MatrixMarket.create() through each path in a child process
and prints one JSON line per run: wall time, text GB/s, entries/s, the child's peak RSS, per-stage device time from CUDA
events and the peak of the device memory pool (device path), with the card name and power limit read in the same run.
The device path runs twice: first after evicting the file from the page cache (posix_fadvise DONTNEED, "cold"), then
with the file cached ("warm").  The host path runs up to --host-max entries, and the two databases are compared
bitwise.  Generation is not timed.

    python benchmarks/mm_ingest_bench.py --out /tmp/mmb --nnz 1e8
    python benchmarks/mm_ingest_bench.py --out /tmp/mmb --nnz 1e9       # device path only
"""
import argparse
import json
import os
import resource
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402


def generate(path, nnz, U, I, decimal, seed=0):
    from tests.mm_files import format_lines
    rng = np.random.default_rng(seed)
    if nnz < U:
        raise SystemExit("--nnz must be at least --users (every row gets one entry)")
    w = np.clip(rng.lognormal(0.0, 1.5, U), 0.0, float(I))
    deg = 1 + np.floor((nnz - U) * w / w.sum()).astype(np.int64)
    deg[: nnz - int(deg.sum())] += 1                  # the rounding remainder, < U
    kind = "real" if decimal else "integer"
    with open(path, "wb") as f:
        f.write(("%%%%MatrixMarket matrix coordinate %s general\n%d %d %d\n" % (kind, U, I, int(deg.sum()))).encode())
        starts = np.concatenate([[0], np.cumsum(deg)])
        u0 = 0
        while u0 < U:
            u1 = int(np.searchsorted(starts, starts[u0] + 4_000_000, side="right"))
            u1 = min(U, max(u1 - 1, u0 + 1))
            rows = np.repeat(np.arange(u0, u1) + 1, deg[u0:u1])
            cols = rng.integers(1, I + 1, len(rows))
            vals = rng.integers(4, 21, len(rows)) if decimal else rng.integers(1, 6, len(rows))
            f.write(format_lines(rows, cols, U, I, vals, decimal))
            if (u0 * 20) // U != (u1 * 20) // U:
                print("generate: %d of %d rows" % (u1, U), file=sys.stderr, flush=True)
            u0 = u1
    return int(deg.sum())


def child(src, db_path, device):
    from buffalo_b200.data import mm as mmmod
    from buffalo import MatrixMarket, MatrixMarketOptions
    mmmod.DEVICE_INGEST_MIN_BYTES = 0 if device else 1 << 62
    opt = MatrixMarketOptions().get_default_option()
    opt.input.main = src
    opt.data.tmp_dir = os.path.dirname(db_path)
    opt.data.path = db_path
    np.random.seed(0)
    if device:
        import torch
        torch.cuda.init()
        from buffalo_b200 import _cabi
        _cabi.lib()
    t0 = time.perf_counter()
    db = MatrixMarket(opt)
    write = []
    orig = db._write_database

    def timed_write(*a, **kw):                         # the database write is common to both paths
        t = time.perf_counter()
        orig(*a, **kw)
        write.append(time.perf_counter() - t)
    db._write_database = timed_write
    db.create()
    wall = time.perf_counter() - t0
    out = dict(wall_s=wall, write_db_s=sum(write), peak_rss_gb=resource.getrusage(resource.RUSAGE_SELF).ru_maxrss * 1024 / 1e9,
               nnz=int(db.get_header()["num_nnz"]))
    if hasattr(db, "ingest_stats"):
        st = db.ingest_stats
        out.update(device_path=True, device_ms=st["device_ms"], host_ms=st["host_ms"],
                   peak_device_gb=st["peak_device_bytes"] / 1e9)
    else:
        out.update(device_path=False)
    print("CHILD " + json.dumps(out), flush=True)


def run_child(src, db_path, device):
    r = subprocess.run([sys.executable, os.path.abspath(__file__), "--child", src, db_path, "1" if device else "0"],
                       stdout=subprocess.PIPE, text=True)
    if r.returncode != 0:
        raise RuntimeError("child failed:\n" + r.stdout[-4000:])
    return json.loads([ln for ln in r.stdout.splitlines() if ln.startswith("CHILD ")][-1][6:])


def evict(path):
    fd = os.open(path, os.O_RDONLY)
    try:
        os.fsync(fd)                                      # dirty pages are not dropped
        os.posix_fadvise(fd, 0, 0, os.POSIX_FADV_DONTNEED)
    finally:
        os.close(fd)


def same_db(a, b):
    za, zb = np.load(a, allow_pickle=False), np.load(b, allow_pickle=False)
    if sorted(za.files) != sorted(zb.files):
        return False
    for k in za.files:
        x, y = za[k], zb[k]
        if x.dtype != y.dtype or x.shape != y.shape or x.tobytes() != y.tobytes():
            return False
    return True


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        pl = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=power.limit", "--format=csv,noheader"],
                            stdout=subprocess.PIPE, text=True, timeout=30).stdout.strip()
    except Exception as e:  # no nvidia-smi: say so rather than guess
        pl = "unknown (%s)" % type(e).__name__
    return name, pl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the generated file and the databases")
    ap.add_argument("--nnz", type=float, default=1e8)
    ap.add_argument("--users", type=int, default=10_000_000)
    ap.add_argument("--items", type=int, default=1_000_000)
    ap.add_argument("--decimal", action="store_true")
    ap.add_argument("--host-max", type=float, default=1e8, help="largest nnz the host path is run at")
    ap.add_argument("--keep", action="store_true", help="keep the generated file and databases")
    args = ap.parse_args()
    os.makedirs(args.out, exist_ok=True)
    nnz = int(args.nnz)
    src = os.path.join(args.out, "c2_%d%s.mtx" % (nnz, "_dec" if args.decimal else ""))
    t0 = time.perf_counter()
    if not os.path.isfile(src):
        generate(src, nnz, args.users, args.items, args.decimal)
    gen_s = time.perf_counter() - t0
    size = os.path.getsize(src)
    name, pl = card()
    base = dict(bench="mm_ingest", nnz=nnz, users=args.users, items=args.items, decimal=args.decimal,
                text_gb=size / 1e9, gpu=name, power_limit=pl, generate_s=gen_s)
    results = []
    runs = [("device", True, "cold"), ("device", True, "warm")]
    if nnz <= args.host_max:
        runs.append(("host", False, "warm"))
    dbs = {}
    for label, device, cache in runs:
        db = os.path.join(args.out, "%s.h5py" % label)
        if cache == "cold":
            evict(src)
        else:
            with open(src, "rb") as f:                   # make sure the text is cached
                while f.read(1 << 26):
                    pass
        r = run_child(src, db, device)
        r.update(base, path=label, page_cache=cache, text_gb_per_s=size / 1e9 / r["wall_s"],
                 entries_per_s=nnz / r["wall_s"])
        print(json.dumps(r), flush=True)
        results.append(r)
        dbs[label] = db
    if "host" in dbs:
        eq = same_db(dbs["device"], dbs["host"])
        print(json.dumps(dict(base, bitwise_equal=eq)), flush=True)
        if not eq:
            sys.exit(1)
    if not args.keep:
        for p in list(dbs.values()) + [src]:
            if os.path.exists(p):
                os.remove(p)


if __name__ == "__main__":
    if len(sys.argv) > 1 and sys.argv[1] == "--child":
        child(sys.argv[2], sys.argv[3], sys.argv[4] == "1")
    else:
        main()

"""Stream session text -> database: the host loop against the device parser (csrc/stream_ingest.cu).

Writes seeded Zipf sessions with a C2-like shape (10M users, a vocabulary of 1M item tokens "i<k>", Zipf(1.1) item
draws, clipped-lognormal session lengths) into --out, optionally with an iid file listing the vocabulary, then runs
Stream.create() through each path in a child process, for both internal data types, and prints one JSON line per run:
wall time, tokens/s, text GB/s, the child's peak RSS, per-stage device time from CUDA events and the peak of the device
memory pool (device path), with the card name and power limit read in the same run.  The host path runs up to
--host-max tokens, and there the two databases are compared bitwise.  Generation is not timed.

    python benchmarks/stream_ingest_bench.py --out /tmp/sib --tokens 1e8
    python benchmarks/stream_ingest_bench.py --out /tmp/sib --tokens 1e9 --host-max 0
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


def generate(path, iid_path, tokens, U, V, seed=0):
    rng = np.random.default_rng(seed)
    w = np.clip(rng.lognormal(0.0, 1.2, U), 0.0, 1e4)
    deg = np.floor(tokens * w / w.sum()).astype(np.int64)
    deg[: tokens - int(deg.sum())] += 1
    vocab = [("i%d" % k).encode() for k in range(V)]
    vlen = np.array([len(v) for v in vocab], np.int64)
    vbuf = np.frombuffer(b"".join(vocab), np.uint8)
    voff = np.concatenate([[0], np.cumsum(vlen)[:-1]])
    with open(iid_path, "wb") as f:
        f.write(b"\n".join(vocab) + b"\n")
    starts = np.concatenate([[0], np.cumsum(deg)])
    with open(path, "wb") as f:
        u0 = 0
        while u0 < U:
            u1 = int(np.searchsorted(starts, starts[u0] + 10_000_000, side="right"))
            u1 = min(U, max(u1 - 1, u0 + 1))
            d = deg[u0:u1]
            n = int(d.sum())
            ids = np.minimum(rng.zipf(1.1, n) - 1, V - 1)
            ln = vlen[ids] + 1                                  # token and its separator
            end = np.cumsum(ln)
            out = np.empty(int(end[-1]) if n else 0, np.uint8)
            tok = np.repeat(np.arange(n), vlen[ids])            # the token of every name byte
            k = np.arange(len(tok)) - np.repeat(np.cumsum(vlen[ids]) - vlen[ids], vlen[ids])
            out[(end - ln)[tok] + k] = vbuf[voff[ids][tok] + k]
            last = np.cumsum(d)[d > 0] - 1                    # the last token of each non-empty session ends its line
            sep = np.full(n, 32, np.uint8)
            sep[last] = 10
            out[end - 1] = sep
            empties = int((d == 0).sum())
            f.write(out.tobytes())
            if empties:
                f.write(b"\n" * empties)                      # the chunk's empty sessions come after its others
            u0 = u1
    return int(deg.sum())


def child(src, iid, db_path, device, matrix):
    from buffalo_b200.data import stream as smod
    from buffalo import Stream, StreamOptions
    smod.DEVICE_INGEST_MIN_BYTES = 0 if device else 1 << 62
    opt = StreamOptions().get_default_option()
    opt.input.main = src
    opt.input.iid = iid or ""
    opt.data.tmp_dir = os.path.dirname(db_path)
    opt.data.path = db_path
    opt.data.internal_data_type = "matrix" if matrix else "stream"
    np.random.seed(1)
    t0 = time.perf_counter()
    db = Stream(opt)
    db.create()
    wall = time.perf_counter() - t0
    out = dict(wall_s=wall, device=hasattr(db, "ingest_stats"), nnz=int(db.get_header()["num_nnz"]),
               items=int(db.get_header()["num_items"]))
    if hasattr(db, "ingest_stats"):
        out.update(db.ingest_stats)
    print(json.dumps(out))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()
        return q[0] if q else "unknown"
    except Exception:
        return "unknown"


def same_db(a, b):
    from buffalo_b200.data import store
    fa, fb = store.File(a, "r"), store.File(b, "r")
    try:
        keys = ("num_users", "num_items", "num_nnz", "completed")
        if [fa.attrs[k] for k in keys] != [fb.attrs[k] for k in keys]:
            return False
        for g in ("rowwise", "colwise", "vali", "idmap"):
            if (g in fa) != (g in fb):
                return False
            if g not in fa:
                continue
            if sorted(fa[g].keys()) != sorted(fb[g].keys()):
                return False
            for k in fa[g].keys():
                x, y = np.asarray(fa[g][k][:]), np.asarray(fb[g][k][:])
                if x.dtype != y.dtype or x.shape != y.shape or x.tobytes() != y.tobytes():
                    return False
        return True
    finally:
        fa.close()
        fb.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True)
    ap.add_argument("--tokens", type=float, default=1e8)
    ap.add_argument("--users", type=int, default=10_000_000)
    ap.add_argument("--vocab", type=int, default=1_000_000)
    ap.add_argument("--host-max", type=float, default=2e7, help="largest token count the host loop is run at")
    ap.add_argument("--child", nargs=5, help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.child:
        src, iid, db, device, matrix = a.child
        return child(src, iid if iid != "-" else None, db, device == "1", matrix == "1")
    os.makedirs(a.out, exist_ok=True)
    T = int(a.tokens)
    src, iid = os.path.join(a.out, "s%d.txt" % T), os.path.join(a.out, "s%d.iid" % T)
    if not os.path.exists(src):
        generate(src, iid, T, a.users, a.vocab)
    size = os.path.getsize(src)
    gpu = card()
    for matrix in (False, True):
        for use_iid in (False, True):
            dbs = {}
            for device in ((True, False) if T <= a.host_max else (True,)):
                db = os.path.join(a.out, "db_%d_%d_%d_%d.h5py" % (T, matrix, use_iid, device))
                before = resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss
                r = subprocess.run([sys.executable, __file__, "--out", a.out, "--child", src, iid if use_iid else "-", db,
                                    str(int(device)), str(int(matrix))], capture_output=True, text=True)
                if r.returncode:
                    print(r.stderr[-4000:], file=sys.stderr)
                    raise SystemExit(r.returncode)
                res = json.loads(r.stdout.strip().splitlines()[-1])
                rss = resource.getrusage(resource.RUSAGE_CHILDREN).ru_maxrss
                res.update(path="device" if device else "host", internal="matrix" if matrix else "stream", iid=use_iid,
                           tokens=T, text_bytes=size, tokens_per_s=T / res["wall_s"], text_GBps=size / res["wall_s"] / 1e9,
                           peak_rss_GB_max_so_far=max(rss, before) / 1e6, gpu=gpu)
                dbs[device] = db
                print(json.dumps(res), flush=True)
            if len(dbs) == 2:
                print(json.dumps(dict(tokens=T, internal="matrix" if matrix else "stream", iid=use_iid,
                                      bitwise_equal=same_db(dbs[True], dbs[False]))), flush=True)
            for db in dbs.values():
                os.remove(db)


if __name__ == "__main__":
    main()

"""Stream ingest (buffalo/data/stream.py): one line per user of whitespace-separated item tokens, oldest ->
newest.  API-compatible container; the three MF trainers only consume data_type == "matrix"
(buffalo/algo/als.py:57), so Stream with internal_data_type="matrix" is the form that feeds them.  SPPMI
(CFR only) is outside the hot-path scope.  Text files of DEVICE_INGEST_MIN_BYTES and more are parsed, interned and
split on the GPU (csrc/stream_ingest.cu) into the same database; files the device path declines go to the host loop."""
import codecs
import locale
import os
import time
from collections import Counter

import numpy as np

from buffalo_b200.data.base import Data, DataOption
from buffalo_b200.data.text_ingest import _Fallback, feed_blocks, find_cut, read_ranges
from buffalo_b200.misc import aux, log


class StreamOptions(DataOption):
    def get_default_option(self):
        return aux.Option({
            "type": "stream",
            "input": {"main": "", "uid": "", "iid": ""},
            "data": {"validation": {"name": "newest", "p": 0.01, "n": 1, "max_samples": 500},
                     "sppmi": {}, "batch_mb": 1024, "use_cache": False, "tmp_dir": "/tmp/",
                     "path": "./stream.h5py", "internal_data_type": "stream", "disk_based": False}})   # stream.py:38-65

    def is_valid_option(self, opt):
        assert super().is_valid_option(opt)
        if not opt["type"] == "stream":
            raise RuntimeError("Invalid data type: %s" % opt["type"])
        return True


def _lines(path):
    with open(path) as fin:
        return [ln.strip() for ln in fin]


# Python's whitespace, the separators of str.split() (a CPU test pins this to str.isspace).  The device parser splits
# on the ASCII ones and declines files that contain any of the others.
WHITESPACE = (0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x1C, 0x1D, 0x1E, 0x1F, 0x20, 0x85, 0xA0, 0x1680) + \
    tuple(range(0x2000, 0x200B)) + (0x2028, 0x2029, 0x202F, 0x205F, 0x3000)

# Text input goes to the device parser (csrc/stream_ingest.cu) when a GPU is present and the file is at least this large.
DEVICE_INGEST_MIN_BYTES = 32 << 20
DEVICE_INGEST_BLOCK_BYTES = 64 << 20     # each of the two pinned staging buffers; a longer line is declined
_DEVICE_BYTES_PER_TOKEN = 48             # peak of the split and CSR build: pairs, kept copies and radix-sort scratch
_HASH_BITS = 64                          # token hash width (tests truncate it to force collisions)
_DECLINE = ((1, "a bare '\\r' line end"), (2, "bytes that are not UTF-8"), (4, "a multi-byte Unicode space"),
            (8, "a token missing from the iid list"), (16, "two distinct tokens with the same 64-bit hash"),
            (32, "too little device memory"), (64, "more than 2^31 - 2 lines or items"))


def _find_cut(buf, total, block):
    """Stream's cut: the end of the last line anywhere in buf[:total]; a line longer than the block declines the file."""
    return find_cut(buf, total, block)


def _device_ingest(path, uids, names, vopt, as_matrix, block_bytes=None):
    """Parse, intern, split and build the CSR groups on the device.
    -> (num_users, item names, csr, vali or None, stats); raises _Fallback.
    stats: device_ms (CUDA-event time per stage), host_ms (file reads, name decoding, validation draw) and
    peak_device_bytes."""
    from buffalo_b200 import backend
    host_ms = dict(read=0.0, names=0.0, sample=0.0)
    block = int(block_bytes or DEVICE_INGEST_BLOCK_BYTES)
    need = 3 * block + (64 << 20)
    free = backend.device_free_bytes()
    if need > free:
        raise _Fallback("estimated %.1f GB of device memory for the parse, %.1f GB free" % (need / 1e9, free / 1e9))
    with backend.StreamIngest(block, WHITESPACE, _HASH_BITS) as ing, open(path, "rb", buffering=0) as fin:
        if names is not None:
            ing.load_iid([s.encode("utf-8") for s in names])
        last_byte = feed_blocks(ing, fin, block, block, host_ms)
        r = ing.finish()
        if r["decline"]:
            why = [s for b, s in _DECLINE if r["decline"] & b]
            raise _Fallback(", ".join(why) + (" (line %d)" % r["decline_line"] if r["decline_line"] >= 0 else ""))
        lines = r["lines"] + (last_byte != b"\n")
        if uids is not None and len(uids) < lines:
            raise _Fallback("%d uid lines for %d lines of sessions" % (len(uids), lines))
        num_users = len(uids) if uids is not None else lines
        total, num_items = r["tokens"], r["items"]
        if num_users == 0 or num_items == 0:
            raise _Fallback("no users or no items")
        need = _DEVICE_BYTES_PER_TOKEN * total + 16 * (num_users + num_items)
        free = backend.device_free_bytes()
        if need > free:
            raise _Fallback("estimated %.1f GB of device memory for %d tokens, %.1f GB free" % (need / 1e9, total, free / 1e9))
        if names is None:
            t0 = time.perf_counter()
            off, ln = ing.names(num_items)
            names = [b.decode("utf-8") for b in read_ranges(path, off, ln)]
            host_ms["names"] = 1e3 * (time.perf_counter() - t0)
        method = vopt.name if vopt else None
        vali_n = vopt.get("n", 0) if method == "newest" else 0
        idx = np.zeros(0, np.int64)
        if method == "sample":
            t0 = time.perf_counter()
            sz = min(vopt.max_samples, int(total * vopt.p))   # the host path's draw, on the same global RNG stream
            idx = np.random.choice(max(total - 1, 1), sz, replace=False) if sz else idx
            host_ms["sample"] = 1e3 * (time.perf_counter() - t0)
        code = {"newest": 1, "sample": 2}.get(method, 0)
        ntrain, (vr, vc, vv) = ing.split(num_users, code, vali_n, idx, as_matrix)
        vali = dict(method=method, n=vali_n, row=vr, col=vc, val=vv) if vopt else None
        csr = {"rowwise": ing.build(0, num_users, ntrain)}
        if as_matrix:
            csr["colwise"] = ing.build(1, num_items, ntrain)
        device_ms, peak = ing.stats()
    return num_users, names, csr, vali, dict(device_ms=device_ms, host_ms=host_ms, peak_device_bytes=peak)


def _locale_is_utf8():
    try:
        return codecs.lookup(locale.getpreferredencoding(False)).name == "utf-8"
    except LookupError:
        return False


class Stream(Data):
    def __init__(self, opt, *args, **kwargs):
        super().__init__(opt, *args, **kwargs)
        self.name = "Stream"
        self.logger = log.get_logger("Stream")
        self.data_type = "stream"

    def _use_device_ingest(self, main):
        from buffalo_b200 import backend
        return (isinstance(main, str) and os.path.isfile(main) and os.path.getsize(main) >= DEVICE_INGEST_MIN_BYTES
                and _locale_is_utf8() and backend.device_available())

    def _create_on_device(self, path):
        """Builds the database through the device parser; False when it declines the file (the host path then runs)."""
        try:
            uids = _lines(self.opt.input.uid) if self.opt.input.uid else None
            names = _lines(self.opt.input.iid) if self.opt.input.iid else None
        except (OSError, UnicodeError) as e:
            self.logger.info("Device text parse skipped (%s); parsing on the host." % e)
            return False
        as_matrix = self.opt.data.internal_data_type == "matrix"
        try:
            num_users, names, csr, vali, self.ingest_stats = _device_ingest(self.opt.input.main, uids, names,
                                                                            self.opt.data.validation, as_matrix)
        except _Fallback as e:
            self.logger.info("Device text parse declined the file (%s); parsing on the host." % e)
            return False
        groups = ("rowwise", "colwise") if as_matrix else ("rowwise",)
        self._write_database(path, num_users, len(names), None, None, None, uids, names, vali, groups=groups, csr=csr)
        self.logger.info("DB built on %s" % path)
        return True

    def create(self):
        path = self.opt.data.path
        if os.path.isfile(path) and self.opt.data.use_cache:
            self.logger.info("Use cached DB on %s" % path)
            self.open(path)
            return
        if self.opt.data.sppmi:
            raise NotImplementedError("SPPMI (CoFactor only) is outside the H100 hot-path scope")
        if self._use_device_ingest(self.opt.input.main) and self._create_on_device(path):
            return
        sessions = [ln.split() for ln in _lines(self.opt.input.main)]
        uids = _lines(self.opt.input.uid) if self.opt.input.uid else None
        num_users = len(uids) if uids is not None else len(sessions)
        if self.opt.input.iid:
            names = _lines(self.opt.input.iid)
        else:  # ids in order of first appearance (the reference enumerates a set, stream.py:120-126)
            names = list(dict.fromkeys(tok for s in sessions for tok in s))
        item_index = {name: i for i, name in enumerate(names)}
        vopt = self.opt.data.validation
        method = vopt.name if vopt else None
        vali_n = vopt.get("n", 0) if method == "newest" else 0
        as_matrix = self.opt.data.internal_data_type == "matrix"
        total = sum(len(s) for s in sessions)
        sample_idx = set()
        if method == "sample":
            sz = min(vopt.max_samples, int(total * vopt.p))
            sample_idx = set(np.random.choice(max(total - 1, 1), sz, replace=False).tolist()) if sz else set()
        tr, va = [], []
        pos = 0
        for u, toks in enumerate(sessions):
            if not toks:
                continue
            cut = len(toks) - min(vali_n, len(toks) - 1)       # stream.py:224-231
            held = [item_index[t] for t in toks[cut:]]
            kept = []
            for k, t in enumerate(toks[:cut]):
                (held if (pos + k) in sample_idx else kept).append(item_index[t])
            pos += cut
            if as_matrix:                                        # collapse duplicates with counts (stream.py:252-256)
                tr += [(u, c, float(n)) for c, n in Counter(kept).items()]
            else:                                                # keep order, value 1 (stream.py:247-251)
                tr += [(u, c, 1.0) for c in kept]
            va += [(u, c, float(n)) for c, n in Counter(held).items()]
        rows = np.array([t[0] for t in tr], dtype=np.int64)
        cols = np.array([t[1] for t in tr], dtype=np.int64)
        vals = np.array([t[2] for t in tr], dtype=np.float32)
        vali = None
        if vopt:
            vali = dict(method=method, n=vali_n, row=[t[0] for t in va], col=[t[1] for t in va], val=[t[2] for t in va])
        groups = ("rowwise", "colwise") if as_matrix else ("rowwise",)
        self._write_database(path, num_users, len(names), rows, cols, vals, uids, names, vali, groups=groups,
                             keep_order=not as_matrix)
        self.logger.info("DB built on %s" % path)

"""MatrixMarket ingest (buffalo/data/mm.py): text file, scipy sparse or dense 2-D array -> database."""
import os

import numpy as np
import scipy.sparse

from buffalo_b200.data.base import Data, DataOption, DataReader
from buffalo_b200.data import prepro
from buffalo_b200.data.text_ingest import _Fallback, feed_blocks, read_ranges
from buffalo_b200.misc import aux, log


class MatrixMarketOptions(DataOption):
    def get_default_option(self):
        return aux.Option({
            "type": "matrix_market",
            "input": {"main": "", "uid": "", "iid": ""},
            "data": {"internal_data_type": "matrix",
                     "validation": {"name": "sample", "p": 0.01, "max_samples": 500},
                     "batch_mb": 1024, "use_cache": False, "tmp_dir": "/tmp/", "path": "./mm.h5py",
                     "disk_based": False}})                       # mm.py:14-37

    def is_valid_option(self, opt):
        assert super().is_valid_option(opt)
        if not opt["type"] == "matrix_market":
            raise RuntimeError("Invalid data type: %s" % opt["type"])
        if opt["data"]["internal_data_type"] != "matrix":
            raise RuntimeError("MatrixMarket only support internal data type(matrix)")
        for field in ["uid", "iid"]:
            v = opt["input"][field]
            ok = v is None or isinstance(v, (str, list)) or (isinstance(v, np.ndarray) and v.ndim == 1)
            assert ok, f"Not supported data type for MatrixMarketOption.input.{field}: {type(v)}"
        main = opt["input"]["main"]
        ok = isinstance(main, str) or (isinstance(main, np.ndarray) and main.ndim == 2) or scipy.sparse.issparse(main)
        assert ok, f"Not supported data type for MatrixMarketOption.input.main field: {type(main)}"
        return True


class MatrixMarketDataReader(DataReader):
    pass


def _read_ids(spec):
    if spec is None or (isinstance(spec, str) and spec == ""):
        return None
    if isinstance(spec, str):
        with open(spec) as fin:
            return [line.rstrip("\n").strip() for line in fin if line.strip() != ""]
    return [str(x) for x in (spec.tolist() if isinstance(spec, np.ndarray) else spec)]


def _read_mm_header(path):
    """-> (num_rows, num_cols, nnz, skip): the "U I nnz" line and the number of lines up to and including it."""
    skip = 0
    with open(path) as fin:
        for line in fin:
            skip += 1
            if not line.strip().startswith("%"):
                header = line
                break
    U, I, nnz = map(int, header.split())
    return U, I, nnz, skip


def _read_mm_text(path):
    """-> (num_rows, num_cols, rows0, cols0, vals) from a coordinate MatrixMarket file (1-based text)."""
    import pandas as pd
    U, I, nnz, skip = _read_mm_header(path)
    if nnz == 0:
        return U, I, np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0, np.float32)
    df = pd.read_csv(path, sep=r"\s+", header=None, skiprows=skip, comment="%", dtype=np.float64, engine="c")
    rows = df[0].to_numpy().astype(np.int64) - 1
    cols = df[1].to_numpy().astype(np.int64) - 1
    vals = df[2].to_numpy().astype(np.float32) if df.shape[1] > 2 else np.ones(len(rows), np.float32)
    return U, I, rows, cols, vals


def _parse_value_tokens(tokens):
    """float32 values of value tokens (bytes) through the same reader and conversion as _read_mm_text's value column,
    so a token the device parser leaves to the host gets the host path's bits."""
    import io
    import pandas as pd
    if not tokens:
        return np.zeros(0, np.float32)
    df = pd.read_csv(io.BytesIO(b"\n".join(tokens) + b"\n"), sep=r"\s+", header=None, comment="%", dtype=np.float64,
                     engine="c")
    if df.shape != (len(tokens), 1):
        raise ValueError("value tokens did not parse one per line")
    return df[0].to_numpy().astype(np.float32)


# Text input goes to the device parser (csrc/mm_ingest.cu) when a GPU is present and the file is at least this large.
DEVICE_INGEST_MIN_BYTES = 32 << 20
DEVICE_INGEST_BLOCK_BYTES = 64 << 20     # each of the two pinned staging buffers
DEVICE_INGEST_MAX_SLOW = 1 << 24         # value tokens the device may leave to the host parser
MAX_LINE = 1024                          # BFL_MM_MAX_LINE: longer lines are grammar rejections
_DEVICE_BYTES_PER_NNZ = 40               # peak of the device build: triples, CSR output and radix-sort scratch


def _data_offset(path, skip):
    """Byte offset of the first line after the header, or None when the header lines use a bare '\r' line end
    (text mode counts those as line ends, a byte split on '\n' would not)."""
    off = 0
    with open(path, "rb") as fin:
        for _ in range(skip):
            line = fin.readline()
            if b"\r" in line.replace(b"\r\n", b""):
                return None
            off += len(line)
    return off


def _device_ingest(path, U, I, nnz_hint, skip, vopt, logger, block_bytes=None):
    """Parse, split and build both CSR orientations on the device.
    -> (nnz, {group: (indptr, key, val)}, vali or None, stats); raises _Fallback or ValueError (index out of range).
    stats: device_ms (CUDA-event time per stage), host_ms (file reads, slow-token parse, validation draw) and
    peak_device_bytes."""
    import time
    from buffalo_b200 import backend
    host_ms = dict(read=0.0, slow_parse=0.0, sample=0.0)
    block = int(block_bytes or DEVICE_INGEST_BLOCK_BYTES)
    data_off = _data_offset(path, skip)
    if data_off is None:
        raise _Fallback("a header line ends with a bare '\\r'")
    need = _DEVICE_BYTES_PER_NNZ * nnz_hint + 8 * (U + I) + 3 * block + (64 << 20)
    free = backend.device_free_bytes()
    if need > free:
        raise _Fallback("estimated %.1f GB of device memory for %d entries, %.1f GB free" % (need / 1e9, nnz_hint, free / 1e9))
    slow_cap = min(nnz_hint, DEVICE_INGEST_MAX_SLOW)
    with backend.MMIngest(U, I, nnz_hint, block, skip, slow_cap) as ing, open(path, "rb", buffering=0) as fin:
        fin.seek(data_off)
        feed_blocks(ing, fin, block, MAX_LINE, host_ms)
        r = ing.finish()
        if r["reject_line"] >= 0:
            raise _Fallback("line %d is outside the device grammar" % r["reject_line"])
        if r["tokmask"] not in (1 << 2, 1 << 3):
            raise _Fallback("data lines mix 2 and 3 tokens" if r["tokmask"] else "no data lines")
        if r["range_line"] >= 0:
            raise ValueError("%s: line %d has an index outside [1, %d] x [1, %d]" % (path, r["range_line"], U, I))
        nnz = r["nnz"]
        if nnz > nnz_hint:
            raise _Fallback("%d data lines, more than the header's %d" % (nnz, nnz_hint))
        if r["n_slow"] > slow_cap:
            raise _Fallback("%d values need the host parser (at most %d)" % (r["n_slow"], slow_cap))
        if r["n_slow"]:
            t0 = time.perf_counter()
            ordinal, offset, length = ing.slow_tokens(r["n_slow"])
            try:
                vals = _parse_value_tokens(read_ranges(path, offset + data_off, length))
            except ValueError as e:
                raise _Fallback("a value the host parser rejects (%s)" % e)
            host_ms["slow_parse"] = 1e3 * (time.perf_counter() - t0)
            ing.patch_values(ordinal, vals)
        vali, idx = None, np.zeros(0, np.int64)
        if vopt:
            t0 = time.perf_counter()
            sz = min(vopt.max_samples, int(nnz * vopt.p))
            idx = np.sort(np.random.choice(nnz - 1, sz, replace=False)) if sz > 0 else np.zeros(0, np.int64)
            host_ms["sample"] = 1e3 * (time.perf_counter() - t0)
        vr, vc, vv = ing.split(idx)
        if vopt:
            vali = dict(method="sample", n=0, indexes=idx, row=vr, col=vc, val=vv)
        ntrain = nnz - len(idx)
        csr = {"rowwise": ing.build(0, U, ntrain), "colwise": ing.build(1, I, ntrain)}
        device_ms, peak = ing.stats()
    return ntrain, csr, vali, dict(device_ms=device_ms, host_ms=host_ms, peak_device_bytes=peak)


class MatrixMarket(Data):
    def __init__(self, opt, *args, **kwargs):
        super().__init__(opt, *args, **kwargs)
        self.name = "MatrixMarket"
        self.logger = log.get_logger("MatrixMarket")
        if isinstance(self.value_prepro, prepro.SPPMI):
            raise RuntimeError(f"{self.opt.data.value_prepro.name} does not support MatrixMarket")
        self.data_type = "matrix"
        self.reader = MatrixMarketDataReader(self.opt)

    def _load_triples(self):
        main = self.opt.input.main
        if isinstance(main, str):
            return _read_mm_text(main)
        if isinstance(main, np.ndarray) and main.ndim == 2:
            main = scipy.sparse.csr_matrix(main)
        if scipy.sparse.issparse(main):
            coo = main.tocoo()
            return coo.shape[0], coo.shape[1], coo.row.astype(np.int64), coo.col.astype(np.int64), coo.data.astype(np.float32)
        raise RuntimeError(f"Unexpected data type for MatrixMarketOption.input.main field: {type(main)}")

    def _use_device_ingest(self, main):
        from buffalo_b200 import backend
        return isinstance(main, str) and os.path.getsize(main) >= DEVICE_INGEST_MIN_BYTES and backend.device_available()

    def create(self):
        path = self.opt.data.path
        if os.path.isfile(path) and self.opt.data.use_cache:
            self.logger.info("Use cached DB on %s" % path)
            self.open(path)
            return
        self.logger.info("Create the database from matrix market file.")
        vopt = self.opt.data.validation
        if vopt and vopt.name != "sample":
            raise RuntimeError("MatrixMarket supports validation.name == 'sample' only")
        main = self.opt.input.main
        if self._use_device_ingest(main):
            U, I, nnz_hint, skip = _read_mm_header(main)
            try:
                if nnz_hint <= 0:
                    raise _Fallback("the header has nnz = %d" % nnz_hint)
                nnz, csr, vali, self.ingest_stats = _device_ingest(main, U, I, nnz_hint, skip, vopt, self.logger)
            except _Fallback as e:
                self.logger.info("Device text parse declined the file (%s); parsing on the host." % e)
            else:
                self._write_database(path, U, I, None, None, None, _read_ids(self.opt.input.uid),
                                     _read_ids(self.opt.input.iid), vali, csr=csr)
                self.logger.info("DB built on %s" % path)
                return
        U, I, rows, cols, vals = self._load_triples()
        nnz = len(rows)
        vali = None
        if vopt:
            # base.py:225-231: sample line indexes, never the last line
            sz = min(vopt.max_samples, int(nnz * vopt.p))
            idx = np.sort(np.random.choice(nnz - 1, sz, replace=False)) if sz > 0 else np.zeros(0, np.int64)
            mask = np.ones(nnz, bool)
            mask[idx] = False
            vali = dict(method="sample", n=0, indexes=idx, row=rows[idx], col=cols[idx], val=vals[idx])
            rows, cols, vals = rows[mask], cols[mask], vals[mask]
        self._write_database(path, U, I, rows, cols, vals, _read_ids(self.opt.input.uid), _read_ids(self.opt.input.iid), vali)
        self.logger.info("DB built on %s" % path)

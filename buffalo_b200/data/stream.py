"""Stream ingest (buffalo/data/stream.py): one line per user of whitespace-separated item tokens, oldest ->
newest.  API-compatible container; the three MF trainers only consume data_type == "matrix"
(buffalo/algo/als.py:57), so Stream with internal_data_type="matrix" is the form that feeds them.  SPPMI
(CFR only) is outside the hot-path scope."""
import os
from collections import Counter

import numpy as np

from buffalo_b200.data.base import Data, DataOption
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


class Stream(Data):
    def __init__(self, opt, *args, **kwargs):
        super().__init__(opt, *args, **kwargs)
        self.name = "Stream"
        self.logger = log.get_logger("Stream")
        self.data_type = "stream"

    def create(self):
        path = self.opt.data.path
        if os.path.isfile(path) and self.opt.data.use_cache:
            self.logger.info("Use cached DB on %s" % path)
            self.open(path)
            return
        if self.opt.data.sppmi:
            raise NotImplementedError("SPPMI (CoFactor only) is outside the H100 hot-path scope")
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

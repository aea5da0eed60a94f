"""Data base classes: the compiled "database" holding both CSR orientations, id maps and the held-out split
(buffalo/data/base.py).  Layout contract kept bit-for-bit (base.py:187-192, fileio.hpp:330-378): per
orientation `indptr` int64[rows] = exclusive END offsets, `key` int32[nnz] zero-based, `val` float32[nnz],
rows sorted by (row, col) resp. (col, row), duplicates kept.  The reference's text -> temp files -> parallel
sort -> HDF5 pipeline is replaced by an in-memory build: NumPy on the host, or the hand-written device radix sort of
csrc/ingest.cu when a GPU is present and the matrix is large (SURVEY 8f.1)."""
import os

import numpy as np

from buffalo_b200.data import prepro, store
from buffalo_b200.misc import aux, log


DEVICE_SORT_MIN_NNZ = 1 << 20   # below this the host sort is faster than the PCIe round trip


def _csr_from_triples_torch(major, minor, vals, num_major, stable_sort, device):
    """The same ordering on a torch device: one stable sort of the combined (major, minor) key -- on a GPU this is
    the radix sort the 1B-nnz ingest needs (SURVEY 8f.1; the reference: text -> temp files -> parallel sort,
    fileio.hpp:263-419).  Works on CPU tensors too (used by the tests to pin it against the NumPy path)."""
    import torch
    mj = torch.as_tensor(np.ascontiguousarray(major), device=device).to(torch.int64)
    mn = torch.as_tensor(np.ascontiguousarray(minor), device=device).to(torch.int64)
    if stable_sort:
        span = int(mn.max().item()) + 1 if mn.numel() else 1
        order = torch.sort(mj * span + mn, stable=True).indices
    else:
        order = torch.sort(mj, stable=True).indices
    indptr = torch.cumsum(torch.bincount(mj, minlength=num_major), 0)
    key = mn[order].to(torch.int32)
    val = torch.as_tensor(np.ascontiguousarray(vals), device=device)[order].to(torch.float32)
    return indptr.cpu().numpy().astype(np.int64), key.cpu().numpy(), val.cpu().numpy()


def csr_from_triples(major, minor, vals, num_major, stable_sort=True, device=None):
    """(indptr_end, key, val) sorted by (major, minor) with a stable sort (fileio.hpp:330-341).
    device: None = the GPU when one is present and the matrix is large, else the host; or an explicit torch device."""
    if device is None and len(major) >= DEVICE_SORT_MIN_NNZ:
        try:
            import torch
            if torch.cuda.is_available():
                device = "cuda"
        except ImportError:
            pass
    if device is not None and str(device).startswith("cuda"):
        # hand-written device radix sort (csrc/ingest.cu); indices must fit the int32 layout the CSR uses anyway
        from buffalo_b200 import backend
        num_minor = int(np.max(minor)) + 1 if len(minor) else 1
        return backend.csr_from_triples_host(major, minor, vals, num_major, num_minor, sort_minor=stable_sort)
    if device is not None:
        return _csr_from_triples_torch(major, minor, vals, num_major, stable_sort, device)
    if stable_sort:
        order = np.lexsort((minor, major))
    else:  # keep the input order inside a row (Stream, internal_data_type="stream")
        order = np.argsort(major, kind="stable")
    indptr = np.cumsum(np.bincount(major, minlength=num_major)).astype(np.int64)
    return indptr, minor[order].astype(np.int32), vals[order].astype(np.float32)


class Data(object):
    def __init__(self, opt, *args, **kwargs):
        self.opt = aux.Option(opt)
        self.tmp_root = self.opt.data.tmp_dir
        os.makedirs(self.tmp_root, exist_ok=True)
        self.handle, self.header = None, None
        self.prepro = prepro.PreProcess(self.opt.data)
        if self.opt.data.value_prepro:
            self.prepro = getattr(prepro, self.opt.data.value_prepro.name)(self.opt.data.value_prepro)
        self.value_prepro = self.prepro
        self.data_type = None
        self.temp_file_list = []
        self.logger = log.get_logger("Data")

    # ---- read side -----------------------------------------------------------------------------
    def open(self, data_path):
        self.handle = store.File(data_path, "r")
        self.path = data_path
        self.verify()

    def verify(self):
        assert self.handle, "Database is not opened"
        if self.get_header()["completed"] != 1:
            raise RuntimeError("Database is corrupted or partially built. Please try again, after remove it.")

    def get_header(self):
        assert self.handle, "Database is not opened"
        if not self.header:
            self.header = {k: self.handle.attrs[k] for k in ("num_nnz", "num_users", "num_items", "completed")}
        return self.header

    def show_info(self):
        h = self.get_header()
        vali = self.get_group("vali").attrs["num_samples"] if self.has_group("vali") else 0
        return "{} Header({}, {}, {}) Validation({} samples)".format(self.name, h["num_users"], h["num_items"],
                                                                   h["num_nnz"], vali)

    def get_group(self, group_name="rowwise"):
        assert group_name in ["rowwise", "colwise", "vali", "idmap", "sppmi"], "Unexpected group_name: {}".format(group_name)
        assert self.handle, "DB is not opened"
        return self.handle[group_name]

    def has_group(self, name):
        return name in self.handle

    def get_scale_info(self, with_sppmi=False, chunk_size=100000):
        ret = {k: self.handle.attrs.get(k, 0) for k in ["num_users", "num_items", "num_nnz", "sppmi_nnz"]}
        ret["vsum"] = float(np.sum(self.handle["rowwise"]["val"][:ret["num_nnz"]], dtype=np.float64))
        return ret

    def iterate(self, axis="rowwise", use_repr_name=False):
        idmap = self.get_group("idmap")
        name_of = [str, str]
        if use_repr_name:
            for i, field in enumerate(("rows", "cols")):
                if idmap[field].shape[0]:
                    name_of[i] = (lambda f: (lambda x: idmap[f][x].decode("utf-8", "ignore")))(field)
            if axis == "colwise":
                name_of.reverse()
        stream = self.opt.data.internal_data_type == "stream"
        assert axis in (["rowwise"] if stream else ["rowwise", "colwise"]), "Unexpected data axis: {}".format(axis)
        g = self.handle[axis]
        keys, vals = g["key"], (None if stream else g["val"])

        def gen():
            beg = 0
            for u, end in enumerate(g["indptr"]):
                for i in range(beg, end):
                    a, b = (name_of[0](u), name_of[1](keys[i])) if use_repr_name else (u, keys[i])
                    yield (a, b) if stream else (a, b, vals[i])
                beg = end
        return gen()

    def get(self, index, axis="rowwise"):
        g = self.handle[axis]
        beg = 0 if index == 0 else g["indptr"][index - 1]
        end = g["indptr"][index]
        if self.opt.data.internal_data_type == "stream":
            return (g["key"][beg:end],)
        return (g["key"][beg:end], g["val"][beg:end])

    def close(self):
        if self.handle:
            self.handle.close()
            self.handle, self.header = None, None

    def temp_file_clear(self):
        for p in self.temp_file_list:
            if isinstance(p, str) and os.path.isfile(p):
                os.remove(p)
        self.temp_file_list = []

    # ---- build side ----------------------------------------------------------------------------
    def _write_database(self, path, num_users, num_items, rows, cols, vals, uids, iids, vali,
                        groups=("rowwise", "colwise"), keep_order=False, csr=None):
        """rows/cols: zero-based int arrays of the TRAINING entries; vali: None or dict(method, n, row, col, val).
        csr: None, or {group: (indptr, key, val)} already built from the training entries with raw values (the device
        MatrixMarket parser); rows/cols/vals are then unused.  value_prepro is element-wise or uses the global min/max,
        so applying it to each orientation's sorted values gives the bits of applying it before the sort."""
        if os.path.exists(path):
            self.logger.info(f"File {path} exists. To build new database, existing file {path} will be deleted.")
            os.remove(path)
        f = store.File(path, "w")
        self.path = path
        if csr is None:
            vals = np.asarray(self.value_prepro(np.asarray(vals, dtype=np.float32).copy()), dtype=np.float32)
            num_nnz = len(rows)
        else:
            num_nnz = len(csr["rowwise"][1])
        self.prepro.pre(f)
        for g, major, minor, nmajor in (("rowwise", rows, cols, num_users), ("colwise", cols, rows, num_items)):
            grp = f.create_group(g)
            if g in groups and csr is not None:
                indptr, key, val = csr[g]
                val = np.asarray(self.value_prepro(np.asarray(val, dtype=np.float32)), dtype=np.float32)
            elif g in groups:
                indptr, key, val = csr_from_triples(major, minor, vals, nmajor, stable_sort=not keep_order)
            else:
                indptr, key, val = np.zeros(nmajor, np.int64), np.zeros(0, np.int32), np.zeros(0, np.float32)
            grp.create_dataset("indptr", data=indptr)
            grp.create_dataset("key", data=key)
            grp.create_dataset("val", data=val)
            if g in groups:
                self.prepro.post(grp)
        if vali is not None:
            v = f.create_group("vali")
            v.attrs["method"], v.attrs["n"] = vali["method"], vali.get("n", 0)
            v.attrs["num_samples"] = len(vali["row"])
            if "indexes" in vali:
                v.create_dataset("indexes", data=np.asarray(vali["indexes"], dtype=np.int64))
            v.create_dataset("row", data=np.asarray(vali["row"], dtype=np.int32))
            v.create_dataset("col", data=np.asarray(vali["col"], dtype=np.int32))
            v.create_dataset("val", data=np.asarray(self.value_prepro(np.asarray(vali["val"], dtype=np.float32)),
                                                    dtype=np.float32))
        idmap = f.create_group("idmap")
        for name, ids, n in (("rows", uids, num_users), ("cols", iids, num_items)):
            if ids is None:
                ids = [str(i) for i in range(1, n + 1)]
            if len(ids) != n:
                raise TypeError("id list for %s has %d entries, %d expected" % (name, len(ids), n))
            enc = [str(s).encode("utf-8") for s in ids]
            idmap.create_dataset(name, data=np.array(enc, dtype="S%d" % (max([len(e) for e in enc] + [1]) + 1)))
        f.attrs.update(num_users=int(num_users), num_items=int(num_items), num_nnz=int(num_nnz), completed=1)
        f.close()
        self.handle = store.File(path, "r")

    def _prepare_validation_data(self):
        """Ground truth / seen sets per validation row (buffalo/data/base.py:255-298)."""
        if hasattr(self, "vali_data"):
            return True
        v = self.handle["vali"]
        row, col, val = v["row"][:], v["col"][:], v["val"][:]
        vali_rows = np.unique(row)
        gt = {int(u): set() for u in vali_rows}
        for r, c in zip(row, col):
            gt[int(r)].add(int(c))
        seen, max_seen = {}, 0
        for u in vali_rows:
            keys, *_ = self.get(int(u))
            seen[int(u)] = set(int(k) for k in keys)
            max_seen = max(max_seen, len(keys))
        self.vali_data = {"row": row, "col": col, "val": val, "vali_rows": vali_rows, "vali_gt": gt,
                          "validation_seen": seen, "validation_max_seen_size": max_seen}
        return True


class DataOption(object):
    def is_valid_option(self, opt):
        assert hasattr(opt["data"], "disk_based") or "disk_based" in opt["data"], "disk_based not defined on data"
        assert isinstance(opt["data"]["disk_based"], bool), "invalid type for data.disk_based"
        v = opt["data"].get("validation")
        if v:
            assert v["name"] in ["sample", "newest"], "Unknown validation.name."
            assert isinstance(v.get("max_samples"), int), "invalid type for data.validation.max_samples"
            if v["name"] == "sample":
                assert isinstance(v.get("p"), float), "invalid type for data.validation.p"
            else:
                assert isinstance(v.get("n"), int), "invalid type for data.validation.n"
        return True


class DataReader(object):
    def __init__(self, opt):
        self.opt = opt
        self.temp_file_list = []

    def get_main_path(self):
        return self.opt.input.main

    def get_uid_path(self):
        return self.opt.input.uid

    def get_iid_path(self):
        return self.opt.input.iid

    def temp_file_clear(self):
        self.temp_file_list = []

"""Host-side mixins shared by the trainers (buffalo/algo/base.py): id maps, top-k queries, similarity,
early stopping / save-best bookkeeping, the trainers' constructor body and epoch loop, and the length-prefixed pickle
container of Serializable.  Pure host glue around the factor matrices; nothing here is on the GPU hot path."""
import abc
import json
import pickle
import struct
import time

import numpy as np

from buffalo_b200 import data as _data
from buffalo_b200.data.base import Data
from buffalo_b200.misc import aux, log

EPS = 1e-8


class Algo(abc.ABC):
    def __init__(self, *args, **kwargs):
        self._idmanager = aux.Option({"userid": [], "userid_map": {}, "itemid": [], "itemid_map": {},
                                      "userid_mapped": False, "itemid_mapped": False})

    # ---- options / lifecycle ------------------------------------------------------------------
    def get_option(self, opt_path):
        """dict options are dumped to a temp JSON whose PATH goes to the native side (base.py:18-24)."""
        if isinstance(opt_path, (dict, aux.Option)):
            opt_path = self.create_temporary_option_from_dict(opt_path)
        opt = aux.Option(opt_path)
        self.is_valid_option(opt)
        return aux.Option(opt), opt_path

    def initialize(self):
        self._es_round, self._es_min = 0, 987654321
        if self.opt.random_seed:
            np.random.seed(self.opt.random_seed)        # base.py:33-34: unseeded when random_seed == 0

    @abc.abstractmethod
    def normalize(self, group="item"):
        raise NotImplementedError

    def _normalize(self, feat):
        return feat / np.sqrt((feat ** 2).sum(-1) + EPS)[..., np.newaxis]

    def periodical(self, period, current):
        return (not period) or (current + 1) % period == 0

    def save_best_only(self, loss, best_loss, i):
        if self.opt.save_best and best_loss > loss and self.periodical(self.opt.save_period, i):
            self.save(self.opt.model_path)
            return loss
        return best_loss

    def early_stopping(self, loss):
        if self.opt.early_stopping_rounds < 1:
            return False
        self._es_round = self._es_round + 1 if self._es_min < loss else 0
        self._es_min = loss                              # base.py:216-221: last loss, not the running minimum
        if self._es_round >= self.opt.early_stopping_rounds:
            self.logger.info("Reached at early_stopping rounds, stopping train.")
            return True
        return False

    # ---- training driver shared by the trainers -------------------------------------------------------
    def _init_trainer(self, name, opt_cls, make_obj, opt_path, init_error, kwargs):
        """Constructor body of a trainer: options, the backend holder make_obj(), data, logging.
        init_error(opt_path, last_error) is the message of the assertion that the holder accepted the options."""
        if opt_path is None:
            opt_path = opt_cls().get_default_option()
        self.logger = log.get_logger(name)
        self.opt, self.opt_path = self.get_option(opt_path)
        self.obj = make_obj()
        assert self.obj.init(bytes(self.opt_path, "utf-8")), init_error(opt_path, getattr(self.obj, "last_error", ""))
        self.data = None
        data = kwargs.get("data")
        data_opt = kwargs.get("data_opt", self.opt.get("data_opt"))
        if data_opt:
            self.data = _data.load(data_opt)
            assert self.data.data_type == "matrix"
            self.data.create()
        elif isinstance(data, Data):
            self.data = data
        self.logger.info("%s(%s)" % (name, json.dumps(self.opt, indent=2)))
        if self.data:
            self.logger.info(self.data.show_info())
            assert self.data.data_type in ["matrix"]

    def _resident_capable(self, need_bytes):
        """True when the device-resident path may run: not switched off by _b200_resident, and need_bytes fits in the
        free device memory with 30% to spare."""
        if self.opt.get("_b200_resident") is False:
            return False
        try:
            import torch
            free, _ = torch.cuda.mem_get_info()
        except Exception:
            return False
        return need_bytes * 1.3 < free

    def _csr_to_device(self, group, dev):
        """(indptr int64, keys int32, vals float32) torch tensors on `dev` of one CSR group of self.data; an empty
        group gets one-element key and value arrays."""
        import torch
        grp = self.data.get_group(group)
        n = int(grp["indptr"][-1]) if len(grp["indptr"]) else 0

        def t(a, dt):
            return torch.from_numpy(np.ascontiguousarray(a, dtype=dt)).to(dev)
        return (t(grp["indptr"][:], np.int64), t(grp["key"][:n] if n else np.zeros(1), np.int32),
                t(grp["val"][:n] if n else np.zeros(1), np.float32))

    def _epoch_loop(self, one_iteration, sync_back, training_callback, loss_label, best_loss):
        """opt.num_iters epochs of one_iteration() -> training loss, with periodic validation and the training
        callback, save-best and early stopping.  sync_back() brings device-resident factors to the host before they
        are validated or saved; best_loss is what save-best compares the first loss against.  Returns the last loss."""
        loss, self.validation_result = None, {}
        for i in range(self.opt.num_iters):
            t0 = time.time()
            loss = one_iteration()
            train_t = time.time() - t0
            metrics = {"train_loss": loss}
            if self.opt.validation and self.opt.evaluation_on_learning and self.periodical(self.opt.evaluation_period, i):
                t0 = time.time()
                sync_back()
                self.validation_result = self.get_validation_results()
                vals = " ".join(f"{k}:{v:0.5f}" for k, v in self.validation_result.items())
                self.logger.info(f"Validation: {vals} Elapsed {time.time() - t0:0.3f} secs")
                metrics.update({"val_%s" % k: v for k, v in self.validation_result.items()})
                if callable(training_callback):
                    training_callback(i, metrics)
            self.logger.info("Iteration %d: %s %.3f Elapsed %.3f secs" % (i + 1, loss_label, loss, train_t))
            if self.opt.save_best:
                sync_back()
            best_loss = self.save_best_only(loss, best_loss, i)
            if self.early_stopping(loss):
                break
        return loss

    # ---- id maps ------------------------------------------------------------------------------
    def _build_map(self, field, count_key, ids_attr, map_attr, flag):
        names = self.data.get_group("idmap")[field]
        n = self.data.get_header()[count_key]
        ids = [str(i) for i in range(n)] if names.shape[0] == 0 else [b.decode("utf-8", "ignore") for b in names[:]]
        self._idmanager[ids_attr] = ids
        self._idmanager[map_attr] = {v: i for i, v in enumerate(ids)}
        self._idmanager[flag] = True

    def build_itemid_map(self):
        self._build_map("cols", "num_items", "itemids", "itemid_map", "itemid_mapped")

    def build_userid_map(self):
        self._build_map("rows", "num_users", "userids", "userid_map", "userid_mapped")

    def get_index(self, keys, group="item"):
        many = isinstance(keys, list)
        keys = keys if many else [keys]
        if group == "item":
            if not self._idmanager.itemid_mapped:
                self.build_itemid_map()
            idx = [self._idmanager.itemid_map.get(k) for k in keys]
        elif group == "user":
            if not self._idmanager.userid_mapped:
                self.build_userid_map()
            idx = [self._idmanager.userid_map.get(k) for k in keys]
        else:
            idx = []
        return np.array(idx) if many else idx[0]

    # ---- new items (DESIGN.md 4.16) ------------------------------------------------------------
    def add_items(self, ids, rows, bias=None):
        """Serves new items: appends `rows` (n, d) to Q and their names `ids` to the item-id map (built from the data
        first if it has not been), and for models with item biases (BPRMF, WARP) `bias` (n,) to Qb, 0 when None.  The
        rows are what fold_in_items returns; under normalize("item") they are normalized too, so cosines stay
        consistent.  Every query path then sees the new items; an item index built before the call reports itself
        stale.  Raises ValueError, changing nothing, on duplicate or already-known ids, a wrong shape, non-finite values
        or a bias for a model without item biases.  A later train() needs data with the grown catalogue."""
        if not isinstance(ids, (list, tuple, np.ndarray)):
            raise ValueError("ids must be a list of item ids, got %s" % type(ids).__name__)
        ids = list(ids)
        if len(set(ids)) != len(ids):
            raise ValueError("ids hold duplicates")
        if not self._idmanager.itemid_mapped:
            self.build_itemid_map()
        known = [i for i in ids if i in self._idmanager.itemid_map]
        if known:
            raise ValueError("ids already known: %s" % known[:10])
        n, d = len(ids), self.opt.d
        X = np.asarray(rows, dtype=np.float32)
        if X.shape != (n, d):
            raise ValueError("rows must be (%d, %d), got %s" % (n, d, X.shape))
        if not np.isfinite(X).all():
            raise ValueError("rows hold non-finite values")
        has_bias = getattr(self, "Qb", None) is not None
        if bias is not None and not has_bias:
            raise ValueError("this model has no item biases")
        b = np.zeros(n, np.float32) if bias is None else np.asarray(bias, dtype=np.float32)
        if b.shape != (n,):
            raise ValueError("bias must be (%d,), got %s" % (n, b.shape))
        if not np.isfinite(b).all():
            raise ValueError("bias holds non-finite values")
        if self.opt._nrz_Q:
            X = self._normalize(X).astype(np.float32)
        G = np.zeros((n, self.Q.shape[1]), np.float32)
        G[:, :d] = X
        self.Q = np.ascontiguousarray(np.vstack([self.Q, G]), dtype=np.float32)
        if has_bias:
            self.Qb = np.ascontiguousarray(np.vstack([np.asarray(self.Qb, np.float32).reshape(-1, 1), b[:, None]]))
        start = len(self._idmanager.itemids)
        self._idmanager.itemids = list(self._idmanager.itemids) + ids
        self._idmanager.itemid_map.update({v: start + i for i, v in enumerate(ids)})

    def _check_catalogue(self):
        """train() on data whose item count no longer matches Q (after add_items) would index past the factors."""
        num_items = self.data.get_header()["num_items"]
        if getattr(self, "Q", None) is not None and self.Q.shape[0] != num_items:
            raise ValueError("Q has %d rows but the data has %d items: items were added with add_items; train on data "
                             "that includes them, or call initialize() to start again" % (self.Q.shape[0], num_items))

    def get_index_pool(self, pool, group="item"):
        if isinstance(pool, list):
            pool = np.array([p for p in self.get_index(pool, group) if p is not None])
        elif not isinstance(pool, np.ndarray):
            raise ValueError("Unexpected type for pool: %s" % type(pool))
        return pool

    # ---- queries ------------------------------------------------------------------------------
    def _get_topk_recommendation(self, p, Q, pb, Qb, pool, topk, num_workers):
        if pool is not None:
            Q = Q[pool]
            Qb = Qb[pool] if Qb is not None else None
        from buffalo_b200 import backend
        if backend.device_available() and 0 < topk <= 4096 and Q.shape[0] >= 1:
            # scores and top-k on the device (csrc/topk.cu); pb is constant per query row and does not change the order
            topks = backend.topk_host(p, Q, Qb, topk)
            return topks if pool is None else np.array([pool[t] for t in topks])
        scores = p.dot(Q.T)
        if pb is not None:
            scores += pb
        if Qb is not None:
            scores += Qb.T
        topks = self.get_topk(scores, k=topk, num_threads=num_workers)
        return topks if pool is None else np.array([pool[t] for t in topks])

    def topk_recommendation(self, keys, topk=10, pool=None):
        many = isinstance(keys, list)
        keys = keys if many else [keys]
        if not self._idmanager.userid_mapped:
            self.build_userid_map()
        if not self._idmanager.itemid_mapped:
            self.build_itemid_map()
        if pool is not None:
            pool = self.get_index_pool(pool, group="item")
            if len(pool) == 0:
                return []
        rows = [self._idmanager.userid_map[k] for k in keys if k in self._idmanager.userid_map]
        recs = list(self._get_topk_recommendation(rows, topk, pool))
        if not recs:
            return []
        named = {self._idmanager.userids[r]: [self._idmanager.itemids[v] for v in vv] for r, vv in recs}
        return named if many else next(iter(named.values()))

    def most_similar(self, key, topk=10, group="item", pool=None):
        if group != "item":
            return []
        if not self._idmanager.itemid_mapped:
            self.build_itemid_map()
        is_vec = isinstance(key, np.ndarray)
        q = key if is_vec else self._idmanager.itemid_map.get(key)
        if q is None:
            return []
        if pool is not None:
            pool = self.get_index_pool(pool, group="item")
            if len(pool) == 0:
                return []
        topks, scores = self._get_most_similar_item(q, topk, pool)
        return [(self._idmanager.itemids[k], v) for k, v in zip(topks, scores) if is_vec or k != q]

    def _get_most_similar_item(self, col, topk, Factor, nrz, pool):
        if isinstance(col, np.ndarray):
            q = col
        else:
            topk += 1
            q = Factor[col]
        cand = Factor if pool is None else Factor[pool]
        dot = q.dot(cand.T)
        if not nrz:
            dot = dot / (np.linalg.norm(q) * np.linalg.norm(cand, axis=1) + EPS)
        topks = self.get_topk(dot, k=topk, num_threads=self.opt.num_workers)
        scores = dot[topks]
        if pool is not None:
            topks = np.array([pool[t] for t in topks])
        return topks, scores

    def get_feature(self, name, group="item"):
        index = self.get_index(name, group=group)
        return None if index is None else self._get_feature(index, group)

    @abc.abstractmethod
    def _get_feature(self, index, group="item"):
        raise NotImplementedError

    def get_weighted_feature(self, weights, group="item", min_length=1):
        if isinstance(weights, dict):
            feat = [(self.get_feature(k), w) for k, w in weights.items()]
            feat = [f * w for f, w in feat if f is not None]
        else:
            feat = [f for f in (self.get_feature(k) for k, _ in weights) if f is not None]
        if len(feat) < min_length:
            return None
        feat = np.array(feat, dtype=np.float64).mean(axis=0)
        return (feat / np.linalg.norm(feat) + EPS).astype(np.float32)


class Serializable(abc.ABC):
    """Container: u64 count, then per object u64 name length, name, u64 payload length, pickle (base.py:275-311)."""

    def __init__(self, *args, **kwargs):
        pass

    def _get_data(self):
        return [("_idmanager", self._idmanager)]

    def save(self, path=None, with_itemid_map=True, with_userid_map=True, data_fields=[]):
        path = self.opt.model_path if path is None else path
        if with_itemid_map and not self._idmanager.itemid_mapped:
            self.build_itemid_map()
        if with_userid_map and not self._idmanager.userid_mapped:
            self.build_userid_map()
        items = [(k, v) for k, v in self._get_data() if not data_fields or k in data_fields]
        with open(path, "wb") as fout:
            fout.write(struct.pack("Q", len(items)))
            for name, obj in items:
                bname, blob = name.encode("utf-8"), pickle.dumps(obj, protocol=4)
                fout.write(struct.pack("Q", len(bname)) + bname + struct.pack("Q", len(blob)) + blob)

    def load(self, path, data_fields=[]):
        with open(path, "rb") as fin:
            (count,) = struct.unpack("Q", fin.read(8))
            for _ in range(count):
                (n,) = struct.unpack("Q", fin.read(8))
                name = fin.read(n).decode("utf8")
                (size,) = struct.unpack("Q", fin.read(8))
                if data_fields and name not in data_fields:
                    fin.seek(size, 1)
                    continue
                setattr(self, name, pickle.loads(fin.read(size)))

    @classmethod
    def instantiate(cls, cls_opt, path, data_fields):
        obj = cls(cls_opt().get_default_option())
        obj.load(path, data_fields)
        return obj

"""Validation metrics on the device (csrc/evaluate.cu, buffalo_b200/evaluate/device.py) against exact references, the
device top-k of the host path, and Evaluable's host loop."""
import os

import numpy as np
import pytest
import scipy.sparse

pytestmark = pytest.mark.gpu


def _t(a, dtype):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def _csr(rows):
    ptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
    keys = np.concatenate([np.asarray(r, dtype=np.int32) for r in rows] + [np.zeros(1, np.int32)])
    return ptr, keys


def masked(P, Q, bias, k, seen_rows):
    from buffalo_b200 import backend
    ptr, keys = _csr([sorted(s) for s in seen_rows])
    out = backend.eval_topk_masked(_t(P, np.float32), _t(Q, np.float32), None if bias is None else _t(bias, np.float32),
                                   k, _t(ptr, np.int64), _t(keys, np.int32), _t(np.arange(len(P)), np.int32))
    return out.cpu().numpy()


def exact_ranked(P, Q, bias, k, seen_rows):
    s = P.astype(np.float64) @ Q.astype(np.float64).T + (0 if bias is None else bias.astype(np.float64)[None, :])
    out = np.full((len(P), k), -1, np.int64)
    for u in range(len(P)):
        keep = np.setdiff1d(np.arange(Q.shape[0]), np.asarray(list(seen_rows[u]), dtype=np.int64))
        order = keep[np.lexsort((keep, -s[u, keep]))][:k]
        out[u, :len(order)] = order
    return out


@pytest.mark.parametrize("k", [1, 10, 4096])
@pytest.mark.parametrize("use_bias", [False, True])
def test_masked_topk_exact_on_integer_factors(cuda_lib, k, use_bias):
    rng = np.random.default_rng(k + use_bias)
    I, d = 9000, 8
    P = rng.integers(-2, 3, size=(12, d)).astype(np.float32)
    Q = rng.integers(-2, 3, size=(I, d)).astype(np.float32)
    bias = rng.integers(-3, 4, size=I).astype(np.float32) if use_bias else None
    every = np.arange(I)
    seen = [set(), {17}, set(rng.choice(I, 5000, replace=False).tolist()), set(every.tolist()) - {5, 4096, 8999},
            {4095, 4096, 4097}, {4095}, {4096}, {4097}, set(range(4000, 4200)), set(range(0, 8192)),
            set(range(8191, 9000)), set(rng.choice(I, 30, replace=False).tolist())]
    got = masked(P, Q, bias, k, seen)
    want = exact_ranked(P, Q, bias, k, seen)
    assert np.array_equal(got, want)
    assert (got[3] >= 0).sum() == min(3, k) and (got[3, 3:] == -1).all()


def test_masked_topk_fewer_items_than_k(cuda_lib):
    rng = np.random.default_rng(1)
    P = rng.integers(-1, 2, size=(5, 4)).astype(np.float32)
    Q = rng.integers(-1, 2, size=(30, 4)).astype(np.float32)
    seen = [set(), {0, 1, 2}, set(range(30)), {29}, set(range(0, 30, 2))]
    got = masked(P, Q, None, 50, seen)
    assert np.array_equal(got, exact_ranked(P, Q, None, 50, seen))
    assert (got[2] == -1).all()


@pytest.mark.parametrize("I,d,k", [(9000, 64, 10), (5000, 33, 100), (20000, 128, 50)])
def test_masked_topk_bitwise_equals_host_pipeline(cuda_lib, I, d, k):
    """The host path: bfl_topk_device top-(k + S), seen items dropped, first k kept."""
    from buffalo_b200 import backend
    rng = np.random.default_rng(I + d)
    P = rng.normal(size=(40, d)).astype(np.float32)
    Q = rng.normal(size=(I, d)).astype(np.float32)
    seen = [set(rng.choice(I, int(rng.integers(0, 300)), replace=False).tolist()) for _ in range(40)]
    S = max(len(s) for s in seen)
    idx, _ = backend.topk_device(_t(P, np.float32), _t(Q, np.float32), None, k + S)
    idx = idx.cpu().numpy()
    got = masked(P, Q, None, k, seen)
    for u in range(40):
        want = [c for c in idx[u] if c not in seen[u]][:k]
        assert got[u].tolist() == want


# ---- Evaluable: device path against the host path --------------------------------------------------------------

def _mm_db(tmp_path, U=500, I=700, density=0.03, p=0.1, max_samples=2000, seed=3):
    from buffalo import MatrixMarket, MatrixMarketOptions
    M = scipy.sparse.random(U, I, density=density, random_state=seed, format="coo")
    M.data[:] = np.random.default_rng(seed).integers(1, 5, size=M.nnz)
    opt = MatrixMarketOptions().get_default_option()
    opt.input.main = M
    opt.data.validation.p, opt.data.validation.max_samples = p, max_samples
    opt.data.path = str(tmp_path / "eval_mm.h5py")
    np.random.seed(seed)
    db = MatrixMarket(opt)
    db.create()
    return db


def _stream_db(tmp_path, U=300, I=400, seed=4, matrix=True):
    from buffalo import Stream, StreamOptions
    rng = np.random.default_rng(seed)
    lines = [" ".join("i%d" % x for x in rng.integers(0, I, size=int(rng.integers(2, 40)))) for _ in range(U)]
    main = tmp_path / "s.main"
    main.write_text("\n".join(lines) + "\n")
    opt = StreamOptions().get_default_option()
    opt.input.main = str(main)
    opt.data.tmp_dir = str(tmp_path)
    opt.data.path = str(tmp_path / "s.h5py")
    opt.data.internal_data_type = "matrix" if matrix else "stream"
    opt.data.validation.update(name="newest", n=2, max_samples=10 ** 7)
    np.random.seed(seed)
    db = Stream(opt)
    db.create()
    return db


def _close(a, b):
    assert set(a) == set(b), (a, b)
    for key in ("ndcg", "map", "accuracy", "auc"):
        if key in a:
            assert abs(a[key] - b[key]) <= 1e-12, (key, a[key], b[key])
    for key in ("rmse", "error"):
        assert abs(a[key] - b[key]) <= 1e-6 * abs(b[key]), (key, a[key], b[key])


def _both(algo, eval_samples=None):
    """(device, host) validation results on the same factors from the same np.random state; the states after agree."""
    algo.opt.validation.eval_samples = eval_samples
    np.random.seed(11)
    dev = algo.get_validation_results()
    s_dev = np.random.get_state()[1].copy()
    algo.opt._b200_device_eval = False
    np.random.seed(11)
    host = algo.get_validation_results()
    s_host = np.random.get_state()[1].copy()
    algo.opt._b200_device_eval = None
    assert np.array_equal(s_dev, s_host)
    return dev, host


CASES = [("ALS", {}), ("PLSI", {}), ("BPRMF", {"use_bias": True}), ("BPRMF", {"use_bias": False}), ("WARP", {}),
         ("WARP", {"score_func": "l2"})]


@pytest.mark.parametrize("name,kw", CASES)
@pytest.mark.parametrize("eval_samples", [None, 150])
def test_metrics_match_host_path(cuda_lib, tmp_path, name, kw, eval_samples):
    import buffalo
    from buffalo import aux
    db = _mm_db(tmp_path)
    opt = getattr(buffalo, name + "Option")().get_default_option()
    opt.update(d=24, random_seed=5, validation=aux.Option({"topk": 10}), **kw)
    algo = getattr(buffalo, name)(opt, data=db)
    algo.initialize()
    rng = np.random.default_rng(2)
    algo.P = rng.normal(size=algo.P.shape).astype(np.float32)
    algo.Q = rng.normal(size=algo.Q.shape).astype(np.float32)
    if name == "PLSI":
        algo.P, algo.Q = np.abs(algo.P), np.abs(algo.Q)
    if hasattr(algo, "Qb"):
        algo.Qb = rng.normal(size=algo.Qb.shape).astype(np.float32)
    dev, host = _both(algo, eval_samples)
    _close(dev, host)


TRAIN = [("ALS", {"_b200_resident": True}), ("ALS", {"_b200_resident": False}), ("PLSI", {"_b200_resident": True}),
         ("PLSI", {"_b200_resident": False}), ("BPRMF", {"use_bias": True}), ("WARP", {})]


@pytest.mark.parametrize("db_kind", ["mm", "stream"])
@pytest.mark.parametrize("name,kw", TRAIN)
def test_train_validation_matches_host_path(cuda_lib, tmp_path, db_kind, name, kw):
    """train() with validation every epoch: at each evaluation the device values equal the host path's on the same
    factors, and train() returns the device values."""
    import buffalo
    from buffalo import aux
    db = _mm_db(tmp_path) if db_kind == "mm" else _stream_db(tmp_path)
    if db_kind == "stream":
        assert len(np.unique(db.get_group("vali")["row"][:])) == db.get_header()["num_users"]
    opt = getattr(buffalo, name + "Option")().get_default_option()
    opt.update(d=16, num_iters=3, random_seed=7, validation=aux.Option({"topk": 10}), evaluation_period=1, **kw)
    algo = getattr(buffalo, name)(opt)
    algo.set_data(db)
    algo.initialize()
    seen = []

    def callback(i, metrics):
        dev = {k[4:]: v for k, v in metrics.items() if k.startswith("val_")}
        algo.opt._b200_device_eval = False
        host = algo.get_validation_results()
        algo.opt._b200_device_eval = None
        _close(dev, host)
        seen.append(dev)
    ret = algo.train(training_callback=callback)
    assert len(seen) == 3
    assert {k: ret["val_" + k] for k in seen[-1]} == seen[-1]


# ---- scale and determinism ---------------------------------------------------------------------------------------

class _ArrayData(object):
    """The slice of the Data interface the device evaluation reads, over in-memory arrays."""

    def __init__(self, U, I, indptr, keys, vrow, vcol, vval):
        self.header = {"num_users": U, "num_items": I, "num_nnz": len(keys)}
        self.groups = {"rowwise": {"indptr": indptr, "key": keys}, "vali": {"row": vrow, "col": vcol, "val": vval}}

    def get_header(self):
        return self.header

    def get_group(self, name):
        return self.groups[name]


def _numpy_metrics(ranked, users, seen_len, gt, num_items, topk):
    """Vectorised fp64 restatement of Evaluable's per-row formulas from ranked lists [n, topk] (-1 padded)."""
    ok = seen_len > 0
    ranked, users = ranked[ok], users[ok]
    valid = ranked >= 0
    hits = np.zeros(ranked.shape)
    for i, (u, r) in enumerate(zip(users, ranked)):
        hits[i] = np.isin(r, gt[u]) & (r >= 0)
    n_pos = np.array([len(gt[u]) for u in users], dtype=np.float64)
    gains = 1.0 / np.log2(np.arange(2, topk + 2))
    ideal = np.cumsum(gains)
    cum = np.cumsum(hits, axis=1)
    miss = ((1 - hits) * valid).sum(1)
    m = np.minimum(n_pos, topk).astype(np.int64)
    n_neg = num_items - n_pos
    auc = ((1 - hits) * cum * valid).sum(1) + (cum[:, -1] + n_pos) / 2.0 * (n_neg - miss)
    return {"ndcg": np.mean((hits * gains).sum(1) / ideal[m - 1]),
            "map": np.mean((hits * cum / np.arange(1, topk + 1)).sum(1) / m),
            "accuracy": np.mean(cum[:, -1] / n_pos), "auc": np.mean(auc / (n_pos * n_neg))}


def test_scale_determinism_and_batches(cuda_lib):
    from buffalo_b200.evaluate import device
    rng = np.random.default_rng(9)
    U, I, d, topk = 200_000, 50_000, 8, 10
    lens = np.minimum(rng.zipf(1.6, size=U), 10_000)
    lens[:3] = [10_000, 9_999, 0]
    rows = [np.sort(rng.choice(I, int(n), replace=False)) if n > 64 else np.unique(rng.integers(0, I, int(n)))
            for n in lens]
    for r in rows[5:2000:3]:
        rng.shuffle(r)                         # unsorted rows: the device sort must put them in order
    indptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
    keys = np.concatenate(rows).astype(np.int32)
    vrow = np.repeat(np.arange(U), 2).astype(np.int32)
    vcol = rng.integers(0, I, size=2 * U).astype(np.int32)
    vval = np.ones(2 * U, np.float32)
    data = _ArrayData(U, I, indptr, keys, vrow, vcol, vval)
    P = rng.integers(-3, 4, size=(U, d)).astype(np.float32)
    Q = rng.integers(-3, 4, size=(I, d)).astype(np.float32)
    model = device.EvalModel(P, Q, None, None, False)
    runs = []
    for max_users in (None, None, 7_777):
        data.__dict__.pop("_b200_validation_state", None)
        ev = device.Evaluation(data, model, max_users=max_users)
        runs.append((ev.ranking(topk, None), ev.scores()))
    assert runs[0] == runs[1] == runs[2]
    assert not ev.st.resident
    # the ranked lists of every user, checked exactly on a sample and fed to the NumPy metric restatement
    import torch
    st = device.Evaluation(data, model).st
    sp, sk, sr = st.seen_for(np.arange(U))
    ranked = torch.cat([device.backend.eval_topk_masked(_t(P[s:s + 50_000], np.float32), _t(Q, np.float32), None,
                                                        topk, sp, sk, sr[s:s + 50_000]) for s in range(0, U, 50_000)])
    ranked = ranked.cpu().numpy()
    sample = np.concatenate([[0, 1, 2], rng.choice(U, 300, replace=False), np.arange(5, 2000, 3)[:100]])
    want = exact_ranked(P[sample], Q, None, topk, [set(rows[u].tolist()) for u in sample])
    assert np.array_equal(ranked[sample], want)
    gt = {}
    for r, c in zip(vrow, vcol):
        gt.setdefault(int(r), set()).add(int(c))
    gt = {u: np.fromiter(s, np.int64) for u, s in gt.items()}
    ref = _numpy_metrics(ranked, np.arange(U), lens, gt, I, topk)
    for key, val in ref.items():
        assert abs(runs[0][0][key] - val) <= 1e-12, (key, runs[0][0][key], val)
    err = (P[vrow] * Q[vcol]).sum(1).astype(np.float64) - vval
    assert abs(runs[0][1]["rmse"] - np.sqrt(np.mean(err ** 2))) <= 1e-9

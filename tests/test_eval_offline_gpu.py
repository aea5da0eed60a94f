"""Offline evaluation on the device (csrc/offline_eval.cu, buffalo_b200/evaluate/offline.py) against the fp64 reference
(tests/eval_offline_ref.py), the lists of ParALS.topk_recommendation, the validation path and the IVF index."""
import numpy as np
import pytest
import scipy.sparse

from tests import eval_offline_ref as ref

pytestmark = pytest.mark.gpu

NAMES = ("hit", "recall", "precision", "ndcg", "map", "mrr")


@pytest.fixture(scope="module", autouse=True)
def _release_cached_memory():
    """The production-size case leaves about a gigabyte in torch's caching allocator: hand it back so that the tests
    after this module see the device as they would without it."""
    yield
    import torch
    torch.cuda.empty_cache()


def _lists(rng, n, K, I, pad_rows=0.3, holes=False):
    """(n, K) int32 lists of distinct items; a share of the rows padded with -1 at the end, or anywhere with holes."""
    out = np.stack([rng.choice(I, K, replace=False) for _ in range(n)]).astype(np.int32)
    for r in np.flatnonzero(rng.random(n) < pad_rows):
        cut = int(rng.integers(0, K + 1))
        out[r, cut:] = -1
    if holes:
        out[rng.random(out.shape) < 0.1] = -1
    return out


def _truth(rng, n, I, lens, ranked=None):
    """A held-out matrix whose row r has lens[r] items, some of them drawn from ranked[r] so that there are hits."""
    rows, cols = [], []
    for r, m in enumerate(lens):
        pick = rng.choice(I, int(m), replace=False)
        if ranked is not None and m:
            from_list = ranked[r][ranked[r] >= 0][:int(m)]
            take = from_list[rng.random(len(from_list)) < 0.5]
            pick = np.unique(np.concatenate([pick[:int(m) - len(take)], take]))
        rows.append(np.full(len(pick), r))
        cols.append(pick)
    r, c = np.concatenate(rows), np.concatenate(cols)
    return scipy.sparse.csr_matrix((np.ones(len(r)), (r, c)), shape=(n, I))


def _check(got, want, rel=1e-12):
    assert got["users"] == want["users"]
    for key, val in want.items():
        if key in ("users", "rows", "per_user"):
            continue
        if key.startswith("coverage"):
            assert got[key] == val, key
        elif key.startswith("ild"):
            assert (np.isnan(val) and np.isnan(got[key])) or abs(got[key] - val) <= 1e-5, (key, got[key], val)
        else:
            assert abs(got[key] - val) <= rel * max(abs(val), 1e-300), (key, got[key], val)
    assert set(got) - {"rows", "per_user"} == set(want) - {"rows", "per_user"}
    if "per_user" in got:
        assert np.array_equal(got["rows"], want["rows"])
        for key, val in want["per_user"].items():
            g = got["per_user"][key]
            if key.startswith("ild"):
                assert np.array_equal(np.isnan(g), np.isnan(val)), key
                ok = ~np.isnan(val)
                assert np.abs(g[ok] - val[ok]).max(initial=0) <= 1e-5, key
            else:
                assert np.allclose(g, val, rtol=1e-12, atol=1e-300), key


@pytest.mark.parametrize("K,cutoffs,holes", [(1, [1], False), (64, [64, 1, 10, 10, 33], True),
                                             (4096, [100, 4096, 1, 100, 2048], False)])
def test_lists_against_reference(cuda_lib, K, cutoffs, holes):
    from buffalo_b200.evaluate import evaluate_lists
    rng = np.random.default_rng(K)
    n, I = 120, 20_000
    ranked = _lists(rng, n, K, I, holes=holes)
    lens = rng.integers(0, 40, n)
    lens[:4] = [1, 10_000, 0, 2]
    T = _truth(rng, n, I, lens, ranked)
    got = evaluate_lists(ranked, T, cutoffs, per_user=True)
    _check(got, ref.evaluate(ranked, T, cutoffs))


def test_diversity_against_reference(cuda_lib):
    from buffalo_b200.evaluate import evaluate_lists
    rng = np.random.default_rng(5)
    n, I, d = 150, 3000, 70                     # d not a multiple of the Gram tile
    Q = rng.normal(size=(I, d)).astype(np.float32)
    Q[rng.choice(I, 300, replace=False)] = 0.0  # zero-norm rows
    ranked = _lists(rng, n, 256, I, holes=True)
    ranked[0, 1:] = -1                          # one valid entry
    ranked[1, :] = -1                           # none
    ranked[2, :2] = [7, 7]                      # a repeated item
    T = _truth(rng, n, I, rng.integers(1, 30, n), ranked)
    cutoffs = [256, 2, 17, 2, 100]
    got = evaluate_lists(ranked, T, cutoffs, item_factors=Q, per_user=True)
    _check(got, ref.evaluate(ranked, T, cutoffs, Q))
    assert np.isnan(got["per_user"]["ild@256"][0]) and np.isnan(got["per_user"]["ild@2"][1])


def test_per_row_values_bitwise_across_runs_and_batches(cuda_lib, monkeypatch):
    from buffalo_b200.evaluate import evaluate_lists, offline
    rng = np.random.default_rng(2)
    n, I, d = 5000, 8000, 32
    ranked = _lists(rng, n, 200, I, holes=True)
    T = _truth(rng, n, I, rng.integers(0, 50, n), ranked)
    Q = rng.normal(size=(I, d)).astype(np.float32)
    runs = []
    for cap in (None, None, 7, 1777):
        monkeypatch.setattr(offline, "BATCH_ROWS", cap)
        runs.append(evaluate_lists(ranked, T, [5, 50, 200], item_factors=Q, per_user=True))
    for r in runs[1:]:
        assert np.array_equal(r["rows"], runs[0]["rows"])
        for key, val in runs[0]["per_user"].items():
            assert np.array_equal(r["per_user"][key], val, equal_nan=True), key
        assert {k: v for k, v in r.items() if k not in ("rows", "per_user")} == \
               {k: v for k, v in runs[0].items() if k not in ("rows", "per_user")}


# ---- Evaluable.evaluate ---------------------------------------------------------------------------------------------

def _model(tmp_path, name, kw, db=None):
    import buffalo
    from buffalo import aux
    from tests.test_eval_gpu import _mm_db
    db = db or _mm_db(tmp_path)
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
    return algo


@pytest.mark.parametrize("name,kw", [("ALS", {}), ("BPRMF", {"use_bias": True}), ("WARP", {}), ("PLSI", {})])
@pytest.mark.parametrize("exclude", ["train", "none", "matrix"])
def test_evaluate_equals_topk_recommendation_lists(cuda_lib, tmp_path, name, kw, exclude):
    from buffalo_b200.evaluate import evaluate_lists
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    algo = _model(tmp_path, name, kw)
    U, I = algo.P.shape[0], algo.Q.shape[0]
    rng = np.random.default_rng(3)
    keep = np.ones(U)
    keep[5] = 0                                 # a row without truth
    T = scipy.sparse.diags(keep) @ scipy.sparse.random(U, I, density=0.02, format="csr", random_state=rng)
    exclude_seen = {"train": True, "none": False,
                    "matrix": scipy.sparse.random(U, I, density=0.05, format="csr", random_state=rng)}[exclude]
    cutoffs = [20, 5, 50]
    got = algo.evaluate(T, cutoffs, exclude_seen=exclude_seen, diversity=True, per_user=True)
    par = (ParBPRMF if name == "BPRMF" else ParALS)(algo)
    _, lists, _ = par.topk_recommendation(np.arange(U, dtype=np.int32), topk=50, exclude_seen=exclude_seen)
    lists = np.asarray(lists)
    from_lists = evaluate_lists(lists, T, cutoffs, item_factors=algo.Q, per_user=True)
    assert {k: v for k, v in got.items() if k not in ("rows", "per_user")} == \
           {k: v for k, v in from_lists.items() if k not in ("rows", "per_user")}
    for key, val in from_lists["per_user"].items():
        assert np.array_equal(got["per_user"][key], val, equal_nan=True), key
    assert 5 not in got["rows"].tolist()
    _check(got, ref.evaluate(lists, T, cutoffs, algo.Q))


def test_evaluate_equals_validation_results(cuda_lib, tmp_path):
    algo = _model(tmp_path, "ALS", {})
    db = algo.data
    v = db.get_group("vali")
    U, I = algo.P.shape[0], algo.Q.shape[0]
    vali = scipy.sparse.csr_matrix((np.asarray(v["val"][:], np.float64), (v["row"][:], v["col"][:])), shape=(U, I))
    ends = np.asarray(db.get_group("rowwise")["indptr"][:], np.int64)
    # the validation path skips users without training items
    vali = scipy.sparse.diags((np.diff(ends, prepend=0) > 0).astype(np.float64)) @ vali
    val = algo.get_validation_results()
    got = algo.evaluate(vali, [10], exclude_seen=True)
    assert got["users"] > 100
    assert abs(got["ndcg@10"] - val["ndcg"]) <= 1e-12
    assert abs(got["map@10"] - val["map"]) <= 1e-12
    assert abs(got["recall@10"] - val["accuracy"]) <= 1e-12


def test_ivf_lists_at_full_nprobe_give_the_exact_metrics(cuda_lib, tmp_path):
    from buffalo_b200.evaluate import evaluate_lists
    from buffalo_b200.parallel.base import ParALS
    algo = _model(tmp_path, "ALS", {})
    U, I = algo.P.shape[0], algo.Q.shape[0]
    T = scipy.sparse.random(U, I, density=0.03, format="csr", random_state=np.random.default_rng(8))
    par = ParALS(algo)
    par.build_index(16)
    users = np.arange(U, dtype=np.int32)
    exact = np.asarray(par.topk_recommendation(users, topk=40)[1])
    ivf = np.asarray(par.topk_recommendation(users, topk=40, nprobe=16)[1])
    a = evaluate_lists(exact, T, [10, 40], item_factors=algo.Q, per_user=True)
    b = evaluate_lists(ivf, T, [10, 40], item_factors=algo.Q, per_user=True)
    assert {k: v for k, v in a.items() if k != "per_user" and k != "rows"} == \
           {k: v for k, v in b.items() if k != "per_user" and k != "rows"}
    for key, val in a["per_user"].items():
        assert np.array_equal(b["per_user"][key], val, equal_nan=True), key


def test_production_size(cuda_lib, monkeypatch):
    """2^18 rows, K = 1000: a sample of rows against the reference, coverage exactly, and the same values with the
    rows cut into batches."""
    from buffalo_b200.evaluate import evaluate_lists, offline
    rng = np.random.default_rng(11)
    n, I, K = 1 << 18, 100_000, 1000
    ranked = rng.integers(0, I, size=(n, K), dtype=np.int32)    # repeats allowed: each occurrence counts
    ranked[rng.random(n) < 0.1, 600:] = -1
    lens = np.minimum(rng.zipf(1.8, n), 500)
    r = np.repeat(np.arange(n), lens)
    c = rng.integers(0, I, len(r))
    hit_rows = rng.random(n) < 0.5                                 # half the rows hold out items of their own list
    r2 = np.flatnonzero(hit_rows)
    c2 = ranked[r2, rng.integers(0, 100, len(r2))]
    keep = c2 >= 0
    T = scipy.sparse.csr_matrix((np.ones(len(r) + keep.sum()), (np.concatenate([r, r2[keep]]),
                                                                np.concatenate([c, c2[keep]]))), shape=(n, I))
    cutoffs = [10, 100, 1000]
    got = evaluate_lists(ranked, T, cutoffs, per_user=True)
    assert got["users"] == n
    sample = np.concatenate([[0, n - 1], rng.choice(n, 300, replace=False)])
    truth = ref.truth_rows(T[sample])
    for K_ in cutoffs:
        for i, row in enumerate(sample):
            want = ref.row_metrics(ranked[row], truth[i], K_)
            for j, name in enumerate(NAMES):
                g = got["per_user"]["%s@%d" % (name, K_)][row]
                assert abs(g - want[j]) <= 1e-12 * max(abs(want[j]), 1e-300), (name, K_, row, g, want[j])
        for name in NAMES:
            per = got["per_user"]["%s@%d" % (name, K_)]
            assert abs(got["%s@%d" % (name, K_)] - per.mean()) <= 1e-12 * abs(per.mean())
        items = ranked[:, :K_]
        assert got["coverage@%d" % K_] == len(np.unique(items[items >= 0])) / I
    monkeypatch.setattr(offline, "BATCH_ROWS", 50_000)
    again = evaluate_lists(ranked, T, cutoffs, per_user=True)
    for key, val in got["per_user"].items():
        assert np.array_equal(again["per_user"][key], val), key
    assert {k: v for k, v in again.items() if k != "per_user" and k != "rows"} == \
           {k: v for k, v in got.items() if k != "per_user" and k != "rows"}


@pytest.mark.parametrize("cutoffs", [[1], [5], [17, 255], [2, 3]])
def test_diversity_with_an_odd_or_small_largest_cutoff(cuda_lib, tmp_path, cutoffs):
    """The diversity kernel's shared-memory layout for every kind of largest cutoff (odd, 1, just under 256): against
    the reference through evaluate_lists, and through evaluate on a model."""
    from buffalo_b200.evaluate import evaluate_lists
    rng = np.random.default_rng(sum(cutoffs))
    n, I, d = 90, 2000, 45
    Q = rng.normal(size=(I, d)).astype(np.float32)
    Q[rng.choice(I, 100, replace=False)] = 0.0
    K = max(cutoffs) + 3
    ranked = _lists(rng, n, K, I, holes=True)
    T = _truth(rng, n, I, rng.integers(1, 20, n), ranked)
    got = evaluate_lists(ranked, T, cutoffs, item_factors=Q, per_user=True)
    _check(got, ref.evaluate(ranked, T, cutoffs, Q))
    algo = _model(tmp_path, "ALS", {})
    U, I = algo.P.shape[0], algo.Q.shape[0]
    T = scipy.sparse.random(U, I, density=0.03, format="csr", random_state=rng)
    res = algo.evaluate(T, cutoffs, exclude_seen=False, diversity=True, per_user=True)
    from buffalo_b200.parallel.base import ParALS
    lists = np.asarray(ParALS(algo).topk_recommendation(np.arange(U, dtype=np.int32), topk=max(cutoffs))[1])
    _check(res, ref.evaluate(lists, T, cutoffs, algo.Q))

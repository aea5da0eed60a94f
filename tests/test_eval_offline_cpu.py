"""Offline evaluation (Evaluable.evaluate, evaluate_lists) where no GPU is needed: every argument check raises before
any device work, without a GPU a valid call raises the backend's "no CPU fallback" error, the fp64 reference
(tests/eval_offline_ref.py) gives hand-computed values, and its ndcg / map / recall are the validation path's ndcg / map /
accuracy on the same lists."""
import numpy as np
import pytest
import scipy.sparse

from tests import eval_offline_ref as ref
from tests.test_fold_in_cpu import cpu_model


@pytest.fixture
def no_device_work(monkeypatch):
    from buffalo_b200 import backend

    def refuse(*a, **k):
        raise AssertionError("device work before the argument checks finished")
    monkeypatch.setattr(backend, "require_device", refuse)
    monkeypatch.setattr(backend, "device_free_bytes", refuse)


def _test(n, I, seed=0):
    return scipy.sparse.random(n, I, density=0.2, format="csr", random_state=np.random.default_rng(seed))


def _warp(score_func):
    from buffalo_b200.algo.options import WARPOption
    from buffalo_b200.algo.warp import WARP
    from buffalo_b200.misc import aux
    m = WARP.__new__(WARP)
    m.opt = aux.Option(WARPOption().get_default_option())
    m.opt.update(dict(d=4, score_func=score_func))
    m.P, m.Q = np.ones((6, 4), np.float32), np.ones((9, 4), np.float32)
    return m


def test_evaluate_lists_checks_before_device_work(no_device_work):
    from buffalo_b200.evaluate import evaluate_lists
    I = 20
    ranked = np.zeros((4, 10), np.int32)
    T = _test(4, I)
    for bad in (np.zeros(4, np.int32), np.zeros((4, 10), np.float32), np.zeros((4, 0), np.int32)):
        with pytest.raises(ValueError, match="ranked"):
            evaluate_lists(bad, T)
    for v in (-2, I):
        r = ranked.copy()
        r[2, 3] = v
        with pytest.raises(ValueError, match="outside"):
            evaluate_lists(r, T)
    with pytest.raises(ValueError, match="test"):
        evaluate_lists(ranked, T.toarray())
    with pytest.raises(ValueError, match="test"):
        evaluate_lists(ranked, _test(5, I))
    for cutoffs in ([0], [4097], [], [True], [2.5], "10", [10, -1]):
        with pytest.raises(ValueError, match="cutoffs"):
            evaluate_lists(ranked, T, cutoffs=cutoffs)
    with pytest.raises(ValueError, match="width"):
        evaluate_lists(ranked, T, cutoffs=[5, 11])
    wide = np.zeros((4, 300), np.int32)
    with pytest.raises(ValueError, match="256"):
        evaluate_lists(wide, T, cutoffs=[257], item_factors=np.ones((I, 3), np.float32))
    for F in (np.ones((I + 1, 3)), np.ones(I), np.ones((I, 0))):
        with pytest.raises(ValueError, match="item_factors"):
            evaluate_lists(ranked, T, item_factors=F)
    bad = T.copy()
    bad.indices[0] = I + 2                     # scipy does not check index ranges after construction
    with pytest.raises(ValueError, match="outside"):
        evaluate_lists(ranked, bad)


def test_evaluate_checks_before_device_work(no_device_work):
    m = cpu_model("als", U=6, I=9)
    T = _test(6, 9)
    with pytest.raises(ValueError, match="test"):
        m.evaluate(_test(6, 10))
    with pytest.raises(ValueError, match="test"):
        m.evaluate(T.toarray())
    for cutoffs in ([0], [4097], (10, 4097)):
        with pytest.raises(ValueError, match="cutoffs"):
            m.evaluate(T, cutoffs=cutoffs)
    with pytest.raises(ValueError, match="256"):
        m.evaluate(T, cutoffs=[10, 257], diversity=True)
    with pytest.raises(ValueError, match="training data"):
        m.evaluate(T, exclude_seen=True)
    with pytest.raises(ValueError, match="exclude_seen"):
        m.evaluate(T, exclude_seen=_test(5, 9))
    with pytest.raises(ValueError, match="l2"):
        _warp("l2").evaluate(T)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from buffalo_b200 import _cabi
    from buffalo_b200.evaluate import evaluate_lists
    T = _test(6, 9)
    with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
        evaluate_lists(np.zeros((6, 3), np.int32), T, cutoffs=[3])
    with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
        cpu_model("als", U=6, I=9).evaluate(T, exclude_seen=False)
    with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
        _warp("dot").evaluate(T, exclude_seen=False)


def test_reference_hand_computed():
    # truth {1, 4, 7}; list 4, 2, 1, -1, 7
    hit, recall, precision, ndcg, ap, rr, _ = ref.row_metrics([4, 2, 1, -1, 7], [1, 4, 7], 5)
    g = 1.0 / np.log2([2, 3, 4, 5, 6])
    assert (hit, recall, precision, rr) == (1.0, 1.0, 3 / 5, 1.0)
    assert np.isclose(ndcg, (g[0] + g[2] + g[4]) / (g[0] + g[1] + g[2]), rtol=1e-15)
    assert np.isclose(ap, (1 / 1 + 2 / 3 + 3 / 5) / 3, rtol=1e-15)
    # at K = 2: one hit of three, ideal over min(3, 2) positions
    hit, recall, precision, ndcg, ap, rr, _ = ref.row_metrics([4, 2, 1, -1, 7], [1, 4, 7], 2)
    assert (hit, recall, precision, rr) == (1.0, 1 / 3, 1 / 2, 1.0)
    assert np.isclose(ndcg, g[0] / (g[0] + g[1]), rtol=1e-15) and np.isclose(ap, 1 / 2, rtol=1e-15)
    # first hit at position 3; a repeated item counts each time; K past the list's width pads
    hit, recall, precision, ndcg, ap, rr, _ = ref.row_metrics([0, 9, 5, 5], [5], 6)
    assert (hit, recall, precision, rr) == (1.0, 2.0, 2 / 6, 1 / 3)
    assert np.isclose(ap, 1 / 3 + 2 / 4, rtol=1e-15)
    # no hit
    assert ref.row_metrics([-1, -1, 3], [5], 3)[:6] == (0.0, 0.0, 0.0, 0.0, 0.0, 0.0)


def test_reference_ild_and_coverage():
    Q = np.array([[1, 0], [0, 1], [1, 1], [0, 0], [2, 0]], np.float64)
    # pairs of (0, 1, 4): 1 - 0, 1 - 1, 1 - 0
    assert np.isclose(ref.row_metrics([0, 1, -1, 4], [0], 4, Q)[6], 2 / 3, rtol=1e-15)
    # the zero row has cos 0 with everything
    assert np.isclose(ref.row_metrics([3, 0], [0], 2, Q)[6], 1.0, rtol=1e-15)
    assert np.isclose(ref.row_metrics([0, 2], [0], 2, Q)[6], 1 - 1 / np.sqrt(2), rtol=1e-15)
    assert ref.row_metrics([0, -1, -1], [0], 3, Q)[6] is None and ref.row_metrics([0, 1], [0], 1, Q)[6] is None
    T = scipy.sparse.csr_matrix(np.array([[1, 0, 0, 0, 0], [0, 0, 0, 0, 0], [0, 1, 0, 0, 0]], np.float32))
    ranked = np.array([[0, 1, 2], [3, 4, 2], [1, -1, 4]])
    res = ref.evaluate(ranked, T, [1, 3], Q)
    assert res["users"] == 2 and res["rows"].tolist() == [0, 2]   # row 1 has no truth
    assert res["coverage@1"] == 2 / 5 and res["coverage@3"] == 4 / 5
    assert res["hit@1"] == 1.0 and res["precision@3"] == 1 / 3
    assert np.isclose(res["ild@3"], np.mean([ref.row_metrics(ranked[0], [0], 3, Q)[6], 1.0]), rtol=1e-15)
    assert np.isnan(res["ild@1"])


def test_reference_truth_sums_duplicates():
    T = scipy.sparse.coo_matrix((np.array([1.0, -1.0, 2.0, 0.0, 3.0]), (np.array([0, 0, 0, 1, 1]),
                                                                          np.array([3, 3, 1, 2, 0]))), shape=(2, 5))
    rows = ref.truth_rows(T)
    assert rows[0].tolist() == [1] and rows[1].tolist() == [0]


def test_truth_csr_matches_reference():
    from buffalo_b200.evaluate.offline import truth_csr
    rng = np.random.default_rng(4)
    n, I = 40, 30
    r, c = rng.integers(0, n, 300), rng.integers(0, I, 300)
    v = rng.integers(-1, 2, 300).astype(np.float64)
    T = scipy.sparse.coo_matrix((v, (r, c)), shape=(n, I))
    ptr, keys, rows = truth_csr(T, n, I)
    want = ref.truth_rows(T)
    beg = np.concatenate([[0], ptr[:-1]])
    assert [keys[beg[i]:ptr[i]].tolist() for i in range(n)] == [w.tolist() for w in want]
    assert rows.tolist() == [i for i in range(n) if len(want[i])]


def test_reference_equals_validation_formulas():
    """The validation host loop (Evaluable._evaluate_ranking_metrics) on fixed candidate lists: its ndcg, map and
    accuracy are the reference's ndcg, map and recall on the lists it keeps (seen items dropped, first topk)."""
    from tests.test_eval_cpu import _Model
    rng = np.random.default_rng(7)
    U, I, topk = 60, 40, 10
    gt = {u: set(rng.choice(I, int(rng.integers(1, 15)), replace=False).tolist()) for u in range(U)}
    seen = {u: set(rng.choice(I, int(rng.integers(1, 12)), replace=False).tolist()) for u in range(U)}
    cand = {u: rng.permutation(I)[:topk + 12 - int(rng.integers(0, 8))] for u in range(U)}
    m = _Model()
    m.opt.validation = type(m.opt.validation)({"topk": topk, "batch": 16, "eval_samples": None})
    m._get_topk_recommendation = lambda rows, topk: [(r, cand[r]) for r in rows]
    m.data.vali_data = {"vali_gt": gt, "vali_rows": np.arange(U), "validation_seen": seen,
                        "validation_max_seen_size": 12}
    m.data.get_header = lambda: {"num_items": I}
    from buffalo_b200.evaluate import Evaluable
    host = Evaluable._evaluate_ranking_metrics(m)   # the real host loop, not _Model's stub
    ranked = np.full((U, topk), -1, np.int64)
    for u in range(U):
        kept = [c for c in cand[u] if c not in seen[u]][:topk]
        ranked[u, :len(kept)] = kept
    T = scipy.sparse.lil_matrix((U, I))
    for u, items in gt.items():
        T[u, sorted(items)] = 1.0
    res = ref.evaluate(ranked, T, [topk])
    assert abs(res["ndcg@10"] - host["ndcg"]) <= 1e-12
    assert abs(res["map@10"] - host["map"]) <= 1e-12
    assert abs(res["recall@10"] - host["accuracy"]) <= 1e-12


def test_per_row_terms_larger_than_the_device_refused(monkeypatch):
    """The [n_cut, rows, 8] fp64 terms are checked against the free device memory before anything is allocated."""
    from buffalo_b200 import backend
    from buffalo_b200.evaluate import evaluate_lists, offline
    monkeypatch.setattr(backend, "require_device", lambda: None)
    monkeypatch.setattr(backend, "device_free_bytes", lambda: 2 * 64 * 3 * 6 - 1)   # just under 6 rows x 3 cutoffs

    def refuse(*a, **k):
        raise AssertionError("device work after the memory check failed")
    monkeypatch.setattr(offline, "_device", refuse)
    T = scipy.sparse.csr_matrix(np.ones((6, 9)))
    with pytest.raises(MemoryError, match="6 rows at 3 cutoffs"):
        evaluate_lists(np.zeros((6, 5), np.int32), T, cutoffs=[1, 3, 5])
    with pytest.raises(MemoryError, match="fewer cutoffs"):
        cpu_model("als", U=6, I=9).evaluate(T, cutoffs=[1, 3, 5], exclude_seen=False)
    offline.check_slab_memory(3, 5)                       # 5 rows fit

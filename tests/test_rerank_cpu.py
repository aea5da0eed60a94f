"""MMR re-ranking (topk_recommendation(diversify=w), rerank_mmr) where no GPU is needed: the fp64 reference against
hand-computed answers, the NumPy path against the reference, diversify=0 against the plain NumPy result, and the
argument errors raised before any device work."""
import numpy as np
import pytest
import scipy.sparse

from tests.rerank_ref import check_greedy, gap_inputs, mmr_ref, random_inputs
from tests.test_ivf_cpu import cpu_model
from tests.test_serve_cand_cpu import pool_matrix, random_rows


@pytest.fixture
def numpy_path(monkeypatch):
    """The NumPy path: no device, whatever the machine has."""
    from buffalo_b200 import backend
    monkeypatch.setattr(backend, "device_available", lambda: False)


@pytest.fixture
def no_device_work(monkeypatch):
    """Any serve-handle step, or the NumPy path, fails the test."""
    from buffalo_b200 import backend
    from buffalo_b200.parallel import base

    def refuse(*a, **k):
        raise AssertionError("device work before the checks finished")
    for name in ("set_items", "set_queries", "bind_queries", "set_pool", "topk", "topk_device", "topk_seen",
                 "topk_seen_device", "topk_candidates", "topk_candidates_device", "rerank_mmr_device"):
        monkeypatch.setattr(backend.Serve, name, refuse)
    monkeypatch.setattr(backend, "Serve", refuse)
    monkeypatch.setattr(base, "mmr_numpy", refuse)
    monkeypatch.setattr(backend, "device_available", lambda: True)


# --- the reference against hand-computed answers ------------------------------------------------------------------

def test_ref_step_by_step():
    # A = (1, 0), B = (1, 0.1) close to A, C = (0, 1); scores 3, 2.9, 1 -> rel 1, 0.95, 0
    F = np.array([[1, 0], [1, 0.1], [0, 1]], np.float32)
    idx, val = np.array([[0, 1, 2]], np.int32), np.array([[3, 2.9, 1]], np.float32)
    cos_ab = 1 / np.sqrt(1.01)
    rel_b = (np.float64(np.float32(2.9)) - 1) / 2
    # w = 0.5: A first; then B has 0.5 rel_b - 0.5 cos_ab < 0 = C's 0.5 * 0 - 0.5 * 0; B last
    assert 0.5 * rel_b - 0.5 * cos_ab < 0
    keys, scores = mmr_ref(idx, val, F, 3, 0.5)
    assert keys.tolist() == [[0, 2, 1]]
    assert scores.tolist() == [[3, 1, np.float32(2.9)]]
    # w = 0.1: B's 0.9 rel_b - 0.1 cos_ab > 0 = C's: plain order
    assert mmr_ref(idx, val, F, 3, 0.1)[0].tolist() == [[0, 1, 2]]
    # w = 0: the first k in order; w = 1: position 0, then the least similar to it, then the rest
    assert mmr_ref(idx, val, F, 2, 0.0)[0].tolist() == [[0, 1]]
    assert mmr_ref(idx, val, F, 3, 1.0)[0].tolist() == [[0, 2, 1]]


def test_ref_four_items_known_cosines():
    # unit rows at 0, 10, 90 and 135 degrees with equal scores (rel = 1 everywhere), w = 0.5: similarity alone decides.
    # step 0: all tie -> position 0; step 1: cos to 0 deg is 0.98, 0, -0.71 -> 135; step 2: max cos to {0, 135} is
    # 0.98 for 10 and cos 45 = 0.71 for 90 -> 90; step 3: 10
    ang = np.radians([0, 10, 90, 135])
    F = np.stack([np.cos(ang), np.sin(ang)], 1).astype(np.float32)
    idx, val = np.array([[0, 1, 2, 3]], np.int32), np.full((1, 4), 0.5, np.float32)
    assert mmr_ref(idx, val, F, 4, 0.5)[0].tolist() == [[0, 3, 2, 1]]


def test_ref_ties_go_to_the_earlier_position():
    F = np.eye(4, dtype=np.float32)                 # orthogonal: every cos is 0
    idx = np.array([[3, 1, 2, 0]], np.int32)
    val = np.array([[1, 1, 1, 1]], np.float32)
    for w in (0.0, 0.3, 1.0):
        assert mmr_ref(idx, val, F, 4, w)[0].tolist() == [[3, 1, 2, 0]]


def test_ref_all_equal_scores_rel_one():
    # rel = 1 for all; w = 0.5: after position 0 (item 0) the orthogonal item 2 beats item 1 (cos 1 to item 0)
    F = np.array([[1, 0], [2, 0], [0, 1]], np.float32)
    idx, val = np.array([[0, 1, 2]], np.int32), np.full((1, 3), 7.0, np.float32)
    assert mmr_ref(idx, val, F, 3, 0.5)[0].tolist() == [[0, 2, 1]]


def test_ref_zero_norm_rows_have_zero_cosine():
    # item 1 is a zero row: cos 0 to everything, so it beats item 2 (cos 1 to item 0) despite a lower score
    F = np.array([[1, 0], [0, 0], [3, 0]], np.float32)
    idx, val = np.array([[0, 2, 1]], np.int32), np.array([[3, 2, 1]], np.float32)
    # rel: 1, 0.5, 0; w = 0.6: item 2 -> 0.4 * 0.5 - 0.6 = -0.4, item 1 -> 0
    keys, scores = mmr_ref(idx, val, F, 3, 0.6)
    assert keys.tolist() == [[0, 1, 2]] and scores.tolist() == [[3, 1, 2]]


def test_ref_duplicates_are_ordinary_candidates():
    # rel 1, 1, 0; after item 0 its duplicate has cos 1 to it: 0.4 - 0.6 < 0 = item 1's 0 at w = 0.6, so it waits
    # (at w = 0.5 both are 0 and the tie goes to the duplicate's earlier position)
    F = np.array([[1, 0], [0, 1]], np.float32)
    idx, val = np.array([[0, 0, 1]], np.int32), np.array([[2, 2, 1]], np.float32)
    assert mmr_ref(idx, val, F, 3, 0.6)[0].tolist() == [[0, 1, 0]]
    assert mmr_ref(idx, val, F, 3, 0.5)[0].tolist() == [[0, 0, 1]]
    # w = 0 keeps the list order, duplicates included
    assert mmr_ref(idx, val, F, 3, 0.0)[0].tolist() == [[0, 0, 1]]


def test_ref_padding_and_empty_rows():
    F = np.eye(3, dtype=np.float32)
    idx = np.array([[2, -1, -1, -1], [-1, -1, -1, -1], [0, -1, 1, -1]], np.int32)
    val = np.array([[5, 0, 0, 0], [0, 0, 0, 0], [3, 0, 2, 0]], np.float32)
    keys, scores = mmr_ref(idx, val, F, 3, 0.3)
    assert keys.tolist() == [[2, -1, -1], [-1, -1, -1], [0, 1, -1]]
    assert scores.tolist() == [[5, 0, 0], [0, 0, 0], [3, 2, 0]]


# --- the NumPy path -------------------------------------------------------------------------------------------------

@pytest.mark.parametrize("w", [0.0, 0.3, 1.0])
@pytest.mark.parametrize("M,d", [(1, 4), (7, 3), (33, 20), (64, 9)])
def test_numpy_path_matches_reference(numpy_path, M, d, w):
    from buffalo_b200.parallel import rerank_mmr
    w = float(np.float32(w))
    idx, val, F = gap_inputs(3, M, d, w, seed=M + d)
    for k in sorted({1, min(10, M), M}):
        want = mmr_ref(idx, val, F, k, w)
        got = rerank_mmr(idx, val, F, k, w)
        np.testing.assert_array_equal(got[0], want[0])
        assert got[1].tobytes() == want[1].tobytes()
    idx, val, F = random_inputs(6, M, d, seed=M * d)
    keys, scores = rerank_mmr(idx, val, F, M, w)
    check_greedy(idx, val, F, w, keys, scores)


@pytest.mark.parametrize("kind", ["als", "bpr"])
def test_diversify_zero_is_the_plain_result(numpy_path, kind):
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    m = cpu_model(kind, U=40, I=120, d=8, use_bias=True)
    par = (ParALS if kind == "als" else ParBPRMF)(m)
    users = np.array([3, 0, 39, 12, 12], np.int32)
    seen = scipy.sparse.random(40, 120, density=0.2, format="csr", random_state=np.random.default_rng(2))
    rows = random_rows(40, 120, 4)
    rows[12] = list(rows[12][:3]) * 2                     # duplicates and a short row
    for kw in (dict(), dict(pool=["i%d" % i for i in range(0, 120, 3)]), dict(exclude_seen=seen),
               dict(pool=pool_matrix(rows, 40, 120)), dict(pool=pool_matrix(rows, 40, 120), exclude_seen=seen)):
        for k in (1, 5, 30):
            _, pk, ps = par.topk_recommendation(users, topk=k, **kw)
            _, dk, ds = par.topk_recommendation(users, topk=k, diversify=0, **kw)
            np.testing.assert_array_equal(dk, pk)
            assert ds.tobytes() == ps.tobytes()


def test_diversified_numpy_path_is_greedy(numpy_path):
    from buffalo_b200.parallel.base import ParBPRMF, dot_topn
    m = cpu_model("bpr", U=20, I=300, d=6, use_bias=True)
    users = np.arange(20, dtype=np.int32)
    _, keys, scores = ParBPRMF(m).topk_recommendation(users, topk=10, diversify=0.4, diversify_candidates=60)
    ck = np.zeros((20, 60), np.int32)
    cv = np.zeros((20, 60), np.float32)
    dot_topn(users, m.P, m.Q, m.Qb, ck, cv, None, 60)
    check_greedy(ck, cv, m.Q, float(np.float32(0.4)), keys, scores)
    # the bias goes into rel, not into the cosine: the picks are the reference's on the same candidates
    want = mmr_ref(ck, cv, m.Q, 10, float(np.float32(0.4)))
    np.testing.assert_array_equal(keys, want[0])


# --- argument checks --------------------------------------------------------------------------------------------------

BAD_DIVERSIFY = [True, False, -0.1, 1.5, float("nan"), "0.3", [0.3]]


@pytest.mark.parametrize("bad", BAD_DIVERSIFY)
def test_bad_diversify_before_device_work(no_device_work, bad):
    from buffalo_b200.parallel.base import ParALS
    par = ParALS(cpu_model("als"))
    with pytest.raises(ValueError, match="diversify"):
        par.topk_recommendation(np.arange(3, dtype=np.int32), topk=5, diversify=bad)


@pytest.mark.parametrize("topk,M", [(5, 4), (5, 257), (5, 0), (5, True), (5, 10.0), (300, None), (257, 257)])
def test_bad_candidates_before_device_work(no_device_work, topk, M):
    from buffalo_b200.parallel.base import ParALS
    par = ParALS(cpu_model("als"))
    with pytest.raises(ValueError, match="topk|diversify_candidates"):
        par.topk_recommendation(np.arange(3, dtype=np.int32), topk=topk, diversify=0.5, diversify_candidates=M)


def test_candidates_without_diversify(no_device_work):
    from buffalo_b200.parallel.base import ParALS
    with pytest.raises(ValueError, match="needs diversify"):
        ParALS(cpu_model("als")).topk_recommendation(np.arange(3, dtype=np.int32), topk=5, diversify_candidates=20)


def test_nprobe_refuses_diversify(no_device_work):
    from buffalo_b200.parallel.base import ParALS
    with pytest.raises(ValueError, match="nprobe does not take diversify"):
        ParALS(cpu_model("als")).topk_recommendation(np.arange(3, dtype=np.int32), topk=5, nprobe=2, diversify=0.3)


def test_default_candidates():
    from buffalo_b200.parallel.base import _check_diversify
    assert _check_diversify(None, None, 10) is None
    assert _check_diversify(0.3, None, 10) == (float(np.float32(0.3)), 40)
    assert _check_diversify(1, None, 100) == (1.0, 256)
    assert _check_diversify(np.float32(0), 7, 7) == (0.0, 7)


@pytest.mark.parametrize("bad", [0.5, True, 2.0, -1])
def test_fold_in_checks_diversify_first(no_device_work, monkeypatch, bad):
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als")

    def refuse(*a, **k):
        raise AssertionError("fold-in before the checks finished")
    m._fold_in_device = refuse
    kw = dict(diversify=bad) if bad != 0.5 else dict(diversify=0.5, diversify_candidates=3)
    with pytest.raises(ValueError, match="diversify"):
        ParALS(m).fold_in_recommendation([[1, 2]], topk=5, **kw)


def test_rerank_mmr_argument_checks(no_device_work):
    from buffalo_b200.parallel import rerank_mmr
    F = np.ones((10, 4), np.float32)
    idx, val = np.zeros((2, 5), np.int32), np.zeros((2, 5), np.float32)
    bad = [
        (dict(cand_idx=idx.astype(np.float32)), "integer"),
        (dict(cand_val=val[:, :4]), "same shape"),
        (dict(cand_idx=np.zeros(5, np.int32)), "integer"),
        (dict(item_factors=np.ones(10, np.float32)), "item_factors"),
        (dict(cand_idx=np.zeros((2, 257), np.int32), cand_val=np.zeros((2, 257), np.float32)), "at most 256"),
        (dict(topk=6), "topk"),
        (dict(topk=0), "topk"),
        (dict(diversify=1.2), "diversify"),
        (dict(diversify=None), "diversify"),
        (dict(cand_idx=idx - 2), "outside"),
        (dict(cand_idx=idx + 10), "outside"),
    ]
    for over, msg in bad:
        kw = dict(cand_idx=idx, cand_val=val, item_factors=F, topk=3, diversify=0.5)
        kw.update(over)
        with pytest.raises(ValueError, match=msg):
            rerank_mmr(**kw)

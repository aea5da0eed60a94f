"""ALS.posterior_sample and the explore option of ParALS where no GPU is needed: every input check raises before any
device work, models without a least-squares posterior are refused, explore needs the training data, without a GPU a
valid call raises the backend's "no CPU fallback" error, and the fp64 reference (tests/explore_ref.py) keeps its own
identities: its Philox words are tests/item_fold_in_ref.py's, its normals pass a moment test and its draws have the
covariance scale^2 A^-1."""
import numpy as np
import pytest
import scipy.sparse

from tests import explore_ref
from tests.test_explain_cpu import _Data, no_device_work  # noqa: F401
from tests.test_fold_in_cpu import cpu_model, history


def test_posterior_sample_checks_before_device_work(no_device_work):  # noqa: F811
    m = cpu_model("als")
    I, d = m.Q.shape[0], m.opt.d
    H = history(4, I)
    mean = np.zeros((4, d), np.float32)
    for scale in (-1.0, float("nan"), float("inf"), 1e39, "1", True, None, [1.0]):
        with pytest.raises(ValueError, match="scale"):
            m.posterior_sample(H, mean, scale=scale)
    for seed in (-1, 2 ** 32, 1.5, True, "0", None):
        with pytest.raises(ValueError, match="seed"):
            m.posterior_sample(H, mean, seed=seed)
    for bad in (np.zeros((3, d)), np.zeros((4, d + 1)), np.zeros(4 * d), np.zeros((4, d), dtype=bool),
                [["a"] * d] * 4):
        with pytest.raises(ValueError, match="mean"):
            m.posterior_sample(H, bad)
    for keys in ([0, 1, 2], [0, 1, 2, 2], [0, -1, 2, 3], np.array([0.0, 1.0, 2.0, 3.0]), np.zeros((4, 1), np.int64),
                 np.array([0, 1, 2, 2 ** 63], dtype=np.uint64)):
        with pytest.raises(ValueError, match="draw_keys"):
            m.posterior_sample(H, mean, draw_keys=keys)
    with pytest.raises(ValueError, match="matrix"):
        m.posterior_sample(history(4, I + 1), mean)
    with pytest.raises(ValueError, match="histories"):
        m.posterior_sample(np.zeros((4, I)), mean)
    wide = cpu_model("als", d=257)
    with pytest.raises(ValueError, match="d <= 256"):
        wide.posterior_sample(H, np.zeros((4, 257), np.float32))
    with pytest.raises(RuntimeError, match="normalized"):
        cpu_model("als", _nrz_Q=True).posterior_sample(H, mean)


def test_par_explore_checks_before_device_work(no_device_work):  # noqa: F811
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als", U=30)
    par = ParALS(m)
    with pytest.raises(ValueError, match="training data"):
        par.topk_recommendation(["u1", "u2"], explore=0.5)
    m.data = _Data(30, m.Q.shape[0])
    for bad in (-0.1, float("nan"), float("inf"), "1", True):
        with pytest.raises(ValueError, match="explore"):
            par.topk_recommendation(["u1"], explore=bad)
        with pytest.raises(ValueError, match="explore"):
            par.fold_in_recommendation(history(2, m.Q.shape[0]), explore=bad)
    for seed in (-1, 2 ** 32, 0.5, False, None):
        with pytest.raises(ValueError, match="explore_seed"):
            par.topk_recommendation(["u1"], explore=1.0, explore_seed=seed)
        with pytest.raises(ValueError, match="explore_seed"):
            par.fold_in_recommendation(history(2, m.Q.shape[0]), explore=1.0, explore_seed=seed)
    with pytest.raises(ValueError, match="d <= 256"):
        wide = cpu_model("als", d=257)
        ParALS(wide).fold_in_recommendation(history(2, wide.Q.shape[0]), explore=1.0)
    # the checks of the modes it joins still come first
    with pytest.raises(ValueError, match="pool"):
        par.topk_recommendation(["u1"], pool=scipy.sparse.csr_matrix((3, 3)), explore=1.0)
    with pytest.raises(ValueError, match="nprobe"):
        par.topk_recommendation(["u1"], nprobe=1, exclude_seen=True, explore=1.0)


@pytest.mark.parametrize("kind", ["bpr", "warp", "plsi"])
def test_models_without_posterior_refused(kind, no_device_work):  # noqa: F811
    from buffalo_b200.algo.bpr import BPRMF
    from buffalo_b200.algo.warp import WARP
    from buffalo_b200.misc import aux
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    if kind == "plsi":
        par = ParALS(cpu_model("plsi"))
    else:
        cls = BPRMF if kind == "bpr" else WARP
        m = cls.__new__(cls)
        m.opt = aux.Option(num_workers=1, use_bias=True)
        par = ParBPRMF(m)
    with pytest.raises(NotImplementedError, match=r"explore needs a least-squares model \(ALS\)"):
        par.topk_recommendation(["u1"], explore=1.0)
    if kind == "plsi":      # BPRMF / WARP have no fold-in, which fold_in_recommendation refuses first
        with pytest.raises(NotImplementedError, match=r"explore needs a least-squares model \(ALS\)"):
            par.fold_in_recommendation([["i1"]], explore=0.0)
    else:
        with pytest.raises(NotImplementedError, match="needs a model with fold_in"):
            par.fold_in_recommendation([["i1"]], explore=0.0)


def test_training_rows_gather_only_the_requested_users():
    """ParALS._training_rows(idx) equals the rows idx (in that order, repeats kept) of the whole training CSR"""
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als", U=30)
    m.data = _Data(30, m.Q.shape[0])
    g = m.data.get_group("rowwise")
    full = scipy.sparse.csr_matrix((g["val"], g["key"], np.concatenate([[0], g["indptr"]])), shape=(30, m.Q.shape[0]))
    for idx in ([3, 0, 29, 3], [], [7]):
        got = ParALS(m)._training_rows(np.array(idx, dtype=np.int64), "explore")
        want = full[np.array(idx, dtype=np.int64)]
        assert got.shape == want.shape
        assert np.array_equal(got.indptr, want.indptr) and np.array_equal(got.indices, want.indices)
        assert np.array_equal(got.data, want.data)


def test_no_cpu_fallback():
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from buffalo_b200 import _cabi
    from buffalo_b200.parallel.base import ParALS
    m = cpu_model("als", U=30)
    with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
        m.posterior_sample(history(3, m.Q.shape[0]), np.zeros((3, m.opt.d)))
    m.data = _Data(30, m.Q.shape[0])
    par = ParALS(m)
    plain = par.topk_recommendation(["u1", "u2"], topk=5)       # explore=None: the NumPy path, unchanged
    assert len(plain[1]) == 2
    for explore in (0.0, 0.5):
        with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
            par.topk_recommendation(["u1", "u2"], topk=5, explore=explore)


def test_reference_words_are_item_fold_in_philox():
    for seed, key, D in ((0, 0, 9), (7, 12345, 16), (2 ** 32 - 1, 2 ** 40 + 3, 5), (99, 2 ** 63 - 1, 12)):
        assert np.array_equal(explore_ref.words(seed, [key], D)[0], explore_ref.words_scalar(seed, key, D))


def test_reference_normals_moments():
    """10^5 normals (12500 keys x d = 8): mean, variance, third and fourth moments, and the cos / sin pairs
    uncorrelated, each within 4 standard errors"""
    Z = explore_ref.normals(3, np.arange(12500), 8)
    z = Z.ravel()
    N = z.size
    assert N == 10 ** 5
    assert abs(z.mean()) < 4 / np.sqrt(N)
    assert abs(z.var() - 1) < 4 * np.sqrt(2 / N)
    assert abs((z ** 3).mean()) < 4 * np.sqrt(15 / N)
    assert abs((z ** 4).mean() - 3) < 4 * np.sqrt(96 / N)
    pair = (Z[:, 0::2] * Z[:, 1::2]).ravel()
    assert abs(pair.mean()) < 4 / np.sqrt(pair.size)
    # odd widths drop the last sine: the first d columns of the next even width
    assert np.array_equal(explore_ref.normals(3, [5, 6], 7), explore_ref.normals(3, [5, 6], 8)[:, :7])


@pytest.mark.parametrize("adaptive_reg", [False, True])
def test_reference_covariance(adaptive_reg):
    """20000 draws of one history: empirical covariance of out - mean within 0.05 (relative Frobenius) of
    scale^2 A^-1, and the failure rule for a singular A"""
    rng = np.random.default_rng(5)
    I, d, n = 40, 4, 20000
    Q = rng.normal(scale=0.3, size=(I, d)).astype(np.float32)
    row = np.sort(rng.integers(0, I, 6)).astype(np.int32)
    indptr = np.arange(1, n + 1, dtype=np.int64) * len(row)
    keys, vals = np.tile(row, n), np.tile(rng.random(len(row)).astype(np.float32) * 3, n)
    mean = np.tile(rng.normal(size=d), (n, 1))
    scale = 0.7
    out, Y, failed = explore_ref.sample_rows(Q, indptr, keys, vals, mean, np.arange(n), 11, scale, 2.0, 0.3,
                                             adaptive_reg)
    assert not failed.any()
    G = Q.astype(np.float64).T @ Q.astype(np.float64)
    A = explore_ref.row_matrix(G, Q, row, vals[:len(row)], 2.0, 0.3, adaptive_reg)
    want = scale ** 2 * np.linalg.inv(A)
    C = np.cov((out - mean).T)
    assert np.linalg.norm(C - want) <= 0.05 * np.linalg.norm(want)
    # an empty row with adaptive_reg and fewer items than d: A = Q'Q is singular (exactly, for these items), the row
    # stays at its mean
    Qs = np.array([[1, 1, 0, 0], [0, 0, 1, 1]], np.float32)
    out, Y, failed = explore_ref.sample_rows(Qs, np.array([0], np.int64), np.zeros(0, np.int32),
                                             np.zeros(0, np.float32), mean[:1], [0], 1, 1.0, 2.0, 0.3, True)
    assert failed.tolist() == [True] and np.array_equal(out, mean[:1])

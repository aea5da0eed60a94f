"""pLSI checks that need no GPU: option defaults, the float32 oracle against the fp64 mirror, a d = 2 case worked by
hand, the EM guarantee, and the package surface."""
import numpy as np
import pytest

from tests.helpers import make_csr, rel_err
from tests.plsi_ref import OraclePLSI, oracle_iteration, plsi_iteration, random_factors


def test_option_defaults_equal_reference():
    from buffalo_b200.algo.options import PLSIOption
    opt = PLSIOption().get_default_option()
    ref = dict(d=20, num_iters=10, num_workers=1, alpha1=1.0, alpha2=1.0, eps=1e-10, model_path="", save_factors=False,
               data_opt={}, inherit_opt={})                                # buffalo/algo/options.py:372-384
    for k, v in ref.items():
        assert opt[k] == v, (k, opt[k], v)
    assert PLSIOption().is_valid_option(opt)


@pytest.mark.parametrize("vals", ["ints", "lognormal"])
def test_oracle_matches_fp64_mirror_over_three_iterations(vals):
    U, I, d = 300, 200, 7
    indptr, keys, v, _ = make_csr(U, I, 4000, seed=3, empty_rows=20)
    if vals == "lognormal":
        v = np.random.default_rng(4).lognormal(0.0, 1.0, len(v)).astype(np.float32)
    P, Q = random_factors(U, d, 1, axis=1), random_factors(I, d, 2, axis=0)
    Po, Qo, Pm, Qm = P, Q, P.astype(np.float64), Q.astype(np.float64)
    for _ in range(3):
        Po, Qo, lo = oracle_iteration(Po, Qo, indptr, keys, v)
        Pm, Qm, lm = plsi_iteration(Pm, Qm, indptr, keys, v)
        assert abs(lo - lm) <= 1e-5 * abs(lm), (lo, lm)
    assert rel_err(Po, Pm) <= 1e-5 and rel_err(Qo, Qm) <= 1e-5, (rel_err(Po, Pm), rel_err(Qo, Qm))


def test_hand_checked_d2():
    """One user, two items, values 1 and 2.  Both entries have norm 0.5, so loss = 3 ln 2; the accumulators are
    P = [1.75, 1.25] and Q = [[0.25, 0.75], [1.5, 0.5]]."""
    P = np.array([[0.5, 0.5]], np.float32)
    Q = np.array([[0.25, 0.75], [0.75, 0.25]], np.float32)
    indptr, keys, vals = np.array([2], np.int64), np.array([0, 1], np.int32), np.array([1.0, 2.0], np.float32)
    for fn in (oracle_iteration, plsi_iteration):
        P1, Q1, loss = fn(P, Q, indptr, keys, vals, alpha1=0.0, alpha2=0.0)
        assert loss == pytest.approx(3 * np.log(2.0), rel=1e-6)
        np.testing.assert_allclose(P1, [[7 / 12, 5 / 12]], rtol=1e-6)
        np.testing.assert_allclose(Q1, [[1 / 7, 0.6], [6 / 7, 0.4]], rtol=1e-6)
        # alpha1 / d = alpha2 / num_items = 0.5 is added before the sums (plsi.cc:112-124)
        P1, Q1, _ = fn(P, Q, indptr, keys, vals, alpha1=1.0, alpha2=1.0)
        np.testing.assert_allclose(P1, [[2.25 / 4, 1.75 / 4]], rtol=1e-6)
        np.testing.assert_allclose(Q1, [[0.75 / 2.75, 1.25 / 2.25], [2.0 / 2.75, 1.0 / 2.25]], rtol=1e-6)


def test_empty_row_without_alpha1_is_nan_like_the_reference():
    P, Q = random_factors(3, 4, 1, axis=1), random_factors(5, 4, 2, axis=0)
    indptr, keys, vals = np.array([2, 2, 3], np.int64), np.array([0, 4, 1], np.int32), np.ones(3, np.float32)
    P1, _, _ = oracle_iteration(P, Q, indptr, keys, vals, alpha1=0.0, alpha2=1.0)
    assert np.isnan(P1[1]).all() and np.isfinite(P1[[0, 2]]).all()


def test_loss_never_increases_without_smoothing():
    """EM: with alpha1 = alpha2 = 0 each iteration maximises the expected log-likelihood, so -sum v log(p) cannot
    grow."""
    U, I, d = 400, 300, 8
    indptr, keys, vals, _ = make_csr(U, I, 6000, seed=9)
    P, Q = random_factors(U, d, 5, axis=1), random_factors(I, d, 6, axis=0)
    losses = []
    for _ in range(10):
        P, Q, loss = plsi_iteration(P, Q, indptr, keys, vals, alpha1=0.0, alpha2=0.0)
        losses.append(loss)
    # the loss of iteration k is measured at the factors before it, so the sequence is non-increasing
    assert all(b <= a * (1 + 1e-12) for a, b in zip(losses, losses[1:])), losses
    assert losses[-1] < losses[0]


def test_oracle_chunks_equal_one_call():
    U, I, d = 200, 150, 5
    indptr, keys, vals, _ = make_csr(U, I, 3000, seed=11, empty_rows=10)
    P, Q = random_factors(U, d, 1, axis=1), random_factors(I, d, 2, axis=0)
    whole = oracle_iteration(P, Q, indptr, keys, vals)
    o = OraclePLSI()
    o.init(dict(d=d))
    P1, Q1 = P.copy(), Q.copy()
    o.initialize_model(P1, Q1)
    o.reset()
    loss = 0.0
    for a, b in ((0, 37), (37, 38), (38, 150), (150, U)):
        beg = 0 if a == 0 else int(indptr[a - 1])
        end = int(indptr[b - 1])
        loss += o.partial_update(a, b, indptr, keys[beg:end], vals[beg:end])
    o.normalize(1.0, 1.0)
    o.swap()
    assert rel_err(P1, whole[0]) < 1e-6 and rel_err(Q1, whole[1]) < 1e-6 and loss == pytest.approx(whole[2], rel=1e-6)


def test_package_surface_plsi():
    import buffalo
    from buffalo import PLSI, PLSIOption  # noqa: F401
    from buffalo.algo import PLSI as _P, PLSIOption as _O  # noqa: F401
    from buffalo.algo.plsi import PLSI as _Q  # noqa: F401
    import buffalo_b200
    assert buffalo.PLSI is buffalo_b200.PLSI is _P is _Q
    assert buffalo.PLSIOption().get_default_option().d == 20
    for name in ("W2V", "CFR", "EALS"):
        with pytest.raises(NotImplementedError):
            getattr(buffalo, name)()

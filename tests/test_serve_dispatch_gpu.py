"""Which backend.Serve entry points each ParALS serving mode calls (DESIGN.md 4.9): the recorded sequence of top-k,
rerank, category-walk and query-binding calls of topk_recommendation, most_similar and fold_in_recommendation in every
mode.  The results of these calls are checked by the serve, rerank, category, explore and fold-in tests; this file pins
the native path, which is what decides each mode's speed."""
import numpy as np
import pytest
import scipy.sparse

pytestmark = pytest.mark.gpu

RECORDED = ("topk", "topk_seen", "topk_candidates", "topk_device", "topk_seen_device", "topk_candidates_device",
            "rerank_mmr_device", "bind_queries", "unbind_queries")


@pytest.fixture
def calls(cuda_lib, monkeypatch):
    """The list every recorded call appends its name to, "+seen" marking candidate calls given seen rows."""
    from buffalo_b200 import backend
    log = []

    def recorder(name, fn):
        def call(*a, **k):
            log.append(name + ("+seen" if k.get("seen") is not None else ""))
            return fn(*a, **k)
        return call
    for name in RECORDED:
        monkeypatch.setattr(backend.Serve, name, recorder(name, getattr(backend.Serve, name)))
    monkeypatch.setattr(backend, "category_walk_device", recorder("category_walk_device", backend.category_walk_device))
    return log


@pytest.fixture
def model():
    """A trained ALS model with its training data; one per test, since most_similar normalises the item factors."""
    from tests.test_explore_gpu import trained
    return trained()


def capped(stage, deeper):
    """The calls of a capped walk: the stage, the walk, then (deeper stage, walk) rounds; the categories below make
    every row need at least one deeper round."""
    def match(log):
        return (len(log) >= 4 and len(log) % 2 == 0 and log[0] == stage and log[2::2] == [deeper] * (len(log) // 2 - 1)
                and log[1::2] == ["category_walk_device"] * (len(log) // 2))
    return match


def modes(rng, U, I, device_seen=False):
    """(name, keyword arguments, expected calls): the plain, diversified and capped modes over no pool, a shared pool
    and a per-user pool, with and without seen rows.  Expected calls are a list, or a predicate for capped walks.
    device_seen: the seen rows are already on the device (fold-in's histories), so plain calls take the stage too."""
    pool = rng.choice(I, 300, replace=False).astype(np.int32)
    per_user = scipy.sparse.random(U, I, density=0.1, format="csr", random_state=rng)
    cats = dict(categories=(np.arange(I) % 32 != 0).astype(np.int32), category_cap=np.array([100, 0], np.int32))
    out = []
    for pname, pkw in [("none", {}), ("list", dict(pool=pool)), ("sparse", dict(pool=per_user))]:
        for seen in (False, True):
            sparse = pname == "sparse"
            plain = ("topk_candidates+seen" if seen else "topk_candidates") if sparse else \
                "topk_seen" if seen else "topk"
            stage = ("topk_candidates_device+seen" if seen else "topk_candidates_device") if sparse else \
                "topk_seen_device" if seen else "topk_device"
            deeper = "topk_candidates_device+seen" if sparse else "topk_seen_device"
            kw = dict(pkw, exclude_seen=seen)
            tag = "%s-%s" % (pname, "seen" if seen else "all")
            out.append((tag, kw, [stage if seen and device_seen else plain]))
            out.append((tag + "-diversify", dict(kw, diversify=0.4), [stage, "rerank_mmr_device"]))
            out.append((tag + "-categories", dict(kw, **cats), capped(stage, deeper)))
    return out


def matches(log, expected):
    return expected(log) if callable(expected) else log == expected


def bound(expected):
    """expected between bind_queries and unbind_queries: a call on device query rows."""
    return lambda log: log[:1] == ["bind_queries"] and log[-1:] == ["unbind_queries"] and matches(log[1:-1], expected)


def check(bad, log, expected, what):
    """Adds (what, log) to bad unless log is the expected call sequence."""
    if not matches(log, expected):
        bad.append((what, list(log)))


def test_topk_recommendation_calls(model, calls):
    from buffalo_b200.parallel.base import ParALS
    m, rng, _ = model
    U, I = m.P.shape[0], m.Q.shape[0]
    par = ParALS(m)
    users = rng.choice(U, 50, replace=False).astype(np.int32)
    bad = []
    for tag, kw, expected in modes(rng, U, I):
        del calls[:]
        par.topk_recommendation(users, 10, **kw)
        check(bad, calls, expected, tag)
        del calls[:]
        par.topk_recommendation(users, 10, explore=0.5, explore_seed=7, **kw)
        check(bad, calls, bound(expected), tag + "-explore")
    assert not bad, bad


def test_most_similar_calls(model, calls):
    from buffalo_b200.parallel.base import ParALS
    m, rng, _ = model
    I = m.Q.shape[0]
    par = ParALS(m)
    items = rng.choice(I, 40, replace=False).astype(np.int32)
    pool = rng.choice(I, 300, replace=False).astype(np.int32)
    cats = (np.arange(I) % 32 != 0).astype(np.int32)
    bad = []
    for kw in (dict(), dict(pool=pool)):
        del calls[:]
        par.most_similar(items, 10, **kw)
        check(bad, calls, ["topk"], sorted(kw))
        del calls[:]
        par.most_similar(items, 10, categories=cats, category_cap=np.array([100, 0], np.int32), **kw)
        check(bad, calls, capped("topk_device", "topk_seen_device"), sorted(kw) + ["categories"])
    assert not bad, bad


def test_fold_in_recommendation_calls(model, calls):
    from buffalo_b200.parallel.base import ParALS
    from tests.helpers import csr_from_lengths
    from tests.test_explain_gpu import to_matrix
    m, rng, _ = model
    I = m.Q.shape[0]
    par = ParALS(m)
    hi, hk, hv = csr_from_lengths(rng.integers(0, 40, 70), I, rng)
    H = to_matrix(hi, hk, hv, I)
    bad = []
    for tag, kw, expected in modes(rng, H.shape[0], I, device_seen=True):
        for ekw in (dict(), dict(explore=0.5, explore_seed=7)):
            del calls[:]
            par.fold_in_recommendation(H, 10, **dict(kw, **ekw))
            check(bad, calls, bound(expected), tag + ("-explore" if ekw else ""))
    assert not bad, bad

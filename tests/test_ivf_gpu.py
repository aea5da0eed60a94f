"""IVF index on the GPU (csrc/ivf.cu, backend.IVF, ParALS.build_index / nprobe): nprobe = nlist is the exact serve
path bit for bit, nprobe < nlist is the exact top-k of the probed lists' rows, the build is deterministic and
consistent with its own assignment, recall on a clustered fixture, and destroy returns the device memory."""
import numpy as np
import pytest

from tests.ivf_ref import gaussian_mixture, update_fp64

pytestmark = pytest.mark.gpu


def exact(items, bias, queries, k, pool=None):
    from buffalo_b200 import backend
    s = backend.Serve()
    s.set_items(items, bias)
    s.set_queries(queries)
    s.set_pool(pool)
    out = s.topk(np.arange(queries.shape[0], dtype=np.int32), k)
    s.close()
    return out


def index(items, bias=None, nlist=16, iters=5, seed=3):
    from buffalo_b200 import backend
    ivf = backend.IVF()
    ivf.build(items, bias, nlist, iters, seed)
    return ivf


def assert_same(got, want):
    (gi, gv), (wi, wv) = got, want
    assert gi.shape == wi.shape
    np.testing.assert_array_equal(gi, wi)
    np.testing.assert_array_equal(gv.view(np.uint32), wv.view(np.uint32))


def rows(n, d, seed):
    return np.random.default_rng(seed).standard_normal((n, d)).astype(np.float32)


@pytest.mark.parametrize("d", [20, 128, 256])
@pytest.mark.parametrize("k", [1, 10, 100])
@pytest.mark.parametrize("with_bias", [False, True])
def test_full_probe_is_exact(d, k, with_bias):
    items, queries = rows(3001, d, 1), rows(300, d, 2)             # 3001 rows: nlist = 16 does not divide it
    bias = np.random.default_rng(3).standard_normal(3001).astype(np.float32) if with_bias else None
    ivf = index(items, bias, nlist=16)
    assert_same(ivf.search(queries, 16, k, use_bias=with_bias), exact(items, bias, queries, k))


def test_long_list_empty_list_duplicates_and_padding():
    # 5000 copies of one row -> one list of more than 4096 rows; 40 distinct other rows repeated -> duplicated rows
    # whose ties go to the smaller id; 64 lists over 41 distinct rows -> empty lists
    rng = np.random.default_rng(4)
    d = 32
    cone = np.tile(rng.standard_normal(d).astype(np.float32), (5000, 1))
    distinct = rng.standard_normal((40, d)).astype(np.float32)
    dup = distinct[rng.integers(0, 40, 2000)]
    items = np.ascontiguousarray(np.concatenate([cone, dup])[rng.permutation(7000)])
    ivf = index(items, None, nlist=64)
    lens = np.diff(ivf.offsets(), prepend=0)
    assert lens.max() > 4096 and (lens == 0).any()
    queries = rows(100, d, 5)
    for k in (1, 10, 100):
        assert_same(ivf.search(queries, 64, k), exact(items, None, queries, k))
    small = rows(50, d, 6)
    ivf_small = index(small, None, nlist=7)
    got = ivf_small.search(queries, 7, 100)
    assert (got[0][:, 50:] == -1).all() and (got[1][:, 50:] == 0).all()
    assert_same(got, exact(small, None, queries, 100))


@pytest.mark.parametrize("batch", [0, 7, 32, 33])
def test_batch_edges(batch):
    items, queries = rows(2000, 64, 7), rows(101, 64, 8)
    ivf = index(items, None, nlist=12)
    ivf._set_batch_rows(batch)
    for nprobe in (12, 3):
        got = ivf.search(queries, nprobe, 10)
        ivf._set_batch_rows(0)
        assert_same(got, ivf.search(queries, nprobe, 10))
        ivf._set_batch_rows(batch)
    assert_same(ivf.search(queries, 12, 10), exact(items, None, queries, 10))


@pytest.mark.parametrize("with_bias", [False, True])
def test_partial_probe_is_exact_over_probed_rows(with_bias):
    items, queries = gaussian_mixture(6000, 48, 40, seed=9), rows(50, 48, 10)
    bias = np.random.default_rng(11).standard_normal(6000).astype(np.float32) if with_bias else None
    nlist, nprobe, k = 32, 5, 20
    ivf = index(items, bias, nlist=nlist)
    got_i, got_v = ivf.search(queries, nprobe, k, use_bias=with_bias)
    cent, offs, ids = ivf.centroids(), ivf.offsets(), ivf.ids()
    probed, _ = exact(np.ascontiguousarray(cent), None, queries, nprobe)
    for q in range(queries.shape[0]):
        pool = np.sort(np.concatenate([ids[(offs[l - 1] if l else 0):offs[l]] for l in probed[q]])).astype(np.int32)
        want = exact(items, bias, queries[q:q + 1], k, pool)
        assert_same((got_i[q:q + 1], got_v[q:q + 1]), want)


def test_build_deterministic_and_consistent():
    items = gaussian_mixture(5000, 24, 30, seed=12)
    a, b = index(items, None, nlist=20, iters=4), index(items, None, nlist=20, iters=4)
    for f in ("centroids", "offsets", "ids"):
        np.testing.assert_array_equal(getattr(a, f)().view(np.uint8), getattr(b, f)().view(np.uint8))
    offs, ids = a.offsets(), a.ids()
    assert offs[-1] == 5000 and np.array_equal(np.sort(ids), np.arange(5000))
    starts = np.concatenate([[0], offs[:-1]])
    lists = np.repeat(np.arange(20), offs - starts)
    for s, e in zip(starts, offs):
        assert (np.diff(ids[s:e]) > 0).all()
    # each row's list is its top-1 against the final centroids
    top1, _ = exact(np.ascontiguousarray(a.centroids()), None, items, 1)
    assign = np.empty(5000, np.int64)
    assign[ids] = lists
    np.testing.assert_array_equal(top1[:, 0], assign)


def test_update_step_against_fp64():
    """The centroids after iters + 1 rounds are one update of the iters-round centroids, from the assignment to them
    (the iters-round index's lists)."""
    items = gaussian_mixture(4000, 40, 25, seed=13)
    nlist = 24
    one, two = index(items, None, nlist=nlist, iters=1), index(items, None, nlist=nlist, iters=2)
    offs, ids = one.offsets(), one.ids()
    assign = np.empty(4000, np.int64)
    assign[ids] = np.repeat(np.arange(nlist), np.diff(offs, prepend=0))
    want = update_fp64(items, assign, one.centroids(), nlist)
    got = two.centroids().astype(np.float64)
    assert np.abs(got - want).max() <= 1e-5 * np.abs(want).max()


def test_recall_clustered():
    """recall@10 against the exact path at nprobe = nlist / 16 on a seeded Gaussian mixture."""
    items = gaussian_mixture(50000, 64, 256, seed=14)
    queries = gaussian_mixture(2000, 64, 256, seed=15)
    nlist = 256
    ivf = index(items, None, nlist=nlist, iters=10)
    got, _ = ivf.search(queries, nlist // 16, 10)
    want, _ = exact(items, None, queries, 10)
    recall = np.mean([len(np.intersect1d(g, w)) / 10.0 for g, w in zip(got, want)])
    print("recall@10 at nprobe = nlist / 16: %.4f" % recall)
    assert recall >= 0.99                                              # 1.0000 measured on an H100 80GB HBM3, 700 W


def test_destroy_returns_memory():
    import torch
    items, queries = rows(20000, 128, 16), rows(1000, 128, 17)
    warm = index(items, None, nlist=64)
    warm.search(queries, 8, 10)
    warm.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    free0 = torch.cuda.mem_get_info()[0]
    ivf = index(items, None, nlist=64)
    ivf.search(queries, 8, 10)
    ivf.close()
    torch.cuda.synchronize()
    torch.cuda.empty_cache()
    assert torch.cuda.mem_get_info()[0] >= free0 - (4 << 20)


def _model(kind, U=400, I=3000, d=32):
    from tests.test_ivf_cpu import cpu_model
    m = cpu_model(kind, U=U, I=I, d=d, use_bias=True)
    rng = np.random.default_rng(18)
    m.P = rng.standard_normal((U, d)).astype(np.float32)
    m.Q = rng.standard_normal((I, d)).astype(np.float32)
    return m


@pytest.mark.parametrize("kind", ["als", "bpr"])
def test_par_full_probe_matches_exact(kind):
    from buffalo_b200.parallel.base import ParALS, ParBPRMF
    par = (ParALS if kind == "als" else ParBPRMF)(_model(kind))
    par.build_index(24)
    users = np.arange(0, 400, 3, dtype=np.int32)
    kept, t0, s0 = par.topk_recommendation(users, topk=15)
    _, t1, s1 = par.topk_recommendation(users, topk=15, nprobe=24)
    assert_same((t1, s1), (t0, s0))
    # most_similar normalises the items: the index on the raw factors is stale until built again
    with pytest.raises(RuntimeError, match="stale"):
        par.most_similar(np.arange(10, dtype=np.int32), topk=7, nprobe=24)
    par.build_index(24)
    items = np.arange(10, dtype=np.int32)
    assert_same(par.most_similar(items, topk=7, nprobe=24), par.most_similar(items, topk=7))
    ids = ["i%d" % i for i in range(10)]
    assert par.most_similar(ids, topk=7, nprobe=24, repr=True)[0] == par.most_similar(ids, topk=7, repr=True)[0]

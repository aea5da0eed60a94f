"""Batch serving on the device (csrc/serve.cu, backend.Serve, buffalo.parallel ParALS / ParBPRMF): keys and scores are
bitwise those of bfl_topk_device on the gathered rows, the ranking is the exact fp64 one outside rounding ties, and
pools, batching, aliasing, the device-pointer path and the handle's memory behave as include/buffalo_b200.h says."""
import os
import threading

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def factors(n, I, ld, d, seed, bias):
    rng = np.random.default_rng(seed)
    P = np.zeros((n, ld), np.float32)
    Q = np.zeros((I, ld), np.float32)
    P[:, :d] = rng.normal(size=(n, d))
    Q[:, :d] = rng.normal(size=(I, d))
    Qb = rng.normal(size=I).astype(np.float32) if bias else None
    return P, Q, Qb


def make(P, Q, Qb, d=None):
    from buffalo_b200 import backend
    h = backend.Serve()
    h.set_items(Q, Qb, d=d)
    h.set_queries(P)
    return h


def reference(P, Q, Qb, qidx, k, pool=None):
    """bfl_topk_device on the gathered rows (same pitches), padded to k with -1 / 0.0 like the handle."""
    import torch
    from buffalo_b200 import backend
    cand = Q if pool is None else Q[pool]
    cb = None if Qb is None else torch.from_numpy(np.ascontiguousarray(Qb if pool is None else Qb[pool])).cuda()
    idx, val = backend.topk_device(torch.from_numpy(P[qidx]).cuda(), torch.from_numpy(cand).cuda(), cb, k)
    torch.cuda.synchronize()
    idx, val = idx.cpu().numpy(), val.cpu().numpy()
    keys = np.full((len(qidx), k), -1, np.int32)
    vals = np.zeros((len(qidx), k), np.float32)
    keys[:, :idx.shape[1]] = idx if pool is None else np.asarray(pool, np.int32)[idx]
    vals[:, :idx.shape[1]] = val
    return keys, vals


def bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("d", [1, 5, 20, 100, 128, 256, 300])
def test_bitwise_equal_to_topk_device(cuda_lib, d, bias):
    # 5003 items: five slices, the last one short and not a whole tile; 70 queries: two CTAs, the last one short
    P, Q, Qb = factors(90, 5003, d, d, 100 + d, bias)
    h = make(P, Q, Qb)
    qidx = np.random.default_rng(d).permutation(90)[:70].astype(np.int32)
    for k in (1, 10, 100, 4096):
        keys, vals = h.topk(qidx, k)
        rk, rv = reference(P, Q, Qb, qidx, k)
        assert np.array_equal(keys, rk), (d, k)
        assert np.array_equal(bits(vals), bits(rv)), (d, k)
    h.close()


def test_bitwise_with_padded_rows(cuda_lib):
    """d = 20 inside rows of pitch 24 and d = 6 inside rows of pitch 7: the pitch decides the accumulation order."""
    import torch
    from buffalo_b200 import backend
    for ld, d in ((24, 20), (7, 6)):
        P, Q, Qb = factors(40, 3001, ld, d, 7, True)
        h = make(P, Q, Qb, d=d)
        qidx = np.arange(40, dtype=np.int32)
        keys, vals = h.topk(qidx, 33)
        Pd, Qd = torch.from_numpy(P).cuda(), torch.from_numpy(Q).cuda()
        idx = torch.empty((40, 33), dtype=torch.int32, device="cuda")
        val = torch.empty((40, 33), dtype=torch.float32, device="cuda")
        assert cuda_lib.bfl_topk_device(Pd.data_ptr(), 40, ld, Qd.data_ptr(), 3001, ld, torch.from_numpy(Qb).cuda().data_ptr(),
                                        d, 33, idx.data_ptr(), val.data_ptr(), backend._stream_ptr(None)) == 0
        torch.cuda.synchronize()
        assert np.array_equal(keys, idx.cpu().numpy()) and np.array_equal(bits(vals), bits(val.cpu().numpy()))
        h.close()


@pytest.mark.parametrize("d,k", [(20, 10), (128, 100), (5, 7)])
def test_exact_ranking_against_fp64(cuda_lib, d, k):
    P, Q, Qb = factors(50, 7001, d, d, 11, True)
    h = make(P, Q, Qb)
    keys, vals = h.topk(np.arange(50, dtype=np.int32), k)
    s = P.astype(np.float64) @ Q.astype(np.float64).T + Qb.astype(np.float64)[None, :]
    order = np.argsort(-s, axis=1, kind="stable")
    # fp32 rounding bound of a d-term dot product plus the bias add
    bound = (d + 2) * 2.0 ** -24 * (np.abs(P).astype(np.float64) @ np.abs(Q).astype(np.float64).T + np.abs(Qb)[None, :])
    checked = 0
    for r in range(50):
        kth, nxt = order[r, k - 1], order[r, k]
        assert np.allclose(vals[r], s[r, keys[r]], rtol=0, atol=2 * bound[r].max())
        assert (np.diff(vals[r]) <= 0).all()
        if s[r, kth] - s[r, nxt] > bound[r, kth] + bound[r, nxt]:
            assert set(keys[r].tolist()) == set(order[r, :k].tolist())
            checked += 1
    assert checked > 40
    h.close()


def test_exact_ties_come_back_in_ascending_id(cuda_lib):
    rng = np.random.default_rng(2)
    P, Q, _ = factors(9, 4000, 16, 16, 5, False)
    best = rng.normal(size=16).astype(np.float32) * 4       # one row planted at scattered ids in different slices
    ids = np.array([3999, 17, 1024, 1023, 2500, 3, 2048], dtype=np.int64)
    Q[ids] = best
    P[:] = best
    h = make(P, Q, None)
    keys, vals = h.topk(np.arange(9, dtype=np.int32), 5)
    assert (keys == np.sort(ids)[:5][None, :]).all()
    assert (bits(vals) == bits(vals)[0, 0]).all()
    h.close()


def test_pool(cuda_lib):
    P, Q, Qb = factors(45, 6000, 20, 20, 21, True)
    h = make(P, Q, Qb)
    qidx = np.arange(45, dtype=np.int32)
    rng = np.random.default_rng(0)
    pool = rng.permutation(6000)[:2100].astype(np.int32)           # unsorted, spans three slices
    h.set_pool(pool)
    keys, vals = h.topk(qidx, 25)
    h2 = make(P, np.ascontiguousarray(Q[pool]), Qb[pool])
    k2, v2 = h2.topk(qidx, 25)
    assert np.array_equal(keys, pool[k2]) and np.array_equal(bits(vals), bits(v2))
    # duplicates: equal scores rank by pool position, as on the gathered matrix
    dup = np.array([7, 7, 5, 7, 5999, 5], dtype=np.int32)
    h.set_pool(dup)
    keys, vals = h.topk(qidx, 8)
    h3 = make(P, np.ascontiguousarray(Q[dup]), Qb[dup])
    k3, v3 = h3.topk(qidx, 8)
    assert (keys[:, 6:] == -1).all() and (vals[:, 6:] == 0).all()              # fewer than k candidates
    assert np.array_equal(keys[:, :6], dup[k3[:, :6]]) and np.array_equal(bits(vals), bits(v3))
    for r in range(45):
        pos = k3[r, :6]
        same = vals[r, :5] == vals[r, 1:6]
        assert (pos[:-1][same] < pos[1:][same]).all()
    # removing the pool restores the full ranking; an empty pool and an index outside the items are errors
    h.set_pool(None)
    assert np.array_equal(h.topk(qidx, 25)[0], reference(P, Q, Qb, qidx, 25)[0])
    with pytest.raises(ValueError, match="pool is empty"):
        h.set_pool([])
    with pytest.raises(ValueError, match="out of range"):
        h.set_pool([6000])
    assert cuda_lib.bfl_serve_set_pool(h._h, pool.ctypes.data, 0) == 4        # BFL_ERR_ARG
    for x in (h, h2, h3):
        x.close()


def test_wide_rows_with_pool_use_the_gathered_path(cuda_lib):
    P, Q, Qb = factors(20, 5000, 300, 300, 8, True)
    pool = np.random.default_rng(1).permutation(5000)[:1500].astype(np.int32)
    h = make(P, Q, Qb)
    h.set_pool(pool)
    qidx = np.arange(20, dtype=np.int32)[::-1].copy()
    keys, vals = h.topk(qidx, 12)
    rk, rv = reference(P, Q, Qb, qidx, 12, pool=pool)
    assert np.array_equal(keys, rk) and np.array_equal(bits(vals), bits(rv))
    h.close()


def test_batching_and_repeated_calls(cuda_lib):
    """k = 4096 on 200k items makes the internal batch 160 queries: 500 queries span four batches."""
    P, Q, _ = factors(600, 200_000, 8, 8, 13, False)
    h = make(P, Q, None)
    qidx = np.random.default_rng(3).integers(0, 600, size=500).astype(np.int32)
    keys, vals = h.topk(qidx, 4096)
    parts = [h.topk(qidx[a:a + 160], 4096) for a in range(0, 500, 160)]
    assert np.array_equal(keys, np.concatenate([p[0] for p in parts]))
    assert np.array_equal(bits(vals), np.concatenate([bits(p[1]) for p in parts]))
    sub = np.array([0, 159, 160, 499])
    rk, rv = reference(P, Q, None, qidx[sub], 4096)
    assert np.array_equal(keys[sub], rk) and np.array_equal(bits(vals[sub]), bits(rv))
    # five queries over 196 slices go to the 4-query kernels (more slices than SMs), 40 to the batch kernel; a pool of
    # 150k candidates keeps both above that limit
    pool = np.random.default_rng(5).permutation(200_000)[:150_000].astype(np.int32)
    for pl in (None, pool):
        h.set_pool(pl)
        for n in (5, 40):
            sk, sv = h.topk(qidx[:n], 10)
            rk, rv = reference(P, Q, None, qidx[:n], 10, pool=pl)
            assert np.array_equal(sk, rk) and np.array_equal(bits(sv), bits(rv)), n
    h.set_pool(None)
    again = h.topk(qidx, 4096, want_scores=False)
    assert again[1] is None and np.array_equal(again[0], keys)
    h.close()


def test_most_similar_aliases_items(cuda_lib):
    _, Q, _ = factors(1, 3000, 24, 24, 17, False)
    Q /= np.linalg.norm(Q, axis=1, keepdims=True)
    from buffalo_b200 import backend
    h = backend.Serve()
    h.set_items(Q)
    h.set_queries(Q)
    qidx = np.array([0, 2999, 1024, 77], dtype=np.int32)
    keys, vals = h.topk(qidx, 6)
    assert np.array_equal(keys[:, 0], qidx) and np.abs(vals[:, 0] - 1).max() <= 1e-6
    rk, rv = reference(Q, Q, None, qidx, 6)
    assert np.array_equal(keys, rk) and np.array_equal(bits(vals), bits(rv))
    h.close()


def test_device_pointer_path_equals_host_path(cuda_lib):
    import torch
    from buffalo_b200 import backend
    P, Q, Qb = factors(300, 9000, 64, 64, 19, True)
    pool = np.arange(8999, 100, -3).astype(np.int32)
    qidx = np.random.default_rng(4).integers(0, 300, size=257).astype(np.int32)
    h = make(P, Q, Qb)
    h.set_pool(pool)
    keys, vals = h.topk(qidx, 50)
    g = backend.Serve()
    g.bind_items(torch.from_numpy(Q).cuda(), torch.from_numpy(Qb).cuda())
    g.bind_queries(torch.from_numpy(P).cuda())
    g.set_pool(pool)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        di, dv = g.topk_device(torch.from_numpy(qidx).cuda(), 50, stream=stream)
    stream.synchronize()
    assert np.array_equal(di.cpu().numpy(), keys) and np.array_equal(bits(dv.cpu().numpy()), bits(vals))
    hk, hv = g.topk(qidx, 50)                      # host arrays against bound device factors
    assert np.array_equal(hk, keys) and np.array_equal(bits(hv), bits(vals))
    h.close()
    g.close()


def test_destroy_returns_device_memory_and_leaves_no_thread(cuda_lib):
    import torch
    P, Q, Qb = factors(2000, 50_000, 32, 32, 23, True)
    qidx = np.arange(2000, dtype=np.int32)

    def use():
        h = make(P, Q, Qb)
        h.set_pool(np.arange(0, 50_000, 2, dtype=np.int32))
        out = h.topk(qidx, 100)
        h.close()
        torch.cuda.synchronize()
        return out
    first = use()                                   # loads the kernels and warms the stream-ordered allocator
    threads = threading.active_count()
    free0 = torch.cuda.mem_get_info()[0]
    second = use()
    assert torch.cuda.mem_get_info()[0] == free0
    assert threading.active_count() == threads
    assert np.array_equal(first[0], second[0])


def test_k_at_least_the_slice_length(cuda_lib):
    """k = 2048 over slices of 1024 candidates: every slice hands all of its candidates to the merge."""
    P, Q, Qb = factors(40, 2500, 12, 12, 29, True)
    h = make(P, Q, Qb)
    qidx = np.arange(40, dtype=np.int32)
    for k in (1024, 2048, 2500, 3000):
        keys, vals = h.topk(qidx, k)
        rk, rv = reference(P, Q, Qb, qidx, k)
        assert np.array_equal(keys, rk) and np.array_equal(bits(vals), bits(rv)), k
    h.close()


def test_new_items_clear_the_queries_and_the_pool(cuda_lib):
    from buffalo_b200 import _cabi
    P, Q, _ = factors(30, 3000, 16, 16, 31, False)
    h = make(Q, Q, None)                            # queries alias the resident items
    h.set_pool(np.arange(100, dtype=np.int32))
    qidx = np.arange(30, dtype=np.int32)
    h.topk(qidx, 5)
    P2, Q2, Qb2 = factors(30, 9000, 40, 40, 32, True)      # more rows (a new buffer) and wider rows than the old queries
    h.set_items(Q2, Qb2)
    out = np.zeros((30, 5), np.int32)
    assert h.num_queries == 0
    assert cuda_lib.bfl_serve_topk(h._h, qidx.ctypes.data, 30, 5, out.ctypes.data, None) == 3     # BFL_ERR_STATE
    with pytest.raises(ValueError, match="at least d columns"):
        h.set_queries(P)
    assert cuda_lib.bfl_serve_set_queries(h._h, P.ctypes.data, 30, 16) == 4                       # BFL_ERR_ARG
    h.set_queries(P2)
    keys, vals = h.topk(qidx, 5)
    rk, rv = reference(P2, Q2, Qb2, qidx, 5)        # all 9000 items again: the pool went with the old items
    assert np.array_equal(keys, rk) and np.array_equal(bits(vals), bits(rv))
    h.close()


def test_bound_item_rows_must_be_aligned(cuda_lib):
    import torch
    from buffalo_b200 import _cabi, backend
    buf = torch.zeros(100 * 8 + 1, dtype=torch.float32, device="cuda")
    g = backend.Serve()
    with pytest.raises(_cabi.BackendError, match="16-byte aligned"):
        g.bind_items(buf[1:].view(100, 8))
    # rows of 7 floats are read one float at a time: any float address will do
    odd = torch.randn(100 * 7 + 1, device="cuda")[1:].view(100, 7)
    g.bind_items(odd)
    g.bind_queries(odd)
    di, dv = g.topk_device(torch.arange(100, dtype=torch.int32, device="cuda"), 4)
    torch.cuda.synchronize()
    Qh = odd.cpu().numpy().copy()
    rk, rv = reference(Qh, Qh, None, np.arange(100), 4)
    assert np.array_equal(di.cpu().numpy(), rk) and np.array_equal(bits(dv.cpu().numpy()), bits(rv))
    g.close()


# ---- API level ----------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def ml100k_like(tmp_path_factory):
    """943 x 1682 with ~100k interactions from a planted rank-8 model, as a MatrixMarket file plus uid / iid files."""
    rng = np.random.default_rng(42)
    U, I, r = 943, 1682, 8
    S = rng.normal(size=(U, r)) @ rng.normal(size=(I, r)).T + rng.gumbel(size=(U, I)) * 0.5 + rng.normal(size=I)[None, :]
    rows, cols = np.nonzero(S > np.quantile(S, 1 - 100000 / (U * I)))
    vals = rng.integers(1, 6, len(rows))
    d = tmp_path_factory.mktemp("serve_ml")
    paths = {n: os.path.join(d, n) for n in ("main", "uid", "iid")}
    with open(paths["main"], "w") as f:
        f.write("%%MatrixMarket matrix coordinate integer general\n%d %d %d\n" % (U, I, len(rows)))
        f.writelines("%d %d %d\n" % (a + 1, b + 1, v) for a, b, v in zip(rows, cols, vals))
    with open(paths["uid"], "w") as f:
        f.write("\n".join("user_%d" % i for i in range(U)))
    with open(paths["iid"], "w") as f:
        f.write("\n".join("item_%d" % i for i in range(I)))
    return dict(paths, dir=str(d))


def train(ml, cls_name, name, **kw):
    import buffalo
    from buffalo.data import MatrixMarketOptions
    o = MatrixMarketOptions().get_default_option()
    o.input.main, o.input.uid, o.input.iid = ml["main"], ml["uid"], ml["iid"]
    o.data.path = os.path.join(ml["dir"], name + ".h5py")
    opt = getattr(buffalo, cls_name + "Option")().get_default_option()
    opt.update(random_seed=7, **kw)
    algo = getattr(buffalo, cls_name)(opt, data_opt=o)
    algo.initialize()
    algo.train()
    return algo


@pytest.mark.parametrize("cls_name,par_name,kw", [("ALS", "ParALS", dict(num_iters=4, d=20)),
                                                  ("BPRMF", "ParBPRMF", dict(num_iters=5, d=20, use_bias=True))])
def test_par_matches_algo_on_trained_model(cuda_lib, ml100k_like, cls_name, par_name, kw):
    import buffalo
    algo = train(ml100k_like, cls_name, "serve_" + cls_name.lower(), **kw)
    algo.build_itemid_map()
    algo.build_userid_map()
    par = getattr(buffalo, par_name)(algo)
    users = ["user_%d" % i for i in range(0, 943, 3)] + ["nobody"]
    kept, names, scores = par.topk_recommendation(users, topk=10, repr=True)
    assert kept == users[:-1] and scores.shape == (len(kept), 10) and scores.dtype == np.float32
    want = algo.topk_recommendation(users, topk=10)
    assert all(names[i] == want[u] for i, u in enumerate(kept))
    _, keys, _ = par.topk_recommendation(users, topk=10)
    assert keys.dtype == np.int32 and [[algo._idmanager.itemids[t] for t in row] for row in keys] == names
    pool = ["item_%d" % i for i in range(5, 400, 7)]
    _, pnames, _ = par.topk_recommendation(users, topk=10, pool=pool, repr=True)
    pwant = algo.topk_recommendation(users, topk=10, pool=pool)
    assert all(pnames[i] == pwant[u] for i, u in enumerate(kept))
    with pytest.raises(RuntimeError, match="pool is empty"):
        par.topk_recommendation(users, topk=10, pool=[])
    # the factors are live arrays: an in-place edit and a second train() (which writes the same arrays in place when d
    # is a multiple of 4) must both show in the next query
    algo.Q[:] = algo.Q[::-1].copy()
    if algo.opt.get("use_bias"):
        algo.Qb[:] = algo.Qb[::-1].copy()
    _, names2, _ = par.topk_recommendation(users, topk=10, repr=True)
    want2 = algo.topk_recommendation(users, topk=10)
    assert all(names2[i] == want2[u] for i, u in enumerate(kept)) and names2 != names
    q_before, key2 = algo.Q, par._serve_key
    algo.train()
    _, names3, _ = par.topk_recommendation(users, topk=10, repr=True)
    want3 = algo.topk_recommendation(users, topk=10)
    assert all(names3[i] == want3[u] for i, u in enumerate(kept)) and par._serve_key != key2
    if algo.Q is q_before:                          # unchanged factors are not uploaded again
        key = par._serve_key
        par.topk_recommendation(users[:5], topk=3)
        assert par._serve_key == key
    # normalising replaces algo.Q; items are then compared with items
    items = algo._idmanager.itemids[:130]
    keys, sims = par.most_similar(items, topk=5)
    assert par._serve.num_items == 1682 and par._serve.num_queries == 130
    assert keys[:, 0].tolist() == list(range(130)) and np.abs(sims[:, 0] - 1).max() < 1e-3   # Algo.normalize adds an epsilon to the norm
    s = algo.Q.astype(np.float64) @ algo.Q.astype(np.float64).T
    assert np.abs(np.take_along_axis(s[:130], keys.astype(np.int64), axis=1) - sims).max() < 1e-5
    with pytest.raises(RuntimeError, match="normalized"):
        par.topk_recommendation(users, topk=10)

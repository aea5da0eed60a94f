"""Batch recommendations without each user's seen items on the device (csrc/serve.cu bfl_seen_topk*, backend.Serve
topk_seen*, ParALS / ParBPRMF.topk_recommendation(exclude_seen=...)): the survivors are exactly the unfiltered call's
items minus the seen ones, in its order and with its score bits, on the batch kernel and on the 4-query path."""
import threading

import numpy as np
import pytest

from tests.test_serve_gpu import bits, factors, make, ml100k_like, train  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu


def seen_rows(n, I, seed, mean=40, long_rows=()):
    """n rows of item ids in [0, I): Zipf lengths around `mean`, duplicates, session order; rows listed in long_rows
    get that many keys.  Returns (END offsets int64, keys int32, list of rows)."""
    rng = np.random.default_rng(seed)
    lens = np.minimum(rng.zipf(1.6, size=n) * (mean // 4), 10 * mean)
    rows = [rng.integers(0, I, size=int(x)).astype(np.int32) for x in lens]
    for r, m in long_rows:
        rows[r] = rng.integers(0, I, size=m).astype(np.int32)
    ptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
    return ptr, (np.concatenate(rows) if ptr[-1] else np.zeros(0, np.int32)), rows


def expected(h, qidx, k, rows, pool=None):
    """The unfiltered call for enough candidates, with each row's seen items dropped, cut to k, -1 / 0.0 padded."""
    ncand = h.num_items if pool is None else len(pool)
    K = min(4096, ncand, k + max(len(np.unique(r)) for r in rows) if pool is None else ncand)
    keys, vals = h.topk(qidx, K)
    ek = np.full((len(qidx), k), -1, np.int32)
    ev = np.zeros((len(qidx), k), np.float32)
    for i, r in enumerate(rows):
        keep = (keys[i] >= 0) & ~np.isin(keys[i], r)
        ek[i, :min(k, keep.sum())] = keys[i][keep][:k]
        ev[i, :min(k, keep.sum())] = vals[i][keep][:k]
    return ek, ev


def fp64_check(P, Q, Qb, qidx, rows, keys, vals, pool=None):
    """The ids are the fp64 ranking's outside rounding ties: scores match within an fp32 bound, descending, and the set
    of the k best unseen candidates is the fp64 one wherever the k-th and (k+1)-th are further apart than that bound."""
    cand = np.arange(Q.shape[0]) if pool is None else np.asarray(pool)
    s = P[qidx].astype(np.float64) @ Q[cand].astype(np.float64).T
    mag = np.abs(P[qidx]).astype(np.float64) @ np.abs(Q[cand]).astype(np.float64).T
    if Qb is not None:
        s += Qb[cand].astype(np.float64)[None, :]
        mag += np.abs(Qb[cand])[None, :]
    bound = (P.shape[1] + 2) * 2.0 ** -24 * mag
    checked = 0
    for i, r in enumerate(rows):
        live = np.nonzero(~np.isin(cand, r))[0]
        order = live[np.argsort(-s[i, live], kind="stable")]
        k = keys.shape[1]
        got = keys[i][keys[i] >= 0]
        assert len(got) == min(k, len(live)) and not np.isin(got, r).any()
        pos = {c: j for j, c in enumerate(cand)} if pool is not None else None
        gp = got if pool is None else np.array([pos[g] for g in got], dtype=np.int64)
        assert np.abs(vals[i, :len(got)] - s[i, gp]).max(initial=0) <= 2 * bound[i].max()
        if len(order) > k and s[i, order[k - 1]] - s[i, order[k]] > bound[i, order[k - 1]] + bound[i, order[k]]:
            assert set(cand[order[:k]].tolist()) == set(got.tolist())
            checked += 1
    return checked


@pytest.mark.parametrize("use_pool", [False, True])
@pytest.mark.parametrize("bias", [False, True])
@pytest.mark.parametrize("d", [1, 5, 20, 128, 256, 300])
def test_equals_unfiltered_minus_seen_and_fp64(cuda_lib, d, bias, use_pool):
    # 5003 items: five slices, the last one short; 70 queries (two CTAs) and 9 (one, mostly empty); one history longer
    # than a slice
    P, Q, Qb = factors(90, 5003, d, d, 300 + d, bias)
    h = make(P, Q, Qb)
    pool = np.random.default_rng(d).permutation(5003)[:2100].astype(np.int32) if use_pool else None
    h.set_pool(pool)
    ptr, keys, rows = seen_rows(70, 5003, d, long_rows=[(3, 1500)])
    qidx = np.random.default_rng(d + 1).permutation(90)[:70].astype(np.int32)
    for n, k in ((70, 10), (70, 100), (9, 10)):
        p = ptr[:n]
        got_k, got_v = h.topk_seen(qidx[:n], k, p, keys)
        ek, ev = expected(h, qidx[:n], k, rows[:n], pool)
        assert np.array_equal(got_k, ek), (n, k)
        assert np.array_equal(bits(got_v), bits(ev)), (n, k)
        checked = fp64_check(P, Q, Qb, qidx[:n], rows[:n], got_k, got_v, pool)
        assert checked >= n // 2
    h.close()


def test_few_queries_over_many_slices_use_the_4_query_path(cuda_lib):
    """5 queries over 150k candidates (more slices than SMs) go to the gathered 4-query kernels; 40 to the batch kernel."""
    P, Q, Qb = factors(60, 160_000, 20, 20, 41, True)
    h = make(P, Q, Qb)
    pool = np.random.default_rng(6).permutation(160_000)[:150_000].astype(np.int32)
    ptr, keys, rows = seen_rows(40, 160_000, 7, mean=200, long_rows=[(1, 5000)])
    qidx = np.arange(40, dtype=np.int32)
    for pl in (None, pool):
        h.set_pool(pl)
        for n in (5, 40):
            got_k, got_v = h.topk_seen(qidx[:n], 10, ptr[:n], keys)
            ek, ev = expected(h, qidx[:n], 10, rows[:n], pl)
            assert np.array_equal(got_k, ek) and np.array_equal(bits(got_v), bits(ev)), n
    h.close()


def test_padding_and_pools_inside_the_history(cuda_lib):
    for d in (20, 300):                             # the batch kernel and the gathered path
        P, Q, Qb = factors(6, 3000, d, d, 51, True)
        h = make(P, Q, Qb)
        qidx = np.arange(6, dtype=np.int32)
        everything = np.arange(3000, dtype=np.int32)[::-1].copy()
        all_but_3 = np.setdiff1d(everything, [5, 1999, 2999]).astype(np.int32)
        rows = [everything, all_but_3, np.zeros(0, np.int32), all_but_3[:10], everything[:2990], all_but_3]
        ptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
        keys = np.concatenate(rows)
        got_k, got_v = h.topk_seen(qidx, 20, ptr, keys)
        assert (got_k[0] == -1).all() and (got_v[0] == 0).all()
        assert sorted(got_k[1, :3].tolist()) == [5, 1999, 2999] and (got_k[1, 3:] == -1).all()
        assert (got_v[1, 3:] == 0).all() and len(set(got_k[4].tolist()) - {-1}) == 10
        ek, ev = expected(h, qidx, 20, rows)
        assert np.array_equal(got_k, ek) and np.array_equal(bits(got_v), bits(ev))
        # a pool entirely seen, and one with two unseen candidates
        h.set_pool(np.array([7, 3, 7, 100], np.int32))
        one = [np.array([100, 3, 7], np.int32)] * 6
        got_k, got_v = h.topk_seen(qidx, 4, np.cumsum([3] * 6).astype(np.int64), np.concatenate(one))
        assert (got_k == -1).all() and (got_v == 0).all()
        got_k, got_v = h.topk_seen(qidx, 4, np.cumsum([2] * 6).astype(np.int64), np.concatenate([[7, 7]] * 6).astype(np.int32))
        ek, ev = expected(h, qidx, 4, [np.array([7], np.int32)] * 6, pool=np.array([7, 3, 7, 100], np.int32))
        assert np.array_equal(got_k, ek) and np.array_equal(bits(got_v), bits(ev))
        assert set(got_k[:, :2].ravel().tolist()) <= {3, 100} and (got_k[:, 2:] == -1).all()
        h.close()


def test_long_histories_and_key_batches(cuda_lib):
    """Histories far longer than a slice and than the pinned result staging (3 queries x k = 1), a single row above the
    2^24 keys of one seen batch, and 40 rows of 500k keys that the key budget cuts into several batches."""
    P, Q, _ = factors(50, 5003, 16, 16, 61, False)
    h = make(P, Q, None)
    rng = np.random.default_rng(8)
    rows = [rng.integers(0, 5003, size=4000).astype(np.int32) for _ in range(3)]
    ptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
    got_k, got_v = h.topk_seen(np.arange(3, dtype=np.int32), 1, ptr, np.concatenate(rows))
    ek, ev = expected(h, np.arange(3, dtype=np.int32), 1, rows)
    assert np.array_equal(got_k, ek) and np.array_equal(bits(got_v), bits(ev))
    big = rng.integers(0, 5000, size=(1 << 24) + 1000).astype(np.int32)        # items 5000..5002 stay unseen
    rows = [big] + [rng.integers(0, 5003, size=500_000).astype(np.int32) for _ in range(40)]
    ptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
    qidx = rng.integers(0, 50, size=41).astype(np.int32)
    got_k, got_v = h.topk_seen(qidx, 5, ptr, np.concatenate(rows))
    assert sorted(got_k[0, :3].tolist()) == [5000, 5001, 5002] and (got_k[0, 3:] == -1).all()
    ek, ev = expected(h, qidx, 5, [np.unique(r) for r in rows])
    assert np.array_equal(got_k, ek) and np.array_equal(bits(got_v), bits(ev))
    h.close()


def test_many_batches_and_alternating_calls(cuda_lib):
    """k = 4096 on 200k items makes the internal batch 160 queries: 400 queries span three batches."""
    P, Q, _ = factors(500, 200_000, 8, 8, 71, False)
    h = make(P, Q, None)
    qidx = np.random.default_rng(3).integers(0, 500, size=400).astype(np.int32)
    ptr, keys, rows = seen_rows(400, 200_000, 9, mean=60)
    plain = h.topk(qidx, 4096)
    first = h.topk_seen(qidx, 4096, ptr, keys)
    again = h.topk(qidx, 4096)
    second = h.topk_seen(qidx, 4096, ptr, keys)
    assert np.array_equal(plain[0], again[0]) and np.array_equal(bits(plain[1]), bits(again[1]))
    assert np.array_equal(first[0], second[0]) and np.array_equal(bits(first[1]), bits(second[1]))
    for i in (0, 159, 160, 399):
        keep = ~np.isin(plain[0][i], rows[i])
        m = min(4096, keep.sum())
        assert np.array_equal(first[0][i, :m], plain[0][i][keep][:m])
        assert np.array_equal(bits(first[1][i, :m]), bits(plain[1][i][keep][:m]))
    h.close()


def test_unsorted_rows_with_duplicates_equal_sorted_rows_and_device_call(cuda_lib):
    import torch
    P, Q, Qb = factors(200, 9000, 64, 64, 81, True)
    h = make(P, Q, Qb)
    h.set_pool(np.arange(8999, 100, -3).astype(np.int32))
    ptr, keys, rows = seen_rows(180, 9000, 10, mean=80)
    qidx = np.random.default_rng(4).integers(0, 200, size=180).astype(np.int32)
    a = h.topk_seen(qidx, 50, ptr, keys)
    srows = [np.unique(r) for r in rows]
    sptr = np.cumsum([len(r) for r in srows]).astype(np.int64)
    b = h.topk_seen(qidx, 50, sptr, np.concatenate(srows).astype(np.int32))
    assert np.array_equal(a[0], b[0]) and np.array_equal(bits(a[1]), bits(b[1]))
    # the device call on unsorted rows (sorted by the radix sort first), and on rows named through seen_row
    di, dv = h.topk_seen_device(torch.from_numpy(qidx).cuda(), 50, torch.from_numpy(ptr).cuda(),
                                torch.from_numpy(keys).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(di.cpu().numpy(), a[0]) and np.array_equal(bits(dv.cpu().numpy()), bits(a[1]))
    perm = np.random.default_rng(5).permutation(180)
    inv = np.argsort(perm)
    prow = [srows[i] for i in perm]
    pptr = np.cumsum([len(r) for r in prow]).astype(np.int64)
    di, dv = h.topk_seen_device(torch.from_numpy(qidx).cuda(), 50, torch.from_numpy(pptr).cuda(),
                                torch.from_numpy(np.concatenate(prow).astype(np.int32)).cuda(),
                                seen_row=torch.from_numpy(inv.astype(np.int32)).cuda())
    torch.cuda.synchronize()
    assert np.array_equal(di.cpu().numpy(), a[0]) and np.array_equal(bits(dv.cpu().numpy()), bits(a[1]))
    h.close()


def test_destroy_returns_device_memory_and_leaves_no_thread(cuda_lib):
    import torch
    P, Q, Qb = factors(2000, 50_000, 32, 32, 23, True)
    qidx = np.arange(2000, dtype=np.int32)
    ptr, keys, _ = seen_rows(2000, 50_000, 11, mean=50)

    def use():
        h = make(P, Q, Qb)
        out = h.topk_seen(qidx, 100, ptr, keys)            # unsorted rows: the device sort runs too
        h.set_pool(np.arange(0, 50_000, 2, dtype=np.int32))
        out2 = h.topk_seen(qidx[:20], 100, ptr[:20], keys)  # the gathered path
        h.close()
        torch.cuda.synchronize()
        return out, out2
    first = use()
    threads = threading.active_count()
    free0 = torch.cuda.mem_get_info()[0]
    second = use()
    assert torch.cuda.mem_get_info()[0] == free0
    assert threading.active_count() == threads
    assert np.array_equal(first[0][0], second[0][0]) and np.array_equal(first[1][0], second[1][0])


@pytest.mark.parametrize("cls_name,par_name,kw", [("ALS", "ParALS", dict(num_iters=4, d=20)),
                                                  ("BPRMF", "ParBPRMF", dict(num_iters=5, d=20, use_bias=True))])
def test_device_equals_numpy_path_on_trained_model(cuda_lib, ml100k_like, monkeypatch, cls_name, par_name, kw):
    import buffalo
    import scipy.sparse
    from buffalo_b200 import backend
    algo = train(ml100k_like, cls_name, "seen_" + cls_name.lower(), **kw)
    algo.build_itemid_map()
    algo.build_userid_map()
    par = getattr(buffalo, par_name)(algo)
    users = ["user_%d" % i for i in range(0, 943, 3)]
    pool = ["item_%d" % i for i in range(5, 1600, 4)]
    grp = algo.data.get_group("rowwise")
    ptr = np.asarray(grp["indptr"][:], np.int64)
    m = scipy.sparse.csr_matrix((np.ones(int(ptr[-1])), np.asarray(grp["key"][:int(ptr[-1])]),
                                 np.concatenate([[0], ptr])), shape=(algo.P.shape[0], algo.Q.shape[0]))
    dev = [par.topk_recommendation(users, topk=10, exclude_seen=True),
           par.topk_recommendation(users, topk=10, exclude_seen=m),
           par.topk_recommendation(users, topk=10, pool=pool, exclude_seen=True)]
    plain = par.topk_recommendation(users, topk=10)
    monkeypatch.setattr(backend, "device_available", lambda: False)
    host = [par.topk_recommendation(users, topk=10, exclude_seen=True),
            par.topk_recommendation(users, topk=10, exclude_seen=m),
            par.topk_recommendation(users, topk=10, pool=pool, exclude_seen=True)]
    for a, b in zip(dev, host):
        assert a[0] == b[0] and np.array_equal(a[1], b[1])
        assert np.abs(a[2] - b[2]).max() < 1e-4
    assert np.array_equal(dev[0][1], dev[1][1]) and np.array_equal(bits(dev[0][2]), bits(dev[1][2]))
    seen = m[[int(u.split("_")[1]) for u in users]]
    assert not any(seen[i, dev[0][1][i]].toarray().any() for i in range(len(users)))
    assert not np.array_equal(plain[1], dev[0][1])

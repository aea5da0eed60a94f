"""End-to-end tests of the drop-in Python API on the GPU: `import buffalo` resolves to the H100 backend and the
reference's own usage (examples/example_als.py, tests/algo/base.py) works unchanged.  The reference's quality
floors (tests/algo/base.py:83-97: ALS ndcg > 0.06, map > 0.04; BPR/WARP ndcg > 0.03, map > 0.02 on ml-100k) are
applied to a synthetic ml-100k-shaped matrix with planted low-rank structure (the real file is an LFS pointer)."""
import os

import numpy as np
import pytest
import scipy.sparse

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ml100k_like(tmp_path_factory):
    """943 x 1682, ~100k interactions drawn from a rank-8 preference model, written as a MatrixMarket FILE plus
    uid / iid files, exactly the inputs of examples/example_als.py:16-17."""
    rng = np.random.default_rng(42)
    U, I, k = 943, 1682, 8
    A, B = rng.normal(size=(U, k)), rng.normal(size=(I, k))
    S = A @ B.T + rng.gumbel(size=(U, I)) * 0.5 + rng.normal(size=I)[None, :]
    thr = np.quantile(S, 1 - 100000 / (U * I))
    rows, cols = np.nonzero(S > thr)
    vals = rng.integers(1, 6, len(rows))
    d = tmp_path_factory.mktemp("ml")
    main = os.path.join(d, "main")
    with open(main, "w") as f:
        f.write("%%MatrixMarket matrix coordinate integer general\n%d %d %d\n" % (U, I, len(rows)))
        for r, c, v in zip(rows, cols, vals):
            f.write("%d %d %d\n" % (r + 1, c + 1, v))
    with open(os.path.join(d, "uid"), "w") as f:
        f.write("\n".join("user_%d" % i for i in range(U)))
    with open(os.path.join(d, "iid"), "w") as f:
        f.write("\n".join("item_%d" % i for i in range(I)))
    return dict(main=main, uid=os.path.join(d, "uid"), iid=os.path.join(d, "iid"), dir=str(d), U=U, I=I)


def data_option(ml, name):
    from buffalo.data import MatrixMarketOptions
    o = MatrixMarketOptions().get_default_option()
    o.input.main, o.input.uid, o.input.iid = ml["main"], ml["uid"], ml["iid"]
    o.data.path = os.path.join(ml["dir"], name + ".h5py")
    o.data.validation.p, o.data.validation.max_samples = 0.1, 10000
    return o


def test_example_als_flow(cuda_lib, ml100k_like):
    """examples/example_als.py:10-25, unchanged apart from the input paths."""
    import json
    from buffalo.algo import ALS, ALSOption
    from buffalo.misc import aux, log
    from buffalo.parallel import ParALS
    log.set_log_level(log.WARN)
    als_option = ALSOption().get_default_option()
    als_option.validation = aux.Option({"topk": 10})
    als_option.random_seed = 7
    als = ALS(als_option, data_opt=data_option(ml100k_like, "ex1"))
    als.initialize()
    assert als.P.shape == (943, 20) and als.Q.shape == (1682, 20)          # tests/algo/base.py:56-68
    ret = als.train()
    res = als.get_validation_results()
    json.dumps(res)
    assert res["ndcg"] > 0.06 and res["map"] > 0.04, res                    # tests/algo/base.py:83-97
    assert ret["train_loss"] > 0 and abs(ret["val_ndcg"] - res["ndcg"]) < 1e-9
    assert als.P.dtype == np.float32 and als.P.shape == (943, 20)
    sims = als.most_similar("item_49")
    assert len(sims) == 10 and all(isinstance(k, str) for k, _ in sims)
    als.normalize("item")
    als.build_itemid_map()
    par = ParALS(als)
    par.num_workers = 4
    topks, _ = par.most_similar(als._idmanager.itemids[:128], repr=True)
    assert len(topks) == 128 and len(topks[0]) == 10
    recs = als.topk_recommendation(["user_0", "user_5"], topk=5)
    assert set(recs) == {"user_0", "user_5"} and len(recs["user_0"]) == 5


@pytest.mark.parametrize("d,optimizer", [(5, "manual_cg"), (32, "ldlt"), (100, "ialspp"), (128, "manual_cg")])
def test_als_resident_equals_chunked_and_quality(cuda_lib, ml100k_like, d, optimizer):
    from buffalo import ALS, ALSOption, aux
    outs = []
    for resident, batch_mb in ((True, 1024), (False, 1)):      # batch_mb=1 forces several chunks per half-epoch
        opt = ALSOption().get_default_option()
        opt.update(d=d, optimizer=optimizer, num_iters=6, random_seed=11, validation=aux.Option({"topk": 10}),
                   block_size=7 if d == 100 else 32, _b200_resident=resident)
        dopt = data_option(ml100k_like, "rc%d" % d)
        dopt.data.batch_mb = batch_mb
        dopt.data.use_cache = True
        np.random.seed(5)          # same validation split in both runs
        als = ALS(opt, data_opt=dopt)
        als.initialize()
        ret = als.train()
        outs.append((als.P.copy(), als.Q.copy(), ret))
    (P1, Q1, r1), (P2, Q2, r2) = outs
    assert np.abs(P1 - P2).max() < 2e-3 * np.abs(P1).max() and np.abs(Q1 - Q2).max() < 2e-3 * np.abs(Q1).max()
    assert abs(r1["train_loss"] - r2["train_loss"]) < 1e-3 * r1["train_loss"]
    assert r1["val_ndcg"] > 0.06 and r1["val_map"] > 0.04, r1


def test_als_callbacks_save_load_early_stop(cuda_lib, ml100k_like, tmp_path):
    from buffalo import ALS, ALSOption, aux
    opt = ALSOption().get_default_option()
    opt.update(d=16, num_iters=4, random_seed=3, validation=aux.Option({"topk": 10}), save_best=True, save_period=1,
               model_path=str(tmp_path / "als.bin"), evaluation_period=2)
    als = ALS(opt, data_opt=data_option(ml100k_like, "cb"))
    als.initialize()
    calls = []
    als.train(training_callback=lambda i, m: calls.append((i, sorted(m))))
    assert [i for i, _ in calls] == [1, 3] and "val_ndcg" in calls[0][1]      # tests/algo/base.py:99-117
    assert os.path.isfile(opt.model_path)
    other = ALS.new(opt.model_path)
    assert other.Q.shape == als.Q.shape and other.opt.d == 16
    assert other.most_similar("item_3", 5)[0][0] == ALS.new(opt.model_path, ["Q", "_idmanager", "opt"]).most_similar("item_3", 5)[0][0]


@pytest.mark.parametrize("cls_name,kw", [
    ("BPRMF", dict(num_iters=30, lr=0.05, d=20)),
    ("BPRMF", dict(num_iters=30, lr=0.05, d=20, optimizer="adam", sampling_power=1.0)),
    ("WARP", dict(num_iters=15, d=32)),
    ("WARP", dict(num_iters=15, d=32, score_func="L2", optimizer="adam", lr=0.01)),
])
def test_sgd_trainers_quality(cuda_lib, ml100k_like, cls_name, kw):
    import buffalo
    from buffalo import aux
    cls = getattr(buffalo, cls_name)
    opt = getattr(buffalo, cls_name + "Option")().get_default_option()
    opt.update(random_seed=7, validation=aux.Option({"topk": 10}), evaluation_period=1000, **kw)
    algo = cls(opt, data_opt=data_option(ml100k_like, cls_name.lower()))
    algo.initialize()
    assert algo.P.shape[0] == 943 and algo.Q.shape[0] == 1682
    first = []
    ret = algo.train(training_callback=None)
    res = algo.get_validation_results()
    assert res["ndcg"] > 0.03 and res["map"] > 0.02, res                    # test_bpr.py:47, test_warp.py:48
    assert algo.P.shape == (943, kw["d"]) and np.isfinite(algo.P).all() and np.isfinite(algo.Q).all()
    if cls_name == "WARP":
        assert np.linalg.norm(algo.P, axis=1).max() <= 1.0 + 1e-4           # warp.cc:196-200
    assert len(algo.most_similar("item_10", 5)) == 5
    assert "train_loss" in ret and first == []


def test_csr_ingest_sort_on_device(cuda_lib):
    """SURVEY 8f.1: the (row, col) ordering of the ingest on the GPU equals the host build."""
    from buffalo_b200.data.base import csr_from_triples
    rng = np.random.default_rng(4)
    n, U, I = 3_000_000, 50_000, 20_000
    rows = rng.integers(0, U, n).astype(np.int64)
    cols = rng.integers(0, I, n).astype(np.int64)
    vals = rng.integers(1, 6, n).astype(np.float32)
    a = csr_from_triples(rows[:200000], cols[:200000], vals[:200000], U)              # < threshold: host path
    b = csr_from_triples(rows[:200000], cols[:200000], vals[:200000], U, device="cuda")
    assert all(np.array_equal(x, y) for x, y in zip(a, b))
    c = csr_from_triples(rows, cols, vals, U)                                        # >= threshold: device path
    assert c[0][-1] == n and np.all(np.diff(c[0]) >= 0)
    beg = np.concatenate([[0], c[0][:-1]])
    for r in (0, 17, U - 1):
        assert np.all(np.diff(c[1][beg[r]:c[0][r]]) >= 0)

"""Item fold-in (ALS / BPRMF / WARP .fold_in_items) and Algo.add_items where no GPU is needed: every input check raises
before any device work, a valid call without a GPU raises the backend's error, add_items appends and round-trips,
train() refuses a grown catalogue, and the NumPy reference of the SGD fold-in passes hand-checked d = 2 cases."""
import math

import numpy as np
import pytest
import scipy.sparse

from tests import item_fold_in_ref as ref


class TinyData(object):
    """The parts of a Data object the fold-in reads: the header and the rowwise group."""

    def __init__(self, U, I, seed=0):
        rng = np.random.default_rng(seed)
        rows = [np.sort(rng.choice(I, size=3, replace=False)) for _ in range(U)]
        self.indptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
        self.keys = np.concatenate(rows).astype(np.int32)
        self.header = {"num_users": U, "num_items": I, "num_nnz": len(self.keys)}

    def get_header(self):
        return self.header

    def get_group(self, name):
        assert name == "rowwise"
        return {"indptr": self.indptr, "key": self.keys, "val": np.ones(len(self.keys), np.float32)}


def cpu_model(kind="als", U=30, I=50, d=8, data=True, **opt):
    """A model object with factors, an item-id map and (data=True) training data, built without the backend holder."""
    from buffalo_b200.algo.als import ALS
    from buffalo_b200.algo.bpr import BPRMF
    from buffalo_b200.algo.options import ALSOption, BPRMFOption, WARPOption
    from buffalo_b200.algo.warp import WARP
    from buffalo_b200.misc import aux
    cls, opt_cls = {"als": (ALS, ALSOption), "bpr": (BPRMF, BPRMFOption), "warp": (WARP, WARPOption)}[kind]
    m = cls.__new__(cls)
    m.opt = aux.Option(opt_cls().get_default_option())
    m.opt.update(dict(d=d, **opt))
    rng = np.random.default_rng(1)
    m.P = rng.random((U, d)).astype(np.float32)
    m.Q = rng.random((I, d)).astype(np.float32)
    if kind != "als":
        m.Qb = rng.random((I, 1)).astype(np.float32)
    m.data = TinyData(U, I) if data else None
    m._idmanager = aux.Option({"userids": ["u%d" % i for i in range(U)], "itemids": ["i%d" % i for i in range(I)],
                               "userid_mapped": True, "itemid_mapped": True})
    m._idmanager.userid_map = {v: i for i, v in enumerate(m._idmanager.userids)}
    m._idmanager.itemid_map = {v: i for i, v in enumerate(m._idmanager.itemids)}
    return m


@pytest.fixture
def no_device_work(monkeypatch):
    """Any step past the input checks (holder creation, upload) fails the test."""
    from buffalo_b200.algo import fold_in

    def refuse(*a, **k):
        raise AssertionError("device work before the input checks finished")
    monkeypatch.setattr(fold_in.ItemState, "refresh", refuse)
    monkeypatch.setattr(fold_in, "to_device", refuse)


def history(n, U, seed=0):
    rng = np.random.default_rng(seed)
    return scipy.sparse.random(n, U, density=0.2, format="csr", random_state=rng, dtype=np.float32)


KINDS = ["als", "bpr", "warp"]


def count_name(kind):
    return "sweeps" if kind == "als" else "epochs"


@pytest.mark.parametrize("kind", KINDS)
def test_input_checks_before_device_work(no_device_work, kind):
    m = cpu_model(kind)
    U, d = m.P.shape[0], m.opt.d
    good = history(4, U)
    with pytest.raises(ValueError, match="matrix"):
        m.fold_in_items(history(4, U + 1))
    bad = good.copy()
    bad.indices[0] = U + 3
    with pytest.raises(ValueError, match="outside"):
        m.fold_in_items(bad)
    for init in (np.zeros((3, d)), np.zeros((4, d + 1)), np.zeros(4 * d)):
        with pytest.raises(ValueError, match="init"):
            m.fold_in_items(good, init=init)
    with pytest.raises(ValueError, match="histories"):
        m.fold_in_items(np.zeros((4, U)))
    with pytest.raises(ValueError, match="history"):
        m.fold_in_items([["u0", "u1"], 5])
    for bad_count in (0, -1, 1.5, True):
        with pytest.raises(ValueError, match=count_name(kind)):
            m.fold_in_items(good, **{count_name(kind): bad_count})


def test_unknown_user_ids_dropped():
    from buffalo_b200.algo import fold_in
    m = cpu_model("bpr", U=12)
    ends, keys, vals = fold_in.history_csr(m, [["u7", "nope", "u2"], [], ["u11", "u0"]], 12, group="user")
    assert ends.tolist() == [2, 2, 4] and keys.tolist() == [2, 7, 0, 11] and vals.tolist() == [1.0] * 4


@pytest.mark.parametrize("kind", KINDS)
def test_normalized_users_refused(no_device_work, kind):
    m = cpu_model(kind, _nrz_P=True)
    with pytest.raises(RuntimeError, match="normalized"):
        m.fold_in_items(history(2, m.P.shape[0]))


@pytest.mark.parametrize("kind", ["bpr", "warp"])
def test_sgd_needs_training_data(no_device_work, kind):
    m = cpu_model(kind, data=False)
    with pytest.raises(ValueError, match="training data"):
        m.fold_in_items(history(2, m.P.shape[0]))


@pytest.mark.parametrize("kind", ["bpr", "warp"])
def test_sgd_models_still_have_no_user_fold_in(kind):
    m = cpu_model(kind)
    assert not callable(getattr(m, "_fold_in_device", None)) and not hasattr(m, "fold_in")


@pytest.mark.parametrize("kind", KINDS)
def test_no_cpu_fallback(kind):
    import torch
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    from buffalo_b200 import _cabi
    m = cpu_model(kind)
    before = [a.copy() for a in (m.P, m.Q, getattr(m, "Qb", m.Q))]
    with pytest.raises(_cabi.BackendError, match="no CPU fallback"):
        m.fold_in_items(history(3, m.P.shape[0]))
    assert all((a == b).all() for a, b in zip(before, (m.P, m.Q, getattr(m, "Qb", m.Q))))


# ---- add_items -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kind", KINDS)
def test_add_items_refusals_change_nothing(kind):
    m = cpu_model(kind)
    d, I = m.opt.d, m.Q.shape[0]
    rows = np.ones((2, d), np.float32)
    cases = [(["n1", "n1"], rows, None, "duplicates"), (["n1", "i3"], rows, None, "already known"),
             (["n1", "n2"], np.ones((2, d + 1)), None, "rows must be"), (["n1"], rows, None, "rows must be"),
             (["n1", "n2"], np.full((2, d), np.nan), None, "non-finite"), ("n1", rows, None, "list")]
    if kind == "als":
        cases.append((["n1", "n2"], rows, np.zeros(2), "no item biases"))
    else:
        cases += [(["n1", "n2"], rows, np.zeros(3), "bias must be"), (["n1", "n2"], rows, [0, np.inf], "non-finite")]
    for ids, r, b, msg in cases:
        with pytest.raises(ValueError, match=msg):
            m.add_items(ids, r, b)
        assert m.Q.shape[0] == I and len(m._idmanager.itemids) == I and "n1" not in m._idmanager.itemid_map
        if kind != "als":
            assert m.Qb.shape == (I, 1)


@pytest.mark.parametrize("kind", KINDS)
def test_add_items_appends_and_round_trips(kind, tmp_path):
    m = cpu_model(kind)
    I, d = m.Q.shape
    Q0 = m.Q.copy()
    rows = np.arange(3 * d, dtype=np.float32).reshape(3, d)
    bias = None if kind == "als" else np.array([0.5, -1.0, 2.0], np.float32)
    m.add_items(["n0", "n1", "n2"], rows, bias)
    assert m.Q.shape == (I + 3, d) and (m.Q[:I] == Q0).all() and (m.Q[I:] == rows).all()
    assert m._idmanager.itemids[I:] == ["n0", "n1", "n2"] and m.get_index("n1") == I + 1
    if kind != "als":
        assert m.Qb.shape == (I + 3, 1) and m.Qb[I:, 0].tolist() == bias.tolist()
        m.add_items(["n3"], rows[:1])
        assert m.Qb[-1, 0] == 0.0
    path = str(tmp_path / "model.bin")
    m.save(path)
    m2 = cpu_model(kind)
    m2.load(path)
    assert (m2.Q == m.Q).all() and m2._idmanager.itemids == m._idmanager.itemids
    assert m2.get_index("n2") == I + 2
    if kind != "als":
        assert (m2.Qb == m.Qb).all()


def test_add_items_normalizes_under_normalized_items():
    m = cpu_model("als")
    m.opt._nrz_Q = True
    rows = np.array([[3.0, 4.0] + [0.0] * (m.opt.d - 2)], np.float32)
    m.add_items(["n0"], rows)
    assert np.allclose(m.Q[-1, :2], [0.6, 0.8], atol=1e-6)


def test_add_items_builds_the_map_from_data():
    m = cpu_model("bpr")
    m._idmanager.itemid_mapped = False
    calls = []
    m.build_itemid_map = lambda: (calls.append(1), m._idmanager.update({"itemid_mapped": True}))
    m.add_items(["n0"], np.zeros((1, m.opt.d), np.float32))
    assert calls == [1] and m._idmanager.itemids[-1] == "n0"


@pytest.mark.parametrize("kind", KINDS)
def test_train_after_add_items_refuses_mismatched_data(kind):
    m = cpu_model(kind)
    m.add_items(["n0"], np.zeros((1, m.opt.d), np.float32))
    with pytest.raises(ValueError, match="add_items"):
        m.train()


# ---- the reference, by hand ------------------------------------------------------------------------------------
def one_user_case(num_items, optimizer, kind="bpr", **o):
    opt = dict(d=2, optimizer=optimizer, lr=0.1, min_lr=0.1, reg_i=0.0, reg_b=0.0, use_bias=False, verify_neg=False,
               random_seed=3, max_trials=10, threshold=1.0, beta1=0.9)
    opt.update(o)
    P = np.array([[1.0, 0.0]], np.float32)
    Q = np.tile(np.array([[0.5, 0.5]], np.float32), (num_items, 1))
    return opt, P, Q


def test_reference_bpr_sgd_by_hand():
    opt, P, Q = one_user_case(1, "sgd")
    X, Xb, negs, _ = ref.fold_in_items("bpr", opt, P, Q, np.zeros(1), np.array([0], np.int64), np.zeros(0, np.int32),
                                       None, np.array([1], np.int64), np.array([0], np.int32), np.zeros((1, 2)),
                                       np.zeros(1), 1)
    logit = 1.0 / (1.0 + math.exp(-0.5))            # x_uij = p . (x - q) = -0.5
    assert negs.tolist() == [[0]]
    assert np.allclose(X, [[0.1 * logit, 0.0]], rtol=1e-6) and Xb.tolist() == [0.0]


def test_reference_bpr_adagrad_by_hand():
    opt, P, Q = one_user_case(1, "adagrad", use_bias=True, reg_b=0.5)
    X, Xb, _, _ = ref.fold_in_items("bpr", opt, P, Q, np.array([0.25]), np.array([0], np.int64),
                                    np.zeros(0, np.int32), None, np.array([1], np.int64), np.array([0], np.int32),
                                    np.zeros((1, 2)), np.zeros(1), 1)
    logit = 1.0 / (1.0 + math.exp(-(-0.5 - 0.25)))   # x_uij = -0.5 + (b_x - b_j) = -0.75
    # adagrad on g = logit * p: the step is g / |g| per coordinate (0 where g = 0); bias the same with reg_b * 0
    assert np.allclose(X, [[0.1, 0.0]], rtol=1e-6)
    assert np.allclose(Xb, [0.1 * logit / (logit + 1e-10)], rtol=1e-6)


def test_reference_warp_dot_by_hand():
    # ten identical negatives, none seen: every draw violates at trial 2, Phi = ln((10 - 0 - 1) // 2) = ln 4
    opt, P, Q = one_user_case(10, "adagrad", kind="warp")
    args = (np.zeros(10), np.array([0], np.int64), np.zeros(0, np.int32), None, np.array([1], np.int64),
            np.array([0], np.int32), np.zeros((1, 2)), np.zeros(1))
    X1, _, negs, trials = ref.fold_in_items("warp", opt, P, Q, *args, 1)
    assert trials.tolist() == [[2]] and 0 <= negs[0, 0] < 10
    assert np.allclose(X1, [[0.1, 0.0]], rtol=1e-6)
    # epoch 2: the accumulator keeps epoch 1's step (1) and adds ln 4; adagrad's v = (ln 4)^2 + (1 + ln 4)^2
    X2, _, _, trials = ref.fold_in_items("warp", opt, P, Q, *args, 2)
    g = 1.0 + math.log(4.0)
    assert trials.tolist() == [[2], [2]]
    assert np.allclose(X2, [[0.1 + 0.1 * g / math.sqrt(math.log(4.0) ** 2 + g * g), 0.0]], rtol=1e-6)


def test_reference_philox_known_answer():
    # Random123 known-answer vector for philox4x32-10
    assert ref.philox([0, 0, 0, 0], [0, 0]) == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]

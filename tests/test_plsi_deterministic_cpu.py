"""Deterministic pLSI without a GPU: an fp64 restatement of the two-pass iteration (item pass over the colwise CSR in
fixed segments, then the row pass) against tests/plsi_ref.plsi_iteration, and the trainer's memory estimate, mode
selection and chunk protocol with the backend replaced by fakes."""
import numpy as np
import pytest

from tests.helpers import rel_err, transpose_csr
from tests.plsi_ref import plsi_iteration, random_factors

SEGMENT = 4096          # kItemSegment in buffalo_b200/csrc/plsi.cu


def two_pass_iteration(P, Q, indptr, keys, vals, cindptr, ckeys, cvals, seg=SEGMENT, alpha1=1.0, alpha2=1.0):
    """fp64: the new item rows from the colwise CSR and the current P and Q, one partial row per segment of `seg`
    entries added in segment order; then the row pass without item accumulation.  Returns (P, Q, loss)."""
    P = np.asarray(P, dtype=np.float64)
    Q = np.asarray(Q, dtype=np.float64)
    d = P.shape[1]
    Qn = np.zeros_like(Q)
    beg = 0
    for i in range(Q.shape[0]):
        end = int(cindptr[i])
        for s0 in range(beg, end, seg):
            s1 = min(end, s0 + seg)
            u = np.asarray(ckeys[s0:s1], dtype=np.int64)
            v = np.asarray(cvals[s0:s1], dtype=np.float64)
            lat = np.maximum(P[u] * Q[i][None, :], 1e-10)
            Qn[i] += (lat / lat.sum(axis=1)[:, None] * v[:, None]).sum(axis=0)
        beg = end
    Pn = np.zeros_like(P)
    loss = 0.0
    beg = 0
    for x in range(P.shape[0]):
        end = int(indptr[x])
        if end > beg:
            c = np.asarray(keys[beg:end], dtype=np.int64)
            v = np.asarray(vals[beg:end], dtype=np.float64)
            lat = np.maximum(P[x][None, :] * Q[c], 1e-10)
            norm = lat.sum(axis=1)
            loss -= float(np.dot(v, np.log(norm)))
            Pn[x] = (lat / norm[:, None] * v[:, None]).sum(axis=0)
        beg = end
    with np.errstate(invalid="ignore", divide="ignore"):
        Pn += alpha1 / d
        Pn /= Pn.sum(axis=1, keepdims=True)
        Qn += alpha2 / Q.shape[0]
        Qn /= Qn.sum(axis=0, keepdims=True)
    return Pn, Qn, loss


def edge_matrix(U=18000, I=400, seed=31):
    """Empty user rows, 1-nnz rows, items nobody touched (the last 20), and item 3 held by every user with entries:
    more than three segments of 4096."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(0, 6, U)
    lens[rng.choice(U, 500, replace=False)] = 0
    lens[[5, 6, 7]] = 1
    rows = []
    for n in lens:
        pick = set(rng.choice(I - 20, size=int(n), replace=False).tolist()) if n else set()
        if n:
            pick.add(3)
        rows.append(sorted(pick))
    indptr = np.cumsum([len(r) for r in rows]).astype(np.int64)
    keys = np.array([k for r in rows for k in r], dtype=np.int32)
    vals = rng.lognormal(0.0, 1.0, len(keys)).astype(np.float32)
    return U, I, indptr, keys, vals


@pytest.mark.parametrize("seg", [SEGMENT, 1000, 1])
def test_two_pass_equals_fp64_mirror_on_edge_cases(seg):
    U, I, indptr, keys, vals = edge_matrix()
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
    clens = np.diff(cind, prepend=0)
    assert clens[3] > 3 * SEGMENT and (clens[-20:] == 0).all() and (np.diff(indptr, prepend=0) == 0).any()
    d = 6
    P, Q = random_factors(U, d, 1, axis=1), random_factors(I, d, 2, axis=0)
    for a1 in (1.0, 0.5):
        Pm, Qm, lm = plsi_iteration(P, Q, indptr, keys, vals, alpha1=a1)
        Pt, Qt, lt = two_pass_iteration(P, Q, indptr, keys, vals, cind, ckeys, cvals, seg=seg, alpha1=a1)
        assert rel_err(Pt, Pm) < 1e-12 and rel_err(Qt, Qm) < 1e-12, (rel_err(Pt, Pm), rel_err(Qt, Qm))
        assert abs(lt - lm) <= 1e-12 * abs(lm)


def test_two_pass_hand_checked_d2():
    """tests/test_plsi_cpu.py::test_hand_checked_d2 through the item pass: Q = [[1/7, 0.6], [6/7, 0.4]]."""
    P = np.array([[0.5, 0.5]], np.float32)
    Q = np.array([[0.25, 0.75], [0.75, 0.25]], np.float32)
    indptr, keys, vals = np.array([2], np.int64), np.array([0, 1], np.int32), np.array([1.0, 2.0], np.float32)
    cind, ckeys, cvals = transpose_csr(indptr, keys, vals, 1, 2)
    P1, Q1, loss = two_pass_iteration(P, Q, indptr, keys, vals, cind, ckeys, cvals, alpha1=0.0, alpha2=0.0)
    assert loss == pytest.approx(3 * np.log(2.0), rel=1e-12)
    np.testing.assert_allclose(P1, [[7 / 12, 5 / 12]], rtol=1e-12)
    np.testing.assert_allclose(Q1, [[1 / 7, 0.6], [6 / 7, 0.4]], rtol=1e-12)


# ---- the trainer with fake device functions --------------------------------------------------------------------
class FakeData(object):
    def __init__(self, U, I, indptr, keys, vals, batch_mb):
        from buffalo_b200.misc import aux
        cind, ckeys, cvals = transpose_csr(indptr, keys, vals, U, I)
        self.opt = aux.Option({"data": {"batch_mb": batch_mb}})
        self.header = {"num_users": U, "num_items": I, "num_nnz": int(indptr[-1])}
        self.groups = {"rowwise": {"indptr": indptr, "key": keys, "val": vals},
                       "colwise": {"indptr": cind, "key": ckeys, "val": cvals}}

    def get_header(self):
        return self.header

    def get_group(self, name):
        return self.groups[name]


class FakeCuPLSI(object):
    """Records the holder calls of the trainer."""

    def __init__(self):
        self.calls = []

    def item_segment_len(self):
        return SEGMENT

    def __getattr__(self, name):
        def record(*args):
            self.calls.append((name,) + tuple(a for a in args if isinstance(a, (int, float))))
            return 1.0 if name == "partial_update" else None
        return record


def fake_trainer(deterministic, U=18000, I=400, batch_mb=None, vdim=8):
    from buffalo_b200.algo.plsi import PLSI
    from buffalo_b200.data.buffered_data import BufferedDataMatrix
    from buffalo_b200.misc import aux, log
    U, I, indptr, keys, vals = edge_matrix(U, I)
    m = PLSI.__new__(PLSI)
    m.logger = log.get_logger("PLSI")
    opt = dict(d=vdim, num_iters=1, alpha1=1.0, alpha2=1.0, eps=1e-10)
    if deterministic is not None:
        opt["deterministic"] = deterministic
    m.opt = aux.Option(opt)
    m.data = FakeData(U, I, indptr, keys, vals, 64 if batch_mb is None else batch_mb)
    m.obj = FakeCuPLSI()
    m.vdim = vdim
    m.P = np.zeros((U, vdim), np.float32)
    m.Q = np.zeros((I, vdim), np.float32)
    m.buf = BufferedDataMatrix()
    m.buf.initialize(m.data)
    return m, indptr, keys, vals


@pytest.mark.parametrize("deterministic", [None, False, True])
def test_resident_bytes(deterministic):
    m, indptr, keys, vals = fake_trainer(deterministic)
    U, I, nnz, vdim = m.P.shape[0], m.Q.shape[0], len(keys), m.vdim
    base = nnz * 8 + U * (vdim * 4 + 9) + I * vdim * 8
    if not deterministic:
        assert m._resident_bytes() == base
        return
    clens = np.diff(m.data.get_group("colwise")["indptr"], prepend=0)
    segments = sum(-(-n // SEGMENT) for n in clens if n > SEGMENT)
    assert segments == -(-int(clens[3]) // SEGMENT) >= 4            # item 3 is the only long item
    assert m._resident_bytes() == base + nnz * 8 + I * 8 + U * 8 + segments * vdim * 4


@pytest.mark.parametrize("deterministic", [False, True])
@pytest.mark.parametrize("fits", [False, True])
def test_mode_selection(deterministic, fits):
    m, _, _, _ = fake_trainer(deterministic)
    need = m._resident_bytes()
    seen = []
    m._resident_capable = lambda n: seen.append(n) or (fits and n == need)
    m._train_resident = lambda cb: "resident"
    m._train_chunked = lambda cb: "chunked"
    m.validation_result = {}
    ret = m.train()
    assert seen == [need]
    assert ret["train_loss"] == ("resident" if fits else "chunked")


def test_chunked_protocol_sends_colwise_chunks_first():
    """batch_mb = 1: several colwise and rowwise chunks.  Deterministic mode: reset, the item pass over every colwise
    chunk in item order, the row pass over every rowwise chunk, normalize, swap."""
    for deterministic in (False, True):
        m, indptr, keys, vals = fake_trainer(deterministic, batch_mb=1)
        nume, deno = m._iterate()
        names = [c[0] for c in m.obj.calls]
        items = [c[1:3] for c in m.obj.calls if c[0] == "partial_update_items"]
        rows = [c[1:3] for c in m.obj.calls if c[0] == "partial_update"]
        assert names[0] == "reset" and names[-2:] == ["normalize", "swap"]
        if deterministic:
            assert len(items) > 1 and items[0][0] == 0 and items[-1][1] == m.Q.shape[0]
            assert all(a[1] == b[0] for a, b in zip(items, items[1:]))
            assert names.index("partial_update") > max(i for i, n in enumerate(names) if n == "partial_update_items")
        else:
            assert not items
        assert len(rows) > 1 and rows[0][0] == 0 and rows[-1][1] == m.P.shape[0]
        assert nume == float(len(rows)) and deno == pytest.approx(float(np.sum(vals, dtype=np.float64)), rel=1e-6)
        assert m.buf.group == "rowwise"

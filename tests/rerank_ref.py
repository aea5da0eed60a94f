"""fp64 NumPy reference of the MMR re-ranking (DESIGN.md 4.15) from its definition, plus the
input generator and the greedy-validity check the tests use.

Per row, over the valid candidates (id >= 0) in list order: rel_j = (s_j - s_min) / (s_max - s_min) (1 when all equal);
cos(a, b) the cosine of the item rows in fp64 (0 when either has zero norm); step t picks the unpicked candidate of the
largest (1 - w) rel_j - w max_{p picked} cos(p, j) (no max term at t = 0), ties to the smaller position."""
import numpy as np


def row_terms(ids, s, F):
    """(rel, cos) of one row's valid candidates: fp64 relevance and the fp64 cosine matrix of their fp32 rows."""
    s = np.asarray(s, np.float32).astype(np.float64)
    lo, hi = s.min(), s.max()
    rel = (s - lo) / (hi - lo) if hi > lo else np.ones(len(s))
    X = np.asarray(F, np.float32)[np.asarray(ids, np.int64)].astype(np.float64)
    G = X @ X.T
    nrm = np.diag(G)
    ok = (nrm[:, None] > 0) & (nrm[None, :] > 0)
    with np.errstate(divide="ignore", invalid="ignore"):
        return rel, np.where(ok, G / np.sqrt(nrm[:, None] * nrm[None, :]), 0.0)


def mmr_row(rel, cos, k, w):
    """(picked positions, per-step gap between the pick's objective and the next best, the next best's position)."""
    m = len(rel)
    picked = np.zeros(m, bool)
    maxsim = np.full(m, -np.inf)
    out, gaps, runner = [], [], []
    for t in range(min(k, m)):
        obj = (1.0 - w) * rel if t == 0 else (1.0 - w) * rel - w * maxsim
        obj = np.where(picked, -np.inf, obj)
        p = int(np.flatnonzero(obj == obj.max())[0])   # ties to the smaller position
        rest = obj.copy()
        rest[p] = -np.inf
        q = int(np.argmax(rest))
        gaps.append(obj[p] - rest[q] if np.isfinite(rest[q]) else np.inf)
        runner.append(q)
        out.append(p)
        picked[p] = True
        maxsim = np.maximum(maxsim, cos[p])
    return out, gaps, runner


def mmr_ref(cand_idx, cand_val, F, k, w):
    """(keys int32, scores float32) [n, k]: the picks in order with their given scores, -1 / 0.0 padded."""
    cand_idx, cand_val = np.asarray(cand_idx), np.asarray(cand_val, np.float32)
    n = cand_idx.shape[0]
    keys = np.full((n, k), -1, np.int32)
    scores = np.zeros((n, k), np.float32)
    for r in range(n):
        pos = np.flatnonzero(cand_idx[r] >= 0)
        if not pos.size:
            continue
        picked, _, _ = mmr_row(*row_terms(cand_idx[r, pos], cand_val[r, pos], F), k, w)
        keys[r, :len(picked)] = cand_idx[r, pos[picked]]
        scores[r, :len(picked)] = cand_val[r, pos[picked]]
    return keys, scores


def gap_inputs(n, M, d, w, seed, gap=1e-4):
    """(cand_idx int32 [n, M], cand_val float32 [n, M], F float32) whose fp64 MMR at k = M has, at every step whose
    ranking involves a cosine (w > 0, t >= 1), an objective gap of at least `gap` between the pick and the next
    candidate; the other steps rank by rel alone, which the device computes with the same fp64 operations.  Scores are
    distinct and best first, as the candidate stage returns them.  A candidate closer than the gap gets a fresh item row
    until the whole row passes (asserted)."""
    rng = np.random.default_rng(seed)
    spare = n * M + 64 * M + 64
    F = rng.standard_normal((spare, d)).astype(np.float32)
    nxt = 0
    cand_idx = np.empty((n, M), np.int32)
    cand_val = np.empty((n, M), np.float32)
    for r in range(n):
        ids = np.arange(nxt, nxt + M, dtype=np.int32)
        nxt += M
        s = (1.0 - np.arange(M) / M - rng.random(M) * 0.5 / M).astype(np.float32)
        for _ in range(64 * M):
            _, gaps, runner = mmr_row(*row_terms(ids, s, F), M, w)
            bad = [t for t in range(1, len(gaps)) if w > 0 and gaps[t] < gap]
            if not bad:
                break
            assert nxt < spare, "generator ran out of item rows"
            ids[runner[bad[0]]] = nxt
            nxt += 1
        else:
            raise AssertionError("no gap-asserted row found")
        cand_idx[r], cand_val[r] = ids, s
    return cand_idx, cand_val, F[:max(nxt, 1)]


def check_greedy(cand_idx, cand_val, F, w, keys, scores, tol=1e-6):
    """Greedy validity of given picks: at every step, given the earlier picks, the pick is an unpicked candidate (same
    id, bitwise the same score) whose fp64 objective is within tol of the largest; -1 / 0.0 exactly when none is left."""
    cand_idx, cand_val = np.asarray(cand_idx), np.asarray(cand_val, np.float32)
    for r in range(cand_idx.shape[0]):
        pos = np.flatnonzero(cand_idx[r] >= 0)
        ids, s = cand_idx[r, pos], cand_val[r, pos]
        rel, cos = row_terms(ids, s, F) if len(pos) else (None, None)
        picked = np.zeros(len(pos), bool)
        maxsim = np.full(len(pos), -np.inf)
        for t in range(keys.shape[1]):
            if picked.all():
                assert keys[r, t] == -1 and scores[r, t] == 0, (r, t, keys[r, t], scores[r, t])
                continue
            assert keys[r, t] >= 0, (r, t, "padding before the candidates ran out")
            obj = (1.0 - w) * rel if t == 0 else (1.0 - w) * rel - w * maxsim
            obj = np.where(picked, -np.inf, obj)
            same = np.flatnonzero((ids == keys[r, t]) & (s.view(np.uint32) == np.float32(scores[r, t]).view(np.uint32))
                                  & ~picked)
            assert same.size, (r, t, "pick is not an unpicked candidate")
            p = int(same[np.argmax(obj[same])])
            assert obj[p] >= obj.max() - tol, (r, t, obj[p], obj.max())
            picked[p] = True
            maxsim = np.maximum(maxsim, cos[p])


def random_inputs(n, M, d, seed, n_items=None, pad_frac=0.2, dup_frac=0.1, zero_rows=3):
    """Unconstrained candidate lists: random items (a few zero rows), scores best first, duplicates and -1 tails."""
    rng = np.random.default_rng(seed)
    n_items = n_items or max(4 * M, 64)
    F = rng.standard_normal((n_items, d)).astype(np.float32)
    F[rng.choice(n_items, size=min(zero_rows, n_items), replace=False)] = 0
    cand_idx = rng.integers(0, n_items, size=(n, M)).astype(np.int32)
    dup = rng.random((n, M)) < dup_frac
    if M > 1:
        cand_idx[:, 1:][dup[:, 1:]] = cand_idx[:, :-1][dup[:, 1:]]
    cand_val = -np.sort(-rng.standard_normal((n, M)).astype(np.float32), axis=1)
    for r in range(n):
        if rng.random() < pad_frac:
            nv = int(rng.integers(0, M + 1))
            cand_idx[r, nv:] = -1
            cand_val[r, nv:] = 0
    return cand_idx, cand_val, F

"""Batch query helpers (buffalo/parallel/base.py): ParALS / ParBPRMF, the dot_topn semantics of
buffalo/parallel/_core.hpp:88-142 (best-first indexes, -1 padded).  With a GPU the queries run on a backend.Serve
handle that keeps the item factors resident (DESIGN.md 4.9); without one, or above its limits, the NumPy
implementation below runs."""
import numpy as np
import scipy.sparse

from buffalo_b200 import backend


def quickselect(scores, result, sorted=True, num_threads=4):
    k = result.shape[1]
    part = np.argpartition(-scores, min(k, scores.shape[1]) - 1, axis=1)[:, :k]
    if sorted:
        vals = np.take_along_axis(scores, part, axis=1)
        part = np.take_along_axis(part, np.argsort(-vals, axis=1, kind="stable"), axis=1)
    result[:, :part.shape[1]] = part


def dot_topn(indexes, P, Q, Qb, out_keys, out_scores, pool, topk, num_workers=4, seen_indptr=None, seen_keys=None):
    """seen_indptr / seen_keys (optional): a CSR of END offsets whose row i holds item ids query i does not get back."""
    cand = Q if pool is None or len(pool) == 0 else Q[pool]
    scores = P[indexes].dot(cand.T)
    if Qb is not None and Qb.size:
        scores = scores + (Qb if pool is None or len(pool) == 0 else Qb[pool]).reshape(1, -1)
    if seen_indptr is not None:
        _topn_unseen(scores, Q.shape[0], pool, topk, seen_indptr, seen_keys, out_keys, out_scores)
        return
    k = min(topk, scores.shape[1])
    part = np.argpartition(-scores, k - 1, axis=1)[:, :k]
    vals = np.take_along_axis(scores, part, axis=1)
    order = np.argsort(-vals, axis=1, kind="stable")
    part, vals = np.take_along_axis(part, order, axis=1), np.take_along_axis(vals, order, axis=1)
    out_keys[:] = -1
    out_scores[:] = 0
    out_keys[:, :k] = part if pool is None or len(pool) == 0 else np.asarray(pool)[part]
    out_scores[:, :k] = vals


def _topn_unseen(scores, num_items, pool, topk, seen_indptr, seen_keys, out_keys, out_scores):
    """dot_topn's result with the seen candidates of each row left out: one stable sort on (seen, -score), so ties go
    to the smaller position and no score value marks a seen candidate; -1 / 0 pad rows left with fewer than topk."""
    n, C = scores.shape
    lens = np.diff(np.asarray(seen_indptr, dtype=np.int64), prepend=0)
    seen = np.zeros((n, num_items), dtype=bool)
    seen[np.repeat(np.arange(n), lens), np.asarray(seen_keys)[:int(lens.sum())]] = True
    if pool is not None and len(pool):
        seen = seen[:, np.asarray(pool)]
    k = min(topk, C)
    order = np.lexsort((-scores, seen), axis=-1)[:, :k]
    valid = np.arange(k)[None, :] < (C - seen.sum(axis=1))[:, None]
    out_keys[:] = -1
    out_scores[:] = 0
    out_keys[:, :k] = np.where(valid, order if pool is None or len(pool) == 0 else np.asarray(pool)[order], -1)
    out_scores[:, :k] = np.where(valid, np.take_along_axis(scores, order, axis=1), 0)


def cand_topn(indexes, P, Q, Qb, topk, cand_indptr, cand_keys, seen_indptr=None, seen_keys=None):
    """dot_topn over a candidate list per query: row i ranks only the items of row i of the CSR (END offsets), in list
    order, ties to the earlier position; with seen rows (a CSR of END offsets, row i per query) those items are left
    out.  (keys int32, scores float32) [n, topk], -1 / 0 padded; an empty list gives a padded row."""
    n = len(indexes)
    keys = np.full((n, topk), -1, dtype=np.int32)
    scores = np.zeros((n, topk), dtype=np.float32)
    cand_indptr = np.asarray(cand_indptr, dtype=np.int64)
    for i, u in enumerate(indexes):
        pool = np.asarray(cand_keys[(cand_indptr[i - 1] if i else 0):cand_indptr[i]], dtype=np.int64)
        if not pool.size:
            continue
        s = P[[u]].dot(Q[pool].T)[0]
        if Qb is not None and Qb.size:
            s = s + Qb.reshape(-1)[pool]
        order = np.argsort(-s, kind="stable")
        if seen_indptr is not None:
            row = seen_keys[(seen_indptr[i - 1] if i else 0):seen_indptr[i]]
            order = order[~np.isin(pool[order], row)]
        order = order[:topk]
        keys[i, :len(order)] = pool[order]
        scores[i, :len(order)] = s[order]
    return keys, scores


def seen_csr(algo, exclude_seen):
    """(END offsets int64, keys) of every user's seen row, as exclude_seen=... names them: the rows of the algo's
    training data ("rowwise" group) for exclude_seen=True, of a scipy sparse (num_users, num_items) matrix otherwise."""
    num_users, num_items = algo.P.shape[0], algo.Q.shape[0]
    if scipy.sparse.issparse(exclude_seen):
        m = exclude_seen.tocsr()
        if m.shape != (num_users, num_items):
            raise ValueError("exclude_seen must be a (%d, %d) matrix, got %s" % (num_users, num_items, m.shape))
        ends = np.asarray(m.indptr[1:], dtype=np.int64)
        keys = np.asarray(m.indices[:int(m.indptr[-1])])
        if keys.size and (keys.min() < 0 or keys.max() >= num_items):
            raise ValueError("exclude_seen holds a column outside [0, %d)" % num_items)
        return ends, keys
    data = getattr(algo, "data", None)
    if data is None:
        raise ValueError("exclude_seen=True needs the training data attached to the model; pass a scipy "
                         "sparse (num_users, num_items) matrix of the seen items instead")
    grp = data.get_group("rowwise")
    ends = np.asarray(grp["indptr"][:], dtype=np.int64)
    return ends, np.asarray(grp["key"][:int(ends[-1]) if len(ends) else 0])


RERANK_BATCH_BYTES = 256 << 20   # device candidate lists (ids + scores) per batch of a diversified call


def _check_diversify(diversify, candidates, topk):
    """(w, M) of topk_recommendation's diversify / diversify_candidates, or None when diversify is None; w is rounded to
    float32 as the device takes it, so both paths use the same weight.  ValueError on anything else."""
    if diversify is None:
        if candidates is not None:
            raise ValueError("diversify_candidates needs diversify")
        return None
    if isinstance(diversify, bool) or not isinstance(diversify, (int, float, np.integer, np.floating)) \
            or not 0 <= diversify <= 1:
        raise ValueError("diversify must be None or a real number in [0, 1], got %r" % (diversify,))
    if not _is_int(topk) or not 1 <= topk <= backend.MMR_MMAX:
        raise ValueError("topk must be an integer in [1, %d] with diversify, got %r" % (backend.MMR_MMAX, topk))
    if candidates is None:
        candidates = min(4 * int(topk), backend.MMR_MMAX)
    if not _is_int(candidates) or not topk <= candidates <= backend.MMR_MMAX:
        raise ValueError("diversify_candidates must be an integer in [topk, %d] = [%d, %d], got %r"
                         % (backend.MMR_MMAX, topk, backend.MMR_MMAX, candidates))
    return float(np.float32(diversify)), int(candidates)


def mmr_numpy(cand_idx, cand_val, F, topk, w):
    """The MMR re-ranking of bfl_mmr_rerank_device (DESIGN.md 4.15) in NumPy: rows of candidate ids (-1 pads) and
    their scores, item rows F (float32, bias excluded) -> (keys int32, scores float32) [n, topk], -1 / 0.0 padded.  The
    cosines are taken in fp64 from the fp32 rows, so they can differ from the device's fp32 dot products in the last
    bits."""
    cand_idx, cand_val = np.asarray(cand_idx), np.asarray(cand_val, dtype=np.float32)
    n = cand_idx.shape[0]
    keys = np.full((n, topk), -1, dtype=np.int32)
    scores = np.zeros((n, topk), dtype=np.float32)
    for r in range(n):
        pos = np.flatnonzero(cand_idx[r] >= 0)
        if not pos.size:
            continue
        ids, s = cand_idx[r, pos], cand_val[r, pos]
        s64 = s.astype(np.float64)
        lo, hi = s64.min(), s64.max()
        rel = (s64 - lo) / (hi - lo) if hi > lo else np.ones(len(pos))
        X = np.asarray(F[ids], dtype=np.float32).astype(np.float64)
        G = X @ X.T
        nrm = np.diag(G)
        ok = (nrm[:, None] > 0) & (nrm[None, :] > 0)
        with np.errstate(divide="ignore", invalid="ignore"):
            cos = np.where(ok, G / np.sqrt(nrm[:, None] * nrm[None, :]), 0.0)
        picked = np.zeros(len(pos), dtype=bool)
        maxsim = np.full(len(pos), -np.inf)
        for t in range(min(topk, len(pos))):
            obj = (1.0 - w) * rel if t == 0 else (1.0 - w) * rel - w * maxsim
            p = int(np.argmax(np.where(picked, -np.inf, obj)))   # the first of equal maxima: the smaller position
            keys[r, t], scores[r, t] = ids[p], s[p]
            picked[p] = True
            maxsim = np.maximum(maxsim, cos[p])
    return keys, scores


def _on_torch(x, dev):
    """x as a CUDA tensor on dev: a torch tensor as it is, a host array copied (an empty one as one zero)."""
    import torch
    return x if isinstance(x, torch.Tensor) else torch.from_numpy(np.ascontiguousarray(_nonempty(x))).to(dev)


def _device_stage(h, M, dev, seen=None, cands=None):
    """stage(q) -> (ids, scores) CUDA [len(q), M]: the candidate call of a serve handle whose queries are set, for the
    query rows q (int32 CUDA), which are also the rows of the seen / candidate CSRs (END offsets, keys; host arrays or
    CUDA tensors).  The pool is the handle's."""
    sv = None if seen is None else (_on_torch(seen[0], dev), _on_torch(seen[1], dev))
    if cands is not None:
        cptr, ckeys = _on_torch(cands[0], dev), _on_torch(cands[1], dev)
        return lambda q: h.topk_candidates_device(q, M, cptr, ckeys, cand_row=q,
                                                  seen=None if sv is None else (sv[0], sv[1], q))
    if sv is not None:
        return lambda q: h.topk_seen_device(q, M, sv[0], sv[1], seen_row=q)
    return lambda q: h.topk_device(q, M)


def _rerank_batches(h, n, topk, w, M, dev, stage):
    """(keys int32, scores float32) host [n, topk]: stage's M candidates of every query row reranked on the device,
    RERANK_BATCH_BYTES of candidate lists at a time (rows are independent, so the split changes nothing)."""
    import torch
    keys = np.empty((n, topk), dtype=np.int32)
    scores = np.empty((n, topk), dtype=np.float32)
    rows = max(1, RERANK_BATCH_BYTES // (8 * M))
    for b0 in range(0, n, rows):
        nb = min(rows, n - b0)
        q = torch.arange(b0, b0 + nb, dtype=torch.int32, device=dev)
        ci, cv = stage(q)
        ri, rv = h.rerank_mmr_device(ci, cv, topk, w)
        keys[b0:b0 + nb], scores[b0:b0 + nb] = ri.cpu().numpy(), rv.cpu().numpy()
    return keys, scores


def rerank_mmr(cand_idx, cand_val, item_factors, topk, diversify):
    """MMR re-ranking (DESIGN.md 4.15) of candidate lists made elsewhere, such as IVF results or another retriever:
    cand_idx an (n, m) integer array of item indexes (-1 pads, duplicates are ordinary candidates, m <= 256), cand_val
    their (n, m) scores, item_factors the (num_items, d) rows whose cosines measure similarity.  Per row, topk of the
    candidates picked greedily: at each step the largest (1 - diversify) rel - diversify max-cos-to-the-picked, rel the
    score scaled to [0, 1] over the row, ties to the earlier position.  Returns (keys int32, scores float32) [n, topk]
    in pick order, the scores as given, -1 / 0.0 once the valid candidates run out.  diversify = 0 keeps the first
    topk candidates of a best-first list.  On the GPU when one is present, in NumPy otherwise."""
    ci, cv = np.asarray(cand_idx), np.asarray(cand_val)
    if ci.ndim != 2 or not np.issubdtype(ci.dtype, np.integer) or ci.shape[1] < 1 or cv.shape != ci.shape:
        raise ValueError("cand_idx must be an (n, m) integer array with m >= 1 and cand_val of the same shape, got %s "
                         "and %s" % (ci.shape, cv.shape))
    F = np.ascontiguousarray(item_factors, dtype=np.float32)
    if F.ndim != 2 or F.shape[0] < 1 or F.shape[1] < 1:
        raise ValueError("item_factors must be a (num_items, d) array, got shape %s" % (F.shape,))
    n, m = ci.shape
    if m > backend.MMR_MMAX:
        raise ValueError("at most %d candidates per row, got %d" % (backend.MMR_MMAX, m))
    if not _is_int(topk) or not 1 <= topk <= m:
        raise ValueError("topk must be an integer in [1, %d], got %r" % (m, topk))
    w, _ = _check_diversify(diversify, m, topk)
    if ci.size and (int(ci.min()) < -1 or int(ci.max()) >= F.shape[0]):
        raise ValueError("cand_idx holds an index outside [-1, %d)" % F.shape[0])
    ci, cv = np.ascontiguousarray(ci, dtype=np.int32), np.ascontiguousarray(cv, dtype=np.float32)
    if not (backend.device_available() and n and F.shape[0] < 2 ** 31):
        return mmr_numpy(ci, cv, F, int(topk), w)
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    h = backend.Serve()
    try:
        h.set_items(F)
        tci, tcv = torch.from_numpy(ci).to(dev), torch.from_numpy(cv).to(dev)
        return _rerank_batches(h, n, int(topk), w, m, dev, lambda q: (tci[q.long()], tcv[q.long()]))
    finally:
        h.close()


CATEGORY_M0 = None                # first candidate depth of a capped call; None: min(SERVE_KMAX, max(4 topk, 64))
CATEGORY_BATCH_BYTES = 1 << 30    # device buffers (deepest candidate lists, walk state, output) per batch of rows


def _category_depth(topk):
    return CATEGORY_M0 if CATEGORY_M0 is not None else min(backend.SERVE_KMAX, max(4 * int(topk), 64))


def _is_int(x):
    return isinstance(x, (int, np.integer)) and not isinstance(x, (bool, np.bool_))


def _check_caps(categories, category_cap, rows):
    """(categories int32 [rows], caps) of a categories / category_cap pair, caps an int (one cap for every category) or
    int32 [C]; ValueError on anything else."""
    cats = np.asarray(categories)
    if cats.ndim != 1 or not np.issubdtype(cats.dtype, np.integer) or len(cats) != rows:
        raise ValueError("categories must be a 1-d integer array with one entry per item row (%d), got %s of shape %s"
                         % (rows, cats.dtype, cats.shape))
    lo, hi = (int(cats.min()), int(cats.max())) if cats.size else (-1, -1)
    if _is_int(category_cap):
        if category_cap < 0:
            raise ValueError("category_cap must be >= 0, got %d" % category_cap)
        caps = int(min(category_cap, 2 ** 31 - 1))
        ncat = hi + 1
    else:
        c = np.asarray(category_cap)
        if c.ndim != 1 or not np.issubdtype(c.dtype, np.integer) or (c.size and int(c.min()) < 0):
            raise ValueError("category_cap must be an integer >= 0 or a 1-d integer array of caps >= 0")
        caps = np.minimum(c, 2 ** 31 - 1).astype(np.int32)
        ncat = len(caps)
    if lo < -1 or hi >= max(ncat, 0):
        raise ValueError("categories must lie in [-1, %d) for this category_cap, got [%d, %d]" % (ncat, lo, hi))
    return np.ascontiguousarray(cats, dtype=np.int32), caps


def _check_categories(categories, category_cap, rows, topk, nprobe=None, diversify=None):
    """(categories int32, caps) of the categories / category_cap keywords (_check_caps, rows() of them), or None when
    neither is given; ValueError on a keyword given alone, on nprobe or diversify next to them, on a topk outside
    [1, SERVE_KMAX] and on bad values."""
    if categories is None and category_cap is None:
        return None
    if categories is None or category_cap is None:
        raise ValueError("categories and category_cap go together")
    if nprobe is not None:
        raise ValueError("nprobe does not take categories (cap_categories caps IVF results)")
    if diversify is not None:
        raise ValueError("diversify does not take categories")
    if not _is_int(topk) or not 1 <= topk <= backend.SERVE_KMAX:
        raise ValueError("topk must be an integer in [1, %d] with categories, got %r" % (backend.SERVE_KMAX, topk))
    return _check_caps(categories, category_cap, rows())


def _check_unique_pool(pool=None, cands=None):
    """ValueError when the shared pool, or a row of the per-user pools (END offsets, keys), lists an item twice: a
    capped call's deeper rounds leave out items already walked, which would drop a later copy."""
    if pool is not None and len(pool) and len(np.unique(pool)) != len(pool):
        raise ValueError("with categories, the pool must not list an item twice")
    if cands is not None and len(cands[1]):
        ends = np.asarray(cands[0], dtype=np.int64)
        keys = np.asarray(cands[1])[:int(ends[-1])]
        row = np.repeat(np.arange(len(ends)), np.diff(ends, prepend=0))
        o = np.lexsort((keys, row))
        if ((row[o][1:] == row[o][:-1]) & (keys[o][1:] == keys[o][:-1])).any():
            raise ValueError("with categories, a pool row must not list an item twice")


def category_walk_numpy(cand_idx, cand_val, categories, caps, topk):
    """The walk of bfl_category_walk_device in NumPy over whole lists: per row, in order, -1 skipped, an item accepted
    when its category is -1 or fewer than its cap of that category are accepted, until topk.  (keys int32, scores
    float32) [n, topk], -1 / 0.0 padded."""
    n = len(cand_idx)
    keys = np.full((n, topk), -1, dtype=np.int32)
    scores = np.zeros((n, topk), dtype=np.float32)
    for r in range(n):
        count, t = {}, 0
        for c, s in zip(cand_idx[r], cand_val[r]):
            if t == topk:
                break
            if c < 0:
                continue
            g = int(categories[c])
            if g >= 0:
                if count.get(g, 0) >= (caps if _is_int(caps) else caps[g]):
                    continue
                count[g] = count.get(g, 0) + 1
            keys[r, t], scores[r, t] = c, s
            t += 1
    return keys, scores


def _csr_row_triples(csr, rows):
    """(major, keys) CUDA int32 of the entries of rows `rows` (int32 CUDA) of a CUDA CSR (END offsets, keys): each
    entry with its row number."""
    import torch
    ptr, keys = csr
    r = rows.long()
    ends = ptr[r]
    starts = torch.cat([ptr.new_zeros(1), ptr[:-1]])[r]
    lens = ends - starts
    first = torch.cumsum(lens, 0) - lens
    off = torch.arange(int(lens.sum().item()), device=ptr.device) + torch.repeat_interleave(starts - first, lens)
    return torch.repeat_interleave(rows, lens), keys[off]


def _capped_batches(h, n, topk, cats, caps, dev, num_items, seen=None, cands=None, stats=None):
    """(keys int32, scores float32) host [n, topk] of the capped walk over the complete ranking of each query row of a
    serve handle whose queries (and pool) are set, with seen / candidate CSRs as _device_stage takes them (DESIGN.md
    4.18).  Per batch of rows: the candidate stage at depth M0, the walk, then rounds for the rows still short whose
    stage returned M valid candidates: the stage again at twice the depth (up to SERVE_KMAX) with seen plus every item
    walked so far left out, which is the next part of the same ranking.  stats (a list) gets (round, rows, M) per
    round."""
    import torch
    if seen is not None:
        seen = (_on_torch(seen[0], dev), _on_torch(seen[1], dev))
    if cands is not None:
        cands = (_on_torch(cands[0], dev), _on_torch(cands[1], dev))
    tcats = torch.from_numpy(cats).to(dev)
    tcaps = caps if _is_int(caps) else _on_torch(caps, dev)
    slots = backend.category_table_slots(topk)
    M0 = _category_depth(topk)
    rows_max = max(1, CATEGORY_BATCH_BYTES // (8 * backend.SERVE_KMAX + 4 * (1 + 2 * slots) + 8 * topk))
    keys = np.empty((n, topk), dtype=np.int32)
    scores = np.empty((n, topk), dtype=np.float32)
    for b0 in range(0, n, rows_max):
        nb = min(rows_max, n - b0)
        state = torch.zeros((nb, 1 + 2 * slots), dtype=torch.int32, device=dev)
        oi = torch.full((nb, topk), -1, dtype=torch.int32, device=dev)
        ov = torch.zeros((nb, topk), dtype=torch.float32, device=dev)
        q = torch.arange(b0, b0 + nb, dtype=torch.int32, device=dev)
        M, rnd = M0, 0
        ci, cv = _device_stage(h, M, dev, seen, cands)(q)
        w_row = w_item = torch.empty(0, dtype=torch.int32, device=dev)
        while True:
            rows = q - b0
            backend.category_walk_device(ci, cv, rows, tcats, tcaps, topk, state, oi, ov)
            if stats is not None:
                stats.append((rnd, len(q), M))
            more = (state[rows.long(), 0] < topk) & (ci[:, M - 1] >= 0)
            if not bool(more.any().item()):
                break
            valid = ci >= 0
            w_row = torch.cat([w_row, torch.repeat_interleave(q, valid.sum(1))])
            w_item = torch.cat([w_item, ci[valid]])
            q = q[more]
            live = torch.zeros(n, dtype=torch.bool, device=dev)
            live[q.long()] = True
            keep = live[w_row.long()]
            w_row, w_item = w_row[keep], w_item[keep]
            major, minor = w_row, w_item
            if seen is not None:
                sm, sk = _csr_row_triples(seen, q)
                major, minor = torch.cat([sm, major]), torch.cat([sk, minor])
            excl = backend.csr_from_triples_device(major, minor, torch.ones(len(major), dtype=torch.float32, device=dev),
                                                   n, num_items)[:2]
            M, rnd = min(2 * M, backend.SERVE_KMAX), rnd + 1
            ci, cv = _device_stage(h, M, dev, excl, cands)(q)
        keys[b0:b0 + nb], scores[b0:b0 + nb] = oi.cpu().numpy(), ov.cpu().numpy()
    return keys, scores


def cap_categories(cand_idx, cand_val, categories, category_cap, topk):
    """Per-category caps over ranked lists made elsewhere, such as IVF results or rerank_mmr output: cand_idx an (n, m)
    integer array of item indexes best first (-1 entries skipped), cand_val their scores, categories one integer per
    item in [-1, C) (-1: not capped), category_cap an integer >= 0 (every category's cap) or an array of C caps >= 0 (0
    bans a category).  Per row, the list is walked in order and an item kept when its category is -1 or fewer than its
    cap items of that category are kept already, until topk are kept.  Returns (keys int32, scores float32) [n, topk],
    the scores as given, -1 / 0.0 padded.  The result is exact with respect to the given lists only: an item that a
    deeper list would have brought in is not considered, so a row can come back short where the ranking it was cut
    from had more to give (topk_recommendation(categories=...) walks the complete ranking).  On the GPU when one is
    present, in NumPy otherwise."""
    ci, cv = np.asarray(cand_idx), np.asarray(cand_val)
    if ci.ndim != 2 or not np.issubdtype(ci.dtype, np.integer) or ci.shape[1] < 1 or cv.shape != ci.shape:
        raise ValueError("cand_idx must be an (n, m) integer array with m >= 1 and cand_val of the same shape, got %s "
                         "and %s" % (ci.shape, cv.shape))
    if not _is_int(topk) or topk < 1:
        raise ValueError("topk must be an integer >= 1, got %r" % (topk,))
    cats = np.asarray(categories)
    cats, caps = _check_caps(cats, category_cap, cats.shape[0] if cats.ndim == 1 else -1)
    if ci.size and (int(ci.min()) < -1 or int(ci.max()) >= len(cats)):
        raise ValueError("cand_idx holds an index outside [-1, %d)" % len(cats))
    n, m = ci.shape
    k = min(int(topk), m)
    ci, cv = np.ascontiguousarray(ci, dtype=np.int32), np.ascontiguousarray(cv, dtype=np.float32)
    keys = np.full((n, int(topk)), -1, dtype=np.int32)
    scores = np.zeros((n, int(topk)), dtype=np.float32)
    if not (backend.device_available() and n and len(cats)):
        keys[:, :k], scores[:, :k] = category_walk_numpy(ci, cv, cats, caps, k)
        return keys, scores
    import torch
    dev = torch.device("cuda", torch.cuda.current_device())
    slots = backend.category_table_slots(k)
    state = torch.zeros((n, 1 + 2 * slots), dtype=torch.int32, device=dev)
    oi = torch.full((n, k), -1, dtype=torch.int32, device=dev)
    ov = torch.zeros((n, k), dtype=torch.float32, device=dev)
    backend.category_walk_device(torch.from_numpy(ci).to(dev), torch.from_numpy(cv).to(dev), None,
                                 torch.from_numpy(cats).to(dev), caps if _is_int(caps) else _on_torch(caps, dev), k,
                                 state, oi, ov)
    keys[:, :k], scores[:, :k] = oi.cpu().numpy(), ov.cpu().numpy()
    return keys, scores


class Parallel(object):
    def __init__(self, algo, *argv, **kwargs):
        self.algo = algo
        self.num_workers = int(kwargs.get("num_workers", algo.opt.num_workers))

    @staticmethod
    def _fingerprint(*arrays):
        """Checksum of the arrays' bits, one pass over the data: the xor of all 32-bit words and the sum of the row
        sums weighted by odd row numbers (so a changed value, and rows that changed places, both show)."""
        out = []
        for x in arrays:
            if x is None:
                out.append(None)
                continue
            w = x.view(np.uint32).reshape(x.shape[0], -1)
            rows = w.sum(axis=1, dtype=np.uint64)
            out.append((x.shape, int(np.bitwise_xor.reduce(w, axis=None)),
                        int((rows * (np.arange(len(rows), dtype=np.uint64) * np.uint64(2) + np.uint64(1))).sum(dtype=np.uint64))))
        return tuple(out)

    def _serve_handle(self, B, Bb):
        """The handle holding items B (and bias Bb) on the device.  The factor arrays are the model's live arrays and
        training, normalize() or the user may rewrite them, in place or not, between two calls; so every call
        checksums them and uploads again when they differ from what is resident."""
        key = self._fingerprint(B, Bb)
        if getattr(self, "_serve_key", None) != key:
            if getattr(self, "_serve", None) is None:
                self._serve = backend.Serve()
            self._serve_key = None
            self._serve.set_items(B, Bb)
            self._serve_key = key
        return self._serve

    @staticmethod
    def _on_device(indexes, A, B, topk, queries=None):
        # On the device when one is present and the call is within the kernels' limits.  The items must fit in device
        # memory next to the gathered query rows: an allocation failure is an error, not a silent switch to NumPy.
        # Device query rows stand in for A, which is then not looked at.
        return (backend.device_available() and len(indexes) and 0 < topk <= backend.SERVE_KMAX
                and B.shape[0] < 2 ** 31
                and all(x.dtype == np.float32 and x.flags["C_CONTIGUOUS"]
                        for x in ((A, B) if queries is None else (B,))))

    @staticmethod
    def _set_queries(h, A, indexes, queries):
        """The handle's queries: the rows A[indexes], or the device rows `queries` (CUDA [len(indexes), >= d]) in their
        place."""
        if queries is not None:
            import torch
            # the host entries read the rows on the handle's own streams, which do not wait for the caller's
            torch.cuda.current_stream(queries.device).synchronize()
            h.bind_queries(queries)
        else:
            # only the rows asked for go to the device, read from the live array at every call
            h.set_queries(np.ascontiguousarray(A[indexes]))

    @staticmethod
    def _host_queries(A, indexes, queries, d):
        """(A, indexes) of the NumPy path: the device rows `queries` copied to the host in place of A[indexes]."""
        if queries is None:
            return A, indexes
        return np.ascontiguousarray(queries[:, :d].cpu().numpy()), np.arange(len(indexes), dtype=np.int32)

    def _rank(self, indexes, A, B, Bb, topk, pool=None, cands=None, seen=None, queries=None, div=None, cat=None):
        """(keys int32, scores float32) [len(indexes), topk]: query i, the row A[indexes[i]] or row i of the CUDA rows
        `queries` in its place, ranked against the items B (bias Bb).  pool: None (or empty) ranks every item, else
        the item indexes every query ranks; cands instead: (END offsets int64, keys int32) whose row i lists the items
        query i ranks.  seen: None, or (END offsets int64, keys int32; host arrays, or CUDA tensors with `queries`)
        whose row i holds the items query i must not get.  div = (w, M) of _check_diversify reranks each query's M best
        by MMR against B; cat = (categories, caps) of _check_categories walks each query's complete ranking under the
        caps (DESIGN.md 4.18).  On the device the candidates never leave it.  The NumPy path takes host seen rows
        only."""
        if Bb is not None and not Bb.size:
            Bb = None
        if pool is not None and len(pool) == 0:
            pool = None
        if self._on_device(indexes, A, B, div[1] if div is not None else _category_depth(topk) if cat is not None
                           else topk, queries):
            import torch
            h = self._serve_handle(B, None if Bb is None else np.ascontiguousarray(Bb, dtype=np.float32))
            n = len(indexes)
            dev = queries.device if queries is not None else torch.device("cuda", torch.cuda.current_device())
            try:
                self._set_queries(h, A, indexes, queries)
                h.set_pool(pool)
                if div is not None:
                    return _rerank_batches(h, n, topk, div[0], div[1], dev, _device_stage(h, div[1], dev, seen, cands))
                if cat is not None:
                    return _capped_batches(h, n, topk, *cat, dev, B.shape[0], seen, cands)
                if seen is not None and not isinstance(seen[0], np.ndarray):
                    ci, cv = _device_stage(h, topk, dev, seen, cands)(torch.arange(n, dtype=torch.int32, device=dev))
                    return ci.cpu().numpy(), cv.cpu().numpy()
                # the host entries batch the queries and overlap each batch's copy back with the next batch
                q = np.arange(n, dtype=np.int32)
                if cands is not None:
                    return h.topk_candidates(q, topk, *cands, seen=seen)
                return h.topk(q, topk) if seen is None else h.topk_seen(q, topk, *seen)
            finally:
                if queries is not None:
                    # the rows belong to the caller; every query on the handle sets its own queries first
                    h.unbind_queries()
        # NumPy: each query's ranked candidates (M of them to rerank, the complete ranking to walk), then the post-step
        A, indexes = self._host_queries(A, indexes, queries, B.shape[1])
        depth = topk if div is None else div[1]
        if cat is not None and cands is not None:
            ends = np.asarray(cands[0], dtype=np.int64)
            depth = max(1, int(np.diff(ends, prepend=0).max()) if len(ends) else 1)
        elif cat is not None:
            depth = B.shape[0] if pool is None else len(pool)
        if cands is not None:
            keys, scores = cand_topn(indexes, A, B, Bb, depth, *cands, *(seen or ()))
        else:
            keys = np.zeros((len(indexes), depth), dtype=np.int32)
            scores = np.zeros((len(indexes), depth), dtype=np.float32)
            dot_topn(indexes, A, B, Bb, keys, scores, pool, depth, self.num_workers, *(seen or ()))
        if div is not None:
            return mmr_numpy(keys, scores, B, topk, div[0])
        if cat is not None:
            return category_walk_numpy(keys, scores, *cat, topk)
        return keys, scores


class ParALS(Parallel):
    _bias = False

    def _resolve(self, keys, pool, group):
        idx = self.algo.get_index_pool(keys, group=group) if isinstance(keys, list) else keys
        kept = [k for k, i in zip(keys, idx) if i is not None]
        idx = np.array([i for i in idx if i is not None], dtype=np.int32)
        if pool is not None:
            pool = self.algo.get_index_pool(pool, group="item" if group == "user" else group)
            if len(pool) == 0:
                raise RuntimeError("pool is empty")
        return kept, idx, pool

    def build_index(self, nlist, group="item", iters=10):
        """Builds the IVF index (DESIGN.md 4.12) of the current item (algo.Q, with algo.Qb for ParBPRMF with use_bias)
        or user (algo.P) factors: spherical k-means into nlist lists, iters rounds, seeded with algo.opt.random_seed.
        topk_recommendation / most_similar with nprobe=... then search it.  It replaces the group's earlier index and
        goes stale when the factors change (normalize() included): build it again then.  On the GPU only."""
        if group not in ("item", "user"):
            raise ValueError(f"Not supported group: {group}")
        F = self.algo.Q if group == "item" else self.algo.P
        Fb = self._index_bias(group)
        if not _is_int(nlist) or not 1 <= nlist <= min(F.shape[0], backend.IVF_MAX_LISTS):
            raise ValueError("nlist must be an integer in [1, min(rows, %d)] = [1, %d], got %r"
                             % (backend.IVF_MAX_LISTS, min(F.shape[0], backend.IVF_MAX_LISTS), nlist))
        if not _is_int(iters) or iters < 1:
            raise ValueError("iters must be an integer of at least 1, got %r" % (iters,))
        F = np.ascontiguousarray(F, dtype=np.float32)
        ivf = backend.IVF()
        ivf.build(F, Fb, int(nlist), int(iters), seed=int(self.algo.opt.random_seed))
        ivf.keys = self._fingerprint(F, Fb)
        if getattr(self, "_indexes", None) is None:
            self._indexes = {}
        self._indexes[group] = ivf

    def _index_bias(self, group):
        Qb = getattr(self.algo, "Qb", None)
        if group != "item" or not self._bias or not self.algo.opt.get("use_bias") or Qb is None or not Qb.size:
            return None
        return np.ascontiguousarray(Qb, dtype=np.float32).reshape(-1)

    def _search_index(self, group, idx, A, topk, nprobe, with_bias, normalized, queries=None):
        """The IVF search of the rows A[idx] (or of the CUDA rows `queries` in their place) in the group's index; every
        check before any device work."""
        ivf = (getattr(self, "_indexes", None) or {}).get(group)
        if ivf is None:
            raise RuntimeError("no %s index: call build_index(nlist, group=%r) first" % (group, group))
        nprobe = ivf._check_nprobe(nprobe)
        topk = backend.Serve._check_k(topk)
        F = np.ascontiguousarray(self.algo.Q if group == "item" else self.algo.P, dtype=np.float32)
        now = self._fingerprint(F, self._index_bias(group) if with_bias else None)
        if now[0] != ivf.keys[0] or (with_bias and now[1] != ivf.keys[1]):
            raise RuntimeError("the %s index is stale: the factors changed since build_index; call build_index again%s"
                               % (group, " after algo.normalize(%r)" % group if normalized else ""))
        if queries is not None:
            ivf._attach()
            out = ivf.search_device(queries, nprobe, topk, use_bias=with_bias and ivf.has_bias)
            return tuple(t.cpu().numpy() for t in out)
        return ivf.search(np.ascontiguousarray(A[idx], dtype=np.float32), nprobe, topk,
                          use_bias=with_bias and ivf.has_bias)

    def most_similar(self, keys, topk=10, group="item", pool=None, repr=False, ef_search=-1, use_mmap=True,
                     nprobe=None, categories=None, category_cap=None):
        """nprobe: None ranks every row; an integer in [1, nlist] searches the group's index (build_index, after
        algo.normalize(group)) and ranks the rows of the nprobe lists nearest each query.  categories / category_cap
        as topk_recommendation takes them, one category per row of the group, without nprobe.  ef_search and use_mmap
        are accepted and ignored."""
        if nprobe is not None and pool is not None:
            raise ValueError("nprobe does not take a pool")
        if group in ("item", "user"):
            cat = _check_categories(categories, category_cap,
                                    lambda: (self.algo.Q if group == "item" else self.algo.P).shape[0], topk, nprobe)
        self.algo.normalize(group=group)
        _, idx, pool = self._resolve(keys, pool, group)
        if group not in ("item", "user"):
            raise ValueError(f"Not supported group: {group}")
        F = self.algo.Q if group == "item" else self.algo.P
        names = self.algo._idmanager.itemids if group == "item" else self.algo._idmanager.userids
        if nprobe is not None:
            topks, scores = self._search_index(group, idx, F, topk, nprobe, False, True)
        else:
            if cat is not None:
                _check_unique_pool(pool)
            topks, scores = self._rank(idx, F, F, None, topk, pool, cat=cat)
        return _names(names, topks) if repr else topks, scores

    @staticmethod
    def _pool_matrix(pool, rows, num_items):
        """(END offsets int64, keys int32) of a scipy sparse (rows, num_items) candidate matrix as tocsr() stores it:
        every row's columns in stored order, duplicates kept, values ignored.  Checks the shape and the columns."""
        m = pool.tocsr()
        if m.shape != (rows, num_items):
            raise ValueError("pool must be a (%d, %d) matrix, got %s" % (rows, num_items, m.shape))
        nnz = int(m.indptr[-1])
        keys = np.asarray(m.indices[:nnz])
        if keys.size and (int(keys.min()) < 0 or int(keys.max()) >= num_items):
            raise ValueError("pool holds a column outside [0, %d)" % num_items)
        return np.asarray(m.indptr[1:], dtype=np.int64), np.ascontiguousarray(keys, dtype=np.int32)

    def _seen_rows(self, idx, exclude_seen):
        """(END offsets int64, keys int32) of the seen rows of users idx (seen_csr)."""
        from buffalo_b200.evaluate.device import _gather_rows
        return _gather_rows(*seen_csr(self.algo, exclude_seen), idx)

    def _check_explore(self, explore, explore_seed):
        """(scale, seed) of explore / explore_seed, or None when explore is None; ValueError on bad values and
        NotImplementedError for models without a least-squares posterior, before any device work."""
        from buffalo_b200.algo import fold_in
        args = fold_in.posterior_args(0.0 if explore is None else explore, explore_seed, "explore", "explore_seed")
        if explore is None:
            return None
        if not callable(getattr(self.algo, "posterior_sample", None)):
            raise NotImplementedError("explore needs a least-squares model (ALS), not %s" % type(self.algo).__name__)
        return args

    def _training_data(self, what):
        data = getattr(self.algo, "data", None)
        if data is None:
            raise ValueError("%s needs the training data attached to the model" % what)
        return data

    def _training_rows(self, idx, what):
        """scipy CSR (len(idx), num_items) of users idx's rows of the algo's training data ("rowwise" group, keys and
        values): only those rows' entries are gathered."""
        from buffalo_b200.evaluate.device import _gather_positions
        grp = self._training_data(what).get_group("rowwise")
        ends = np.asarray(grp["indptr"][:], dtype=np.int64)
        nnz = int(ends[-1]) if len(ends) else 0
        out_ptr, pos = _gather_positions(ends, idx)
        keys = np.asarray(grp["key"][:nnz])[pos]
        vals = np.asarray(grp["val"][:nnz], dtype=np.float32)[pos]
        return scipy.sparse.csr_matrix((vals, keys, np.concatenate([[0], out_ptr])),
                                       shape=(len(out_ptr), self.algo.Q.shape[0]))

    def _explore_rows(self, idx, explore):
        """CUDA [len(idx), vdim]: posterior_sample of the training rows of users idx around P[idx], draw key = user
        index.  A user listed twice is sampled once and gets the same row at both places."""
        idx = np.asarray(idx, dtype=np.int64)
        users, where = np.unique(idx, return_inverse=True)
        rows = self.algo._posterior_sample_device(self._training_rows(users, "explore"),
                                                  self.algo.P[users, :self.algo.opt.d], *explore, draw_keys=users)
        if np.array_equal(users, idx):
            return rows
        import torch
        return rows[torch.from_numpy(where.reshape(-1)).to(rows.device)]

    def topk_recommendation(self, keys, topk=10, pool=None, repr=False, exclude_seen=False, nprobe=None,
                            diversify=None, diversify_candidates=None, explore=None, explore_seed=0, categories=None,
                            category_cap=None):
        """pool: None ranks every item; a list of item ids (or an index array) is one candidate pool for every user; a
        scipy sparse (num_users, num_items) matrix gives each user its own candidates, row u (as tocsr() stores it,
        values ignored, duplicates kept, ties to the earlier entry): a user's row of the result is then what a call
        with that user alone and that row as the pool returns.  An empty row gives a row of -1 / 0.0; topk must be in
        [1, 4096].  exclude_seen: False; True to leave out each user's training items (the "rowwise" rows of the algo's
        data); or a scipy sparse (num_users, num_items) matrix whose row u lists the items user u does not get back.
        Rows left with fewer than topk candidates are padded with -1 / 0.0.  nprobe: None ranks every item; an integer
        in [1, nlist] searches the item index (build_index) and ranks the items of the nprobe lists nearest each user,
        without pool or exclude_seen.  diversify: None ranks by score; a real number w in [0, 1] reranks each user's
        diversify_candidates best candidates (M, default min(4 topk, 256), in [topk, 256]) by Maximal Marginal
        Relevance (DESIGN.md 4.15): topk picks, each the candidate of the largest (1 - w) relevance - w largest cosine
        of its item factors to the picks before it, with the candidates' scores (not sorted).  Every candidate stage
        above takes it, nprobe does not (rerank_mmr reranks IVF results); w = 0 gives the plain result.

        explore: None ranks with P[u]; a finite real sigma >= 0 ranks with one Thompson-sampling draw per user instead,
        algo.posterior_sample(user u's training row, mean P[u], scale=sigma, seed=explore_seed, draw key u) (DESIGN.md
        4.17): P[u] moved within the Gaussian posterior of the user row that the least-squares objective implies, with
        sigma^2 its noise variance.  Smaller sigma explores less; 0 gives the plain result.  A user's draw depends only on
        explore_seed (an integer in [0, 2^32)) and the user, not on the batch, so a fresh seed per impression gives fresh
        lists.  Every mode above takes it, pool, exclude_seen, diversify and nprobe included; the draws stay on the
        device.  ALS only, with its training data attached; on the GPU only.

        categories / category_cap: None, or both: categories a 1-d integer array with one category in [-1, C) per item
        row (algo.Q.shape[0], items of add_items included; -1: not capped), category_cap an integer >= 0 (the cap of
        every category, C = max(categories) + 1) or an integer array of C caps >= 0 (0 bans a category).  Each row is
        then the walk of the user's complete ranking (what this call without them returns at topk = the number of
        candidates: pool, per-user pool, exclude_seen, explore and bias included), in order, that accepts an item when
        its category is -1 or fewer than its cap items of that category are accepted already, until topk (DESIGN.md
        4.18), with that ranking's keys and score bits, -1 / 0.0 padded when it runs out.  Not with nprobe or diversify
        (cap_categories caps lists made elsewhere); a pool must not list an item twice; topk in [1, 4096]."""
        div = _check_diversify(diversify, diversify_candidates, topk)
        cat = _check_categories(categories, category_cap, lambda: self.algo.Q.shape[0], topk, nprobe, diversify)
        exp = self._check_explore(explore, explore_seed)
        if nprobe is not None:
            if div is not None:
                raise ValueError("nprobe does not take diversify")
            if pool is not None:
                raise ValueError("nprobe does not take a pool")
            if scipy.sparse.issparse(exclude_seen) or exclude_seen:
                raise ValueError("nprobe does not take exclude_seen")
        if self.algo.opt._nrz_P or self.algo.opt._nrz_Q:
            raise RuntimeError("Cannot make topk recommendation with normalized factors")
        Qb = self.algo.Qb if self._bias and self.algo.opt.get("use_bias") else None
        if exp is not None:
            self._training_data("explore")
        cands = None
        if scipy.sparse.issparse(pool):
            kept, idx, _ = self._resolve(keys, None, "user")
            topk = backend.Serve._check_k(topk)
            from buffalo_b200.evaluate.device import _gather_rows
            cands = _gather_rows(*self._pool_matrix(pool, self.algo.P.shape[0], self.algo.Q.shape[0]), idx)
            pool = None
        else:
            kept, idx, pool = self._resolve(keys, pool, "user")
        if cat is not None:
            _check_unique_pool(pool, cands)
        seen = self._seen_rows(idx, exclude_seen) if nprobe is None and (
            scipy.sparse.issparse(exclude_seen) or exclude_seen) else None
        q = None if exp is None else self._explore_rows(idx, exp)
        if nprobe is not None:
            topks, scores = self._search_index("item", idx, self.algo.P, topk, nprobe,
                                               self._index_bias("item") is not None, False, queries=q)
        else:
            topks, scores = self._rank(idx, self.algo.P, self.algo.Q, Qb, topk, pool, cands, seen, q, div, cat)
        return kept, _names(self.algo._idmanager.itemids, topks) if repr else topks, scores

    def fold_in_recommendation(self, histories, topk=10, pool=None, exclude_seen=True, repr=False, diversify=None,
                               diversify_candidates=None, explore=None, explore_seed=0, categories=None,
                               category_cap=None):
        """(topks, scores), one row per history row, for users folded into the model (DESIGN.md 4.10): the rows of
        algo.fold_in(histories) with its defaults, ranked against the items as topk_recommendation ranks (pools, -1 / 0.0
        padding).  pool may also be a scipy sparse (n, num_items) matrix: row i lists history row i's own candidates,
        as topk_recommendation takes a per-user pool.  exclude_seen: leave each row's history items out.  All on the device: the folded rows are bound as the
        serve handle's queries and never reach the host.  diversify / diversify_candidates as topk_recommendation takes
        them: the folded rows' candidates are reranked on the device too.  Models with fold_in: ALS and PLSI.
        explore / explore_seed as topk_recommendation takes them (ALS only): each folded row is replaced on the device by
        algo.posterior_sample of its history around it, with draw key = its history row index.  categories /
        category_cap as topk_recommendation takes them: each row walks the folded row's complete ranking."""
        if not callable(getattr(self.algo, "_fold_in_device", None)):
            raise NotImplementedError("fold_in_recommendation needs a model with fold_in (ALS, PLSI), not %s"
                                      % type(self.algo).__name__)
        div = _check_diversify(diversify, diversify_candidates, topk)
        cat = _check_categories(categories, category_cap, lambda: self.algo.Q.shape[0], topk, None, diversify)
        exp = self._check_explore(explore, explore_seed)
        if exp is not None and self.algo.opt.d > self.algo.EXPLAIN_DMAX:
            raise ValueError("explore supports d <= %d, got %d" % (self.algo.EXPLAIN_DMAX, self.algo.opt.d))
        topk = backend.Serve._check_k(topk)
        cands = None
        if scipy.sparse.issparse(pool):
            if not (scipy.sparse.issparse(histories) or isinstance(histories, (list, tuple))):
                raise ValueError("histories must be a scipy sparse matrix or a list of lists of item ids, got %s"
                                 % type(histories).__name__)
            n_hist = histories.shape[0] if scipy.sparse.issparse(histories) else len(histories)
            cands = self._pool_matrix(pool, n_hist, self.algo.Q.shape[0])
            pool = None
        elif pool is not None:
            pool = self.algo.get_index_pool(pool, group="item")
            if len(pool) == 0:
                raise RuntimeError("pool is empty")
        if cat is not None:
            _check_unique_pool(pool, cands)
        tX, (indptr, keys, vals) = self.algo._fold_in_device(histories)
        n = tX.shape[0]
        if n == 0:
            return np.zeros((0, topk), np.int32), np.zeros((0, topk), np.float32)
        if exp is not None:
            import torch
            from buffalo_b200.algo import fold_in
            from buffalo_b200.backend import CuALS
            st, fh = fold_in.resident_state(self.algo, CuALS)
            tX = self.algo._sample_rows(st, fh, (indptr, keys, vals), tX,
                                        torch.arange(n, dtype=torch.int64, device=tX.device), seed=exp[1], scale=exp[0])
        # the folded rows and the history CSR stay on the device, so _rank takes its device path
        Q = np.ascontiguousarray(self.algo.Q, dtype=np.float32)
        topks, scores = self._rank(np.arange(n, dtype=np.int32), None, Q, None, topk, pool, cands,
                                   (indptr, keys) if exclude_seen else None, tX, div, cat)
        return _names(self.algo._idmanager.itemids, topks) if repr else topks, scores

    def explain(self, keys, items, topm=5, repr=False):
        """(scores, keys, contributions) of algo.explain (DESIGN.md 4.11) for trained users: their histories are their
        rows of the training data ("rowwise" group, keys and values).  keys: user ids (a list) or user indexes (an
        array); every one must resolve.  items as algo.explain takes them, so the keys and topks that
        topk_recommendation returns can be passed straight in.  repr=True returns the explaining items as item ids,
        without the -1 padding.  Models with explain: ALS (a score is a sum of per-item terms only for least-squares
        rows)."""
        if not callable(getattr(self.algo, "explain", None)):
            raise NotImplementedError("explain needs a least-squares model (ALS), not %s" % type(self.algo).__name__)
        num_users = self.algo.P.shape[0]
        if isinstance(keys, list):
            idx = self.algo.get_index(keys, group="user") if keys else []
            missing = [k for k, i in zip(keys, idx) if i is None]
            if missing:
                raise ValueError("unknown user keys: %s" % missing[:5])
            idx = np.asarray(idx, dtype=np.int64)
        else:
            idx = np.asarray(keys)
            if idx.ndim != 1 or (idx.size and not np.issubdtype(idx.dtype, np.integer)):
                raise ValueError("keys must be a list of user ids or a 1-d array of user indexes")
            if idx.size and (int(idx.min()) < 0 or int(idx.max()) >= num_users):
                raise ValueError("user index outside [0, %d)" % num_users)
        scores, out_keys, contrib = self.algo.explain(self._training_rows(idx, "explain"), items, topm)
        if repr:
            out_keys = [_names(self.algo._idmanager.itemids, row) for row in out_keys]
        return scores, out_keys, contrib


class ParBPRMF(ParALS):
    _bias = True


def _nonempty(a):
    """a, or one zero when a is empty (a device array handed to the library holds at least one element)."""
    return a if a.size else np.zeros(1, a.dtype)


def _names(names, topks):
    """repr=True's rows: each row of indexes topks as names[index], the -1 padding dropped."""
    return [[names[t] for t in tt if t != -1] for tt in topks]


def _unsupported(name):
    def ctor(*a, **k):
        raise NotImplementedError(name + " is outside the H100 hot-path scope")
    return ctor


ParW2V = _unsupported("ParW2V")
ParCFR = _unsupported("ParCFR")

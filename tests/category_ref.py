"""Plain-Python reference of the per-category cap walk (DESIGN.md 4.18): over each row of a given ranking, in order,
take an item when its category is -1 or fewer than the category's cap items of it are taken already, until topk are
taken.  Shares no code with buffalo_b200."""
import numpy as np


def cap_of(cap, g):
    return int(cap) if np.ndim(cap) == 0 else int(cap[g])


def walk(ranked, scores, categories, cap, topk):
    """ranked / scores: rows of item ids best first (-1 skipped) and their scores -> (keys int32, scores float32)
    [n, topk], -1 / 0.0 padded."""
    ranked = np.asarray(ranked)
    scores = np.asarray(scores, dtype=np.float32)
    out_k = np.full((len(ranked), topk), -1, dtype=np.int32)
    out_s = np.zeros((len(ranked), topk), dtype=np.float32)
    for r in range(len(ranked)):
        taken = {}
        picked = []
        for item, s in zip(ranked[r].tolist(), scores[r]):
            if len(picked) == topk:
                break
            if item == -1:
                continue
            g = int(categories[item])
            if g != -1:
                if taken.get(g, 0) >= cap_of(cap, g):
                    continue
                taken[g] = taken.get(g, 0) + 1
            picked.append((item, s))
        for t, (item, s) in enumerate(picked):
            out_k[r, t] = item
            out_s[r, t] = s
    return out_k, out_s

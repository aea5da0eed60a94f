"""float32 NumPy restatement of the BPRMF / WARP item fold-in (DESIGN.md 4.16, sgd_fold_in_items_kernel), row by row
in CSR order with the kernel's Philox keys, so its draws can be compared exactly and its rows to 1e-5.

Dot products follow the kernel's order: each float4 slice summed left to right, slices added per lane in slice order,
then the lanes by the xor butterfly (no fused multiply-adds here, hence the tolerance)."""
import math

import numpy as np

FOLD_DOMAIN = 0xF01D0000
M32 = 0xFFFFFFFF
f32 = np.float32


def philox(c, k):
    """Philox4x32-10 (Salmon et al., SC'11) on counter c[4] and key k[2]."""
    c, k = list(c), list(k)
    for _ in range(10):
        p0 = 0xD2511F53 * c[0]
        p1 = 0xCD9E8D57 * c[2]
        c = [((p1 >> 32) ^ c[1] ^ k[0]) & M32, p1 & M32, ((p0 >> 32) ^ c[3] ^ k[1]) & M32, p0 & M32]
        k = [(k[0] + 0x9E3779B9) & M32, (k[1] + 0xBB67AE85) & M32]
    return c


def draw_u32(seed, epoch, idx, t):
    return philox([idx & M32, idx >> 32, t >> 2, epoch & M32], [seed & M32, 0x5EED])[t & 3]


def draw_range(seed, epoch, idx, t, rng):
    return (draw_u32(seed, epoch, idx, t) * rng) >> 32


def warp_sum(terms4):
    """terms4: float32 [nv4, 4] per-column terms; the kernel's lane partials and butterfly."""
    e = ((terms4[:, 0] + terms4[:, 1]) + terms4[:, 2]) + terms4[:, 3]
    lanes = np.zeros(32, f32)
    for c in range(len(e)):
        lanes[c % 32] = lanes[c % 32] + e[c]
    idx = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        lanes = lanes + lanes[idx ^ o]
    return lanes[0]


def score(p, q, l2):
    if l2:
        diff = p - q
        return -warp_sum((diff * diff).reshape(-1, 4))
    return warp_sum((p * q).reshape(-1, 4))


def pad4(A):
    A = np.asarray(A, f32)
    w = (A.shape[1] + 3) // 4 * 4
    out = np.zeros((A.shape[0], w), f32)
    out[:, :A.shape[1]] = A
    return out


def row(indptr, r):
    return (0 if r == 0 else int(indptr[r - 1])), int(indptr[r])


def bpr_negative(o, epoch, sid, seen, num_items, cum):
    t = 0
    while True:
        if cum is None:
            neg = draw_range(o["random_seed"], epoch, sid, t, num_items)
        else:
            tot = int(cum[-1])
            r64 = (draw_u32(o["random_seed"], epoch, sid, 2 * t) << 32) | draw_u32(o["random_seed"], epoch, sid, 2 * t + 1)
            neg = min(int(np.searchsorted(cum, (r64 * tot) >> 64, side="left")), num_items - 1)
        if not o.get("verify_neg", True) or neg not in seen:
            return neg
        if t >= 64:
            return neg
        t += 1


def warp_draw(o, epoch, sid, seen, num_items, p, ui, Q, l2):
    trial, t, neg, uj = 1, 0, 0, f32(0)
    max_trials, threshold = o.get("max_trials", 500), f32(o.get("threshold", 1.0))
    while trial <= max_trials:
        neg = draw_range(o["random_seed"], epoch, sid, t, num_items)
        t += 1
        if neg in seen:
            if t > 64 * max_trials + 4096:
                trial = max_trials + 1
                break
            continue
        trial += 1
        uj = score(p, Q[neg], l2)
        if f32(ui - uj) < threshold:
            break
        trial += 1
    return trial, neg, uj


def step(o, th, g, m, v, cnt, reg, bc1):
    """sgd_apply_kernel's element step; returns (theta, step kept in the accumulator, m, v)."""
    b1, omb1, lr0 = f32(o.get("beta1", 0.9)), f32(1.0 - o.get("beta1", 0.9)), f32(o.get("lr", 0.05))
    s = g
    if o.get("per_coordinate_normalize", False) and cnt:
        s = s / f32(cnt)
    s = s - th * (f32(2) * f32(reg))
    if o["optimizer"] == "adam":
        m = b1 * m + omb1 * s
        v = b1 * v + omb1 * (s * s)
        s = (m / bc1) / (np.sqrt(v / bc1) + f32(1e-10))
    else:
        v = v + s * s
        s = s / (np.sqrt(v) + f32(1e-10))
    return th + lr0 * s, s, m, v


def fold_in_items(kind, o, P, Q, Qb, train_indptr, train_keys, cum, indptr, users, X0, Xb0, epochs):
    """Returns (rows float32 [n, d], bias float32 [n], negatives int32 [epochs, nnz * per], WARP trials int32
    [epochs, nnz] or None).  o: the model's options (dict); P, Q: [rows, d]; Qb: [Q rows]; END-offset CSRs."""
    d = X0.shape[1]
    warp = kind == "warp"
    P, Q, X = pad4(P), pad4(Q), pad4(X0)
    Qb = np.asarray(Qb, f32).reshape(-1)
    Xb = np.asarray(Xb0, f32).copy()
    num_items = Q.shape[0]
    per = 1 if warp else max(int(o.get("num_negative_samples", 1)), 1)
    nnz = len(users)
    negs = np.full((epochs, nnz * per), -2, np.int32)
    trials = np.zeros((epochs, nnz), np.int32) if warp else None
    l2 = warp and str(o.get("score_func", "dot")).lower() == "l2"
    use_bias = (not warp) and o.get("use_bias", True)
    reg_i, reg_b = f32(o.get("reg_i", 0.0)), f32(o.get("reg_b", 0.0))
    lr0, min_lr = float(o.get("lr", 0.05)), float(o.get("min_lr", 0.0001))
    for r in range(X.shape[0]):
        hb, he = row(indptr, r)
        x, xb = X[r].copy(), f32(Xb[r])
        g, m, v = np.zeros_like(x), np.zeros_like(x), np.zeros_like(x)
        gb = mb = vb = f32(0)
        b1pow = 1.0
        for e in range(epochs):
            epoch = FOLD_DOMAIN + e
            lr = f32(max(lr0 - (lr0 - min_lr) * (e * (1.0 / epochs)), min_lr))
            cnt = 0
            for it in range(hb, he):
                u = int(users[it])
                ub, ue = row(train_indptr, u)
                seen = set(int(k) for k in train_keys[ub:ue])
                p = P[u]
                sid0 = (r << 32) + (it - hb) * per
                if warp:
                    ui = score(p, x, l2)
                    trial, neg, uj = warp_draw(o, epoch, sid0, seen, num_items, p, ui, Q, l2)
                    discard = trial >= o.get("max_trials", 500)
                    negs[e, it] = -1 if discard else neg
                    trials[e, it] = 0 if discard else trial
                    if discard:
                        continue
                    ratio = max(int((num_items - (ue - ub) - 1) / trial), 1)
                    phi = f32(math.log(ratio))
                    di = phi * (p - x) if l2 else phi * p
                    g = g + (di - reg_i * x)
                    cnt += 1
                else:
                    for s in range(per):
                        neg = bpr_negative(o, epoch, sid0 + s, seen, num_items, cum)
                        negs[e, it * per + s] = neg
                        xs = warp_sum((p * (x - Q[neg])).reshape(-1, 4))
                        if use_bias:
                            xs = xs + (xb - Qb[neg])
                        logit = f32(0) if xs > 6 else (f32(1) if xs < -6 else f32(1) / (f32(1) + np.exp(xs)))
                        if o["optimizer"] == "sgd":
                            x = x + lr * (logit * p - reg_i * x)
                            if use_bias:
                                xb = xb + lr * (logit - reg_b * xb)
                        else:
                            g = g + logit * p
                            gb = gb + logit
                    cnt += 1
            if o["optimizer"] != "sgd":
                b1pow *= o.get("beta1", 0.9)
                bc1 = f32(1.0 - b1pow)
                x, g, m, v = step(o, x, g, m, v, cnt, reg_i, bc1)
                if use_bias:
                    xb, gb, mb, vb = step(o, xb, gb, mb, vb, cnt, reg_b, bc1)
            if warp:
                nrm = np.sqrt(warp_sum((x * x).reshape(-1, 4)))
                if nrm > 1:
                    x = x / nrm
        X[r], Xb[r] = x, xb
    return X[:, :d].astype(f32), Xb.astype(f32), negs, trials

"""References for the device CSR sort of csrc/ingest.cu (test infrastructure only; the product never imports this
module).

``known_answer`` builds the sorted (major, minor) sequence directly -- per-major counts, then non-decreasing minors
inside every major run, with duplicate keys on purpose -- and permutes it into the input, so the answer is known
without sorting.  ``check_csr_sort`` decides in O(n) whether (indptr, key, payload) is *the* stable sort of an input
whose payload is its input position: every entry sits in the right major and carries its own key, the payload is a
permutation, keys ascend and the payload ascends inside every run of equal keys.  Both are torch integer code that runs
on the CPU or on the device and shares nothing with the kernel.  ``numpy_csr`` is the host build the data layer uses
below its device threshold (np.lexsort).
"""
import numpy as np
import torch


def numpy_csr(major, minor, vals, num_major, stable_sort):
    order = np.lexsort((minor, major)) if stable_sort else np.argsort(major, kind="stable")
    indptr = np.cumsum(np.bincount(major, minlength=num_major)).astype(np.int64)
    return indptr, minor[order].astype(np.int32), vals[order].astype(np.float32)


def positions(n, device):
    """float32 payload whose bits are the input position (exact for every n < 2^31, unlike float values)."""
    return torch.arange(n, dtype=torch.int32, device=device).view(torch.float32)


def edge_draws(num, n, gen, device):
    """n indices in [0, num): a third at 0, a third at num - 1, a third uniform -- so the top digit pass decides."""
    r = torch.randint(0, 3, (n,), generator=gen, device=device)
    u = torch.randint(0, num, (n,), generator=gen, device=device)
    return torch.where(r == 0, 0, torch.where(r == 1, num - 1, u))


def counts_of(draws, num_major):
    """int64 per-major counts of a tensor of major indices."""
    return torch.bincount(draws.to(torch.int64), minlength=num_major)


def sorted_minors(counts, num_minor, mode, gen, step=4):
    """int32 minors in [0, num_minor), non-decreasing inside every major run of `counts`.

    mode "spread": over the whole range; "edges": a third of each run at 0, a third at num_minor - 1, the rest spread
    between; "two": half at 0, half at num_minor - 1; an int: every minor equals it.  Inside a run the minors follow
    the run's cumulative sum x of random increments in [0, step) (0 repeats the key), mapped monotonically from
    [0, x_last] onto the range; all in int64, exact while 3 * step * n * num_minor < 2^63.
    """
    dev = counts.device
    n = int(counts.sum())
    if isinstance(mode, int) or n == 0:
        return torch.full((n,), 0 if n == 0 else mode, dtype=torch.int32, device=dev)
    c = torch.cumsum(torch.randint(0, step, (n,), generator=gen, device=dev), 0)
    ends = torch.cumsum(counts, 0)
    starts = ends - counts
    before = torch.where(starts > 0, c[(starts - 1).clamp(min=0)], 0)
    last = c[(ends - 1).clamp(min=0)]
    x = c - torch.repeat_interleave(before, counts, output_size=n)
    span = torch.repeat_interleave(last - before, counts, output_size=n) + 1        # x < span
    top = num_minor - 1
    if mode == "spread":
        m = x * num_minor // span
    elif mode == "edges":
        t = 3 * x
        m = torch.where(t < span, 0, torch.where(t >= 2 * span, top, (t - span) * num_minor // span))
    elif mode == "two":
        m = torch.where(2 * x < span, 0, top)
    else:
        raise ValueError(mode)
    return m.to(torch.int32)


def major_sequence(counts):
    """int32 major index of every sorted position."""
    n = int(counts.sum())
    return torch.repeat_interleave(torch.arange(counts.numel(), dtype=torch.int32, device=counts.device), counts,
                                   output_size=n)


def known_answer(counts, num_minor, minors, gen, order="shuffle"):
    """(major, minor, want_minor): input triples (int32) whose sort by (major, minor) has `counts` per major and the
    minors want_minor.  order: "shuffle" (seeded permutation), "sorted" (the answer itself) or "reversed"."""
    want_major = major_sequence(counts)
    want_minor = sorted_minors(counts, num_minor, minors, gen)
    n = want_major.numel()
    if order == "shuffle":
        perm = torch.randperm(n, generator=gen, device=counts.device)
    elif order == "sorted":
        perm = torch.arange(n, device=counts.device)
    elif order == "reversed":
        perm = torch.arange(n - 1, -1, -1, device=counts.device)
    else:
        raise ValueError(order)
    return want_major[perm].contiguous(), want_minor[perm].contiguous(), want_minor


def check_csr_sort(major, minor, indptr, key, payload, counts, sort_minor=True, want_minor=None):
    """Raise AssertionError unless (indptr, key, payload) is the stable CSR build of the input (major, minor) whose
    payload was positions(n): sorted by (major, minor), or by major alone when not sort_minor, equal keys in input
    order.  These conditions determine the output, so passing them is exact equality with the true answer."""
    n = major.numel()
    assert indptr.shape == counts.shape and torch.equal(indptr, torch.cumsum(counts, 0)), "indptr != cumsum(counts)"
    assert key.numel() == n and payload.numel() == n, "output length"
    if n == 0:
        return
    p = payload.contiguous().view(torch.int32).to(torch.int64)
    assert bool(((p >= 0) & (p < n)).all()), "payload is not an input position"
    hit = torch.zeros(n, dtype=torch.bool, device=p.device)
    hit[p] = True
    assert bool(hit.all()), "payload is not a permutation of the input positions"
    out_major = major_sequence(counts)
    assert torch.equal(major[p], out_major), "an entry sits in the wrong major"
    assert torch.equal(minor[p], key), "a key does not travel with its payload"
    same = out_major[1:] == out_major[:-1]
    if sort_minor:
        assert not bool((same & (key[1:] < key[:-1])).any()), "keys descend inside a major"
        same &= key[1:] == key[:-1]
    assert not bool((same & (p[1:] <= p[:-1])).any()), "equal keys are out of input order (unstable)"
    if want_minor is not None:
        assert torch.equal(key, want_minor), "keys differ from the constructed sequence"

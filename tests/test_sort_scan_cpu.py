"""The references of tests/test_sort_scan_gpu.py, without a GPU: the known-answer generator of tests/sort_ref.py agrees
with np.lexsort, and the O(n) checker accepts exactly the stable sort -- it rejects an unstable, misordered or
mis-indexed output, so the device tests cannot pass vacuously."""
import numpy as np
import pytest
import torch

from tests.sort_ref import (check_csr_sort, counts_of, edge_draws, known_answer, numpy_csr, positions, sorted_minors)


def lexsort_answer(major, minor, num_major, sort_minor):
    """The reference output for a torch input with position payload: (indptr, key, payload) as torch tensors."""
    mj, mn = major.numpy(), minor.numpy()
    ind, key, val = numpy_csr(mj, mn, positions(len(mj), "cpu").numpy(), num_major, sort_minor)
    return torch.from_numpy(ind), torch.from_numpy(key), torch.from_numpy(val)


@pytest.mark.parametrize("order", ["shuffle", "sorted", "reversed"])
@pytest.mark.parametrize("minors", ["spread", "edges", "two", 7])
@pytest.mark.parametrize("num_major,num_minor,n", [(1, 1, 50), (2, 2, 300), (257, 65537, 5000), (40, 3, 2000),
                                                   (5000, 1 << 24, 800), (3, 2 ** 31 - 1, 4000), (100, 10, 0)])
def test_known_answer_matches_lexsort(num_major, num_minor, n, minors, order):
    gen = torch.Generator().manual_seed(num_major + n)
    counts = counts_of(edge_draws(num_major, n, gen, "cpu"), num_major)
    minors = min(minors, num_minor - 1) if isinstance(minors, int) else minors
    major, minor, want_minor = known_answer(counts, num_minor, minors, gen, order)
    assert major.dtype == minor.dtype == torch.int32 and major.numel() == n
    if n:
        assert int(minor.min()) >= 0 and int(minor.max()) < num_minor and int(major.max()) < num_major
    for sort_minor in (True, False):
        ind, key, val = lexsort_answer(major, minor, num_major, sort_minor)
        assert torch.equal(ind, torch.cumsum(counts, 0))
        if sort_minor:
            assert torch.equal(key, want_minor)
        check_csr_sort(major, minor, ind, key, val, counts, sort_minor, want_minor if sort_minor else None)


def test_edge_modes_reach_the_ends():
    """"edges" puts keys at 0 and num - 1 with others between; "two" only at the ends: the top digit pass decides."""
    gen = torch.Generator().manual_seed(1)
    counts = torch.tensor([0, 3000, 1, 0, 2000], dtype=torch.int64)
    top = (1 << 24)
    for mode, want in (("edges", None), ("two", {0, top})):
        m = sorted_minors(counts, top + 1, mode, gen)
        run = m[:3000]
        assert int(run[0]) == 0 and int(run[-1]) == top
        assert bool((run[1:] >= run[:-1]).all())
        if want is not None:
            assert set(m.tolist()) == want
        else:
            assert int(((run > 0) & (run < top)).sum()) > 500
    d = edge_draws(1 << 24 | 1, 30000, gen, "cpu")
    assert int((d == 0).sum()) > 9000 and int((d == 1 << 24).sum()) > 9000


def test_hand_written_cases():
    """Duplicates, empty rows, n = 0 and sort_minor = 0 against a hand-computed answer."""
    major = torch.tensor([3, 0, 3, 3, 0, 3, 0], dtype=torch.int32)
    minor = torch.tensor([5, 2, 1, 5, 2, 0, 9], dtype=torch.int32)
    counts = torch.tensor([3, 0, 0, 4, 0], dtype=torch.int64)            # rows 1, 2 and 4 empty
    ind, key, val = lexsort_answer(major, minor, 5, True)
    assert ind.tolist() == [3, 3, 3, 7, 7]
    assert key.tolist() == [2, 2, 9, 0, 1, 5, 5]
    assert val.view(torch.int32).tolist() == [1, 4, 6, 5, 2, 0, 3]       # duplicates (0, 2), (3, 5) in input order
    check_csr_sort(major, minor, ind, key, val, counts, True, torch.tensor([2, 2, 9, 0, 1, 5, 5], dtype=torch.int32))
    ind, key, val = lexsort_answer(major, minor, 5, False)
    assert key.tolist() == [2, 2, 9, 5, 1, 5, 0]                         # input order inside a major
    assert val.view(torch.int32).tolist() == [1, 4, 6, 0, 2, 3, 5]
    check_csr_sort(major, minor, ind, key, val, counts, False)
    empty = torch.zeros(0, dtype=torch.int32)
    check_csr_sort(empty, empty, torch.zeros(4, dtype=torch.int64), empty, empty.view(torch.float32),
                   torch.zeros(4, dtype=torch.int64))


def _swap(t, i, j):
    t = t.clone()
    t[[i, j]] = t[[j, i]]
    return t


def test_checker_rejects_wrong_outputs():
    major = torch.tensor([1, 0, 1, 1, 0, 1, 0, 1], dtype=torch.int32)
    minor = torch.tensor([4, 2, 4, 3, 2, 4, 1, 3], dtype=torch.int32)
    counts = torch.tensor([3, 5], dtype=torch.int64)
    ind, key, val = lexsort_answer(major, minor, 2, True)
    # sorted: (0,1)p6 (0,2)p1 (0,2)p4 | (1,3)p3 (1,3)p7 (1,4)p0 (1,4)p2 (1,4)p5
    p = val.view(torch.int32)
    assert p.tolist() == [6, 1, 4, 3, 7, 0, 2, 5]
    check_csr_sort(major, minor, ind, key, val, counts, True)
    bad = {
        "unstable": (ind, key, _swap(p, 1, 2)),                       # equal keys, payloads swapped
        "unstable in the last run": (ind, key, _swap(p, 5, 7)),
        "misordered keys": (ind, _swap(key, 3, 5), _swap(p, 3, 5)),   # whole entries swapped across key runs
        "wrong major": (ind, _swap(key, 2, 3), _swap(p, 2, 3)),       # an entry moved across the major boundary
        "key without payload": (ind, _swap(key, 0, 1), p),
        "duplicated payload": (ind, key, torch.where(p == 5, 2, p)),
        "payload out of range": (ind, key, torch.where(p == 5, 8, p)),
        "indptr": (ind + torch.tensor([1, 0]), key, p),
        "truncated": (ind, key[:-1], p[:-1]),
    }
    for name, (bi, bk, bp) in bad.items():
        with pytest.raises(AssertionError):
            check_csr_sort(major, minor, bi, bk, bp.view(torch.float32), counts, True)
    with pytest.raises(AssertionError):       # a right answer that is not the constructed sequence
        check_csr_sort(major, minor, ind, key, val, counts, True, want_minor=_swap(key, 0, 1))
    # sort_minor = 0: input order inside a major; a by-minor order is rejected
    ind0, key0, val0 = lexsort_answer(major, minor, 2, False)
    check_csr_sort(major, minor, ind0, key0, val0, counts, False)
    with pytest.raises(AssertionError):
        check_csr_sort(major, minor, ind, key, val, counts, False)
    with pytest.raises(AssertionError):
        check_csr_sort(major, minor, ind0, key0, val0, counts, True)


@pytest.mark.parametrize("seed", range(5))
def test_checker_rejects_random_corruptions(seed):
    """One transposition of a correct larger output is always caught: either keys, majors or stability break."""
    gen = torch.Generator().manual_seed(seed)
    counts = counts_of(edge_draws(300, 20000, gen, "cpu"), 300)
    major, minor, want = known_answer(counts, 257, "edges", gen)
    for sort_minor in (True, False):
        ind, key, val = lexsort_answer(major, minor, 300, sort_minor)
        p = val.view(torch.int32)
        rng = np.random.default_rng(seed)
        for _ in range(20):
            i, j = sorted(rng.choice(20000, 2, replace=False).tolist())
            with pytest.raises(AssertionError):
                check_csr_sort(major, minor, ind, _swap(key, i, j), _swap(p, i, j).view(torch.float32), counts,
                               sort_minor)

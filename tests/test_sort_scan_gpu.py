"""The two primitives under every device CSR build, at their boundaries and at production scale (csrc/ingest.cu):

* ``bfl_csr_from_triples_device``, a stable LSD radix sort of the (major << 32 | minor) key in 8-bit digits, one pass
  per digit of ``bits_for(num_minor)`` and ``bits_for(num_major)``, 8192-entry warp sub-tiles, 65536-entry CTAs and a
  scan of the 256 x warps digit counter matrix;
* ``inclusive_scan_i64``, three kernels over 2048-element tiles recursing over the tile sums (1 level up to 2048
  elements, 2 up to 2048^2, 3 above), reached through ``indptr`` and the popularity table.

The sort cases are known answers (tests/sort_ref.py): the sorted sequence is built first and permuted into the input,
the payload is the input position, and the O(n) checker runs on the device.  Small cases also meet np.lexsort."""
import numpy as np
import pytest
import torch

from tests.sort_ref import (check_csr_sort, counts_of, edge_draws, known_answer, numpy_csr, positions)

pytestmark = pytest.mark.gpu

DEV = "cuda"
MINORS = [1, 2, 255, 256, 257, 65535, 65536, 65537, 1 << 24, (1 << 24) + 1, 2 ** 31 - 1]
MAJORS = [1, 2, 256, 257, 65537, (1 << 24) + 1]
TILE_EDGES = [0, 1, 31, 32, 33, 8191, 8192, 8193, 65535, 65536, 65537]
SCAN_TILE = 2048


@pytest.fixture(scope="module", autouse=True)
def release_device_cache():
    """Hand the GBs this module's tensors cached back to the device for the library calls of later tests."""
    yield
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def scan_levels(n):
    levels = 1
    while n > SCAN_TILE:
        n, levels = -(-n // SCAN_TILE), levels + 1
    return levels


def sort_device(major, minor, vals, num_major, num_minor, sort_minor, stream=None):
    from buffalo_b200 import backend
    return backend.csr_from_triples_device(major, minor, vals, num_major, num_minor, sort_minor, stream)


def sort_aliased(cuda_lib, major, minor, vals, num_major, num_minor, sort_minor, stream):
    """bfl_csr_from_triples_device with d_val_out == d_vals (the in-place value sort of the seen-item staging)."""
    from buffalo_b200 import _cabi
    n = major.numel()
    indptr = torch.empty(num_major, dtype=torch.int64, device=DEV)
    key = torch.empty(max(n, 1), dtype=torch.int32, device=DEV)
    _cabi.check(cuda_lib.bfl_csr_from_triples_device(
        major.data_ptr(), minor.data_ptr(), vals.data_ptr(), n, num_major, num_minor, int(sort_minor),
        indptr.data_ptr(), key.data_ptr(), vals.data_ptr(), stream.cuda_stream), "bfl_csr_from_triples_device")
    return indptr, key[:n], vals


def run_known(counts, num_minor, minors, seed, sort_minor, order="shuffle"):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    major, minor, want = known_answer(counts, num_minor, minors, gen, order)
    ind, key, val = sort_device(major, minor, positions(major.numel(), DEV), counts.numel(), num_minor, sort_minor)
    check_csr_sort(major, minor, ind, key, val, counts, bool(sort_minor), want if sort_minor else None)
    return major, minor, ind, key, val


def edge_counts(num_major, n, seed):
    gen = torch.Generator(device=DEV).manual_seed(seed)
    return counts_of(edge_draws(num_major, n, gen, DEV), num_major)


@pytest.mark.parametrize("sort_minor", [1, 0])
@pytest.mark.parametrize("num_major", MAJORS)
@pytest.mark.parametrize("num_minor", MINORS)
def test_digit_pass_counts(cuda_lib, num_minor, num_major, sort_minor):
    """Every pass-count edge of bits_for (1 to 4 minor passes, 1 to 4 major passes, odd and even totals, so the result
    ends in either buffer), with keys piled at 0 and num - 1 so that a missing or capped top pass misorders them."""
    n = 70001
    run_known(edge_counts(num_major, n, num_minor ^ num_major), num_minor, "edges", num_major + num_minor, sort_minor)


@pytest.mark.parametrize("sort_minor", [1, 0])
@pytest.mark.parametrize("nnz", TILE_EDGES)
def test_warp_and_cta_tile_edges(cuda_lib, nnz, sort_minor):
    """nnz at the warp sub-tile (8192) and CTA (65536) edges, across the 1 -> 2 level counter scan (256 * warps > 2048
    from 65537 on), against the known answer and np.lexsort."""
    num_major, num_minor = 1000, 70000
    major, minor, ind, key, val = run_known(edge_counts(num_major, nnz, nnz), num_minor, "spread", nnz + 1, sort_minor)
    ind0, key0, val0 = numpy_csr(major.cpu().numpy(), minor.cpu().numpy(), positions(nnz, "cpu").numpy(), num_major,
                                 sort_minor)
    assert np.array_equal(ind.cpu().numpy(), ind0)
    assert np.array_equal(key.cpu().numpy(), key0)
    assert np.array_equal(val.cpu().numpy().view(np.int32), val0.view(np.int32))


@pytest.mark.parametrize("case", ["one key", "one key at the top", "two keys", "two majors", "zipf", "sorted",
                                  "reversed", "sorted, one major", "reversed, one major"])
@pytest.mark.parametrize("sort_minor", [1, 0])
def test_skewed_digits(cuda_lib, case, sort_minor):
    """One digit bucket holding every key of a pass, a few keys, Zipf(1.1) heads over 10^6 rows, and input that is
    already sorted or reverse-sorted (every warp ranks long runs of equal digits)."""
    n = 300007
    num_major, num_minor, minors, order = 5000, (1 << 24) + 1, "spread", "shuffle"
    counts = torch.zeros(num_major, dtype=torch.int64, device=DEV)
    if case == "one key":
        counts[0], minors = n, 0
    elif case == "one key at the top":
        counts[-1], minors = n, num_minor - 1
    elif case == "two keys":
        counts[-1], minors = n, "two"
    elif case == "two majors":
        counts[0], counts[-1], minors = n // 2, n - n // 2, num_minor - 1
    elif case == "zipf":
        n, num_major = 4_000_000, 1_000_000
        draws = (np.random.default_rng(11).zipf(1.1, n) - 1) % num_major
        counts = counts_of(torch.from_numpy(draws).to(DEV), num_major)
        assert int(counts[0]) > n // 20             # the head row alone holds about 9 % of the entries
    else:
        order = case.split(",")[0]
        if "one major" in case:
            counts[7] = n
        else:
            counts = edge_counts(num_major, n, 5)
    run_known(counts, num_minor, minors, 3, sort_minor, order)


SPECIAL_BITS = [0x7FC00000, 0xFFC00000, 0x7FA00000, 0x7F800001, 0xFFBFFFFF, 0x7FFFFFFF,   # quiet / signalling NaNs
                0x00000000, 0x80000000, 0x00000001, 0x807FFFFF, 0x00400000,               # +-0, denormals
                0x7F800000, 0xFF800000, 0x7F7FFFFF, 0x00800000]                           # +-inf, max, min normal


@pytest.mark.parametrize("sort_minor", [1, 0])
def test_payload_bits(cuda_lib, sort_minor):
    """Values are carried, never computed on: random bit patterns with NaNs, -0.0, denormals and infinities come back
    bit for bit through the host entry, the device entry and the aliased device entry."""
    from buffalo_b200 import backend
    rng = np.random.default_rng(2)
    n, num_major, num_minor = 300000, 5000, 257
    bits = rng.integers(0, 1 << 32, n, dtype=np.uint64).astype(np.uint32)
    at = rng.choice(n, 40 * len(SPECIAL_BITS), replace=False)
    bits[at] = np.tile(np.array(SPECIAL_BITS, dtype=np.uint32), 40)
    vals = bits.view(np.float32)
    major = rng.integers(0, num_major, n).astype(np.int32)
    minor = rng.integers(0, num_minor, n).astype(np.int32)
    want = numpy_csr(major, minor, vals, num_major, sort_minor)
    got_host = backend.csr_from_triples_host(major, minor, vals, num_major, num_minor, sort_minor)
    dmaj, dmin, dval = (torch.from_numpy(a).to(DEV) for a in (major, minor, vals))
    got_dev = [t.cpu().numpy() for t in sort_device(dmaj, dmin, dval, num_major, num_minor, sort_minor)]
    got_alias = [t.cpu().numpy() for t in sort_aliased(cuda_lib, dmaj, dmin, dval.clone(), num_major, num_minor,
                                                       sort_minor, torch.cuda.current_stream())]
    for got in (got_host, got_dev, got_alias):
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert np.array_equal(got[2].view(np.uint32), want[2].view(np.uint32))


@pytest.mark.parametrize("num_minor,num_major,sort_minor", [(257, 257, 1),       # 2 + 2 passes: ends in k0 / d_val_out
                                                            (65537, 257, 1),     # 3 + 2: ends in k1 / v1, copied back
                                                            (7, 65537, 1),       # 1 + 3
                                                            (70000, 257, 0),     # 0 + 2
                                                            (70000, 65537, 0)])  # 0 + 3
@pytest.mark.parametrize("default_stream", [True, False])
def test_aliased_values(cuda_lib, num_minor, num_major, sort_minor, default_stream):
    """d_vals == d_val_out, as the seen-item staging passes them, for odd and even pass totals: the values come out
    sorted in place, and the keys and indptr equal the unaliased call's."""
    n = 200003
    counts = edge_counts(num_major, n, 17)
    gen = torch.Generator(device=DEV).manual_seed(17)
    major, minor, want = known_answer(counts, num_minor, "edges", gen)
    stream = torch.cuda.current_stream() if default_stream else torch.cuda.Stream()
    inplace = positions(n, DEV).clone()
    ref = sort_device(major, minor, positions(n, DEV), num_major, num_minor, sort_minor)
    stream.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(stream):
        ind, key, val = sort_aliased(cuda_lib, major, minor, inplace, num_major, num_minor, sort_minor, stream)
    stream.synchronize()
    assert val.data_ptr() == inplace.data_ptr()
    check_csr_sort(major, minor, ind, key, val, counts, bool(sort_minor), want if sort_minor else None)
    assert torch.equal(ind, ref[0]) and torch.equal(key, ref[1])
    assert torch.equal(val.view(torch.int32), ref[2].view(torch.int32))


@pytest.mark.parametrize("alias", [False, True])
def test_back_to_back_on_a_side_stream(cuda_lib, alias):
    """Two calls on one non-default stream with no sync between them, the second sorting the first's output into the
    other orientation (optionally in place over the first's values): each call's device work, allocations and frees
    are ordered on the caller's stream."""
    n, num_major, num_minor = 3_000_017, 40000, 70001
    counts = edge_counts(num_major, n, 23)
    gen = torch.Generator(device=DEV).manual_seed(23)
    major, minor, want = known_answer(counts, num_minor, "spread", gen)
    rows = torch.repeat_interleave(torch.arange(num_major, dtype=torch.int32, device=DEV), counts, output_size=n)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        ind1, key1, val1 = sort_device(major, minor, positions(n, DEV), num_major, num_minor, 1, stream=side)
        first_vals = val1.clone()
        if alias:
            ind2, key2, val2 = sort_aliased(cuda_lib, key1, rows, val1, num_minor, num_major, 1, side)
        else:
            ind2, key2, val2 = sort_device(key1, rows, val1, num_minor, num_major, 1, stream=side)
    side.synchronize()
    check_csr_sort(major, minor, ind1, key1, first_vals, counts, True, want)
    check_csr_sort(minor, major, ind2, key2, val2, counts_of(minor, num_minor), True)


def test_counter_scan_three_levels(cuda_lib):
    """The BASELINE shape's scan depths: 2^27 + 2^20 entries make 16512 warp sub-tiles, so the 256 x 16512 digit
    counter matrix is scanned at 3 levels in each of the 6 passes, and 10^7 majors give indptr 3 levels too.  Both
    have more than 2049 first-level tiles, so the third level's prefix reaches the result (at 2049 tiles, the least
    size with 3 levels, the one prefix it corrects is never read)."""
    n, num_major, num_minor = (1 << 27) + (1 << 20), 10_000_000, 1_000_000
    counters = 256 * -(-n // 8192)
    for m in (counters, num_major):
        assert scan_levels(m) == 3 and -(-m // SCAN_TILE) > SCAN_TILE + 1
    gen = torch.Generator(device=DEV).manual_seed(5)
    counts = counts_of(torch.randint(0, num_major, (n,), generator=gen, device=DEV), num_major)
    run_known(counts, num_minor, "spread", 5, 1)


@pytest.mark.parametrize("power", [0, 1, 2, 3])
@pytest.mark.parametrize("n_items", [1, 2047, 2048, 2049, 4194304, 4194305, 4196353, 6000000])
def test_popularity_table_scan_depth(cuda_lib, n_items, power):
    """bfl_popularity_table_host at 1, 2 and 3 scan levels against np.cumsum(np.bincount(...) ** power), with counts
    small enough that count ** power and the total stay below 2^63.  4194305 is the least size with 3 levels, 4196353
    (2049 * 2048 + 1) the least whose third level's prefix is read."""
    from buffalo_b200 import backend
    rng = np.random.default_rng(n_items * 4 + power)
    nnz = 1_500_000
    keys = np.where(rng.random(nnz) < 0.5, (rng.zipf(1.3, nnz) - 1) % n_items, rng.integers(0, n_items, nnz))
    keys = keys.astype(np.int32)
    table = np.bincount(keys, minlength=n_items).astype(np.int64)
    assert (table.astype(np.float64) ** power).sum() < 2.0 ** 62          # no int64 overflow on either side
    got = backend.popularity_table_host(keys, n_items, power)
    assert np.array_equal(got, np.cumsum(table ** power))


@pytest.mark.parametrize("power", [0, 1, 3])
@pytest.mark.parametrize("n_items", [1, 2049, 4194305])
def test_popularity_table_no_keys(cuda_lib, n_items, power):
    from buffalo_b200 import backend
    got = backend.popularity_table_host(np.zeros(0, np.int32), n_items, power)
    want = np.arange(1, n_items + 1, dtype=np.int64) if power == 0 else np.zeros(n_items, np.int64)
    assert np.array_equal(got, want)


def test_popularity_table_device_on_a_side_stream(cuda_lib):
    """The device entry, twice back to back on a non-default stream, into two tables at the 3-level depth."""
    from buffalo_b200 import _cabi
    n_items, nnz = 4194305, 3_000_000
    rng = np.random.default_rng(8)
    keys = ((rng.zipf(1.2, nnz) - 1) % n_items).astype(np.int32)
    dkeys = torch.from_numpy(keys).to(DEV)
    torch.cuda.synchronize()
    side = torch.cuda.Stream()
    with torch.cuda.stream(side):
        tables = [torch.empty(n_items, dtype=torch.int64, device=DEV) for _ in range(2)]
        for power, t in zip((1, 2), tables):
            _cabi.check(cuda_lib.bfl_popularity_table_device(dkeys.data_ptr(), nnz, n_items, power, t.data_ptr(),
                                                             side.cuda_stream), "bfl_popularity_table_device")
    side.synchronize()
    counts = np.bincount(keys, minlength=n_items).astype(np.int64)
    for power, t in zip((1, 2), tables):
        assert np.array_equal(t.cpu().numpy(), np.cumsum(counts ** power))


@pytest.mark.parametrize("shape", ["uniform", "zipf"])
def test_consumers_at_three_level_indptr(cuda_lib, shape):
    """backend.csr_from_triples_host and data.base.csr_from_triples (which routes >= 1M entries to the device) with
    5 * 10^6 majors, so indptr is scanned at 3 levels, against the NumPy build."""
    from buffalo_b200 import backend
    from buffalo_b200.data import base
    rng = np.random.default_rng(31)
    num_major, num_minor = 5_000_000, 300_000
    assert scan_levels(num_major) == 3
    if shape == "uniform":
        n = 20_000_000
        major = rng.integers(0, num_major, n).astype(np.int32)
    else:
        n = 8_000_000
        major = ((rng.zipf(1.1, n) - 1) % num_major).astype(np.int32)
    minor = rng.integers(0, num_minor, n).astype(np.int32)
    vals = np.arange(n, dtype=np.int32).view(np.float32)
    want = numpy_csr(major, minor, vals, num_major, True)
    for got in (backend.csr_from_triples_host(major, minor, vals, num_major, num_minor),
                base.csr_from_triples(major, minor, vals, num_major)):
        assert np.array_equal(got[0], want[0]) and np.array_equal(got[1], want[1])
        assert np.array_equal(got[2].view(np.int32), want[2].view(np.int32))

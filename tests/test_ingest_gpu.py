"""Device ingest helpers (csrc/ingest.cu, SURVEY.md 8(f-1), 8(f-4)) against the NumPy paths they replace:
CSR build by a hand-written stable radix sort (fileio.hpp:330-378 ordering) and the cumulative popularity table of
BPRMF.prepare_sampling (bpr.py:99-111)."""
import numpy as np
import pytest

from tests.sort_ref import numpy_csr

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("U,I,nnz,sort_minor", [(50, 30, 400, True), (3000, 70000, 250000, True), (100000, 900, 600000, True),
                                                 (1, 5, 20, True), (5000, 5000, 0, True), (4000, 300, 90000, False)])
def test_csr_from_triples_matches_numpy(cuda_lib, U, I, nnz, sort_minor):
    from buffalo_b200 import backend
    rng = np.random.default_rng(U + nnz)
    rows = rng.integers(0, U, nnz).astype(np.int32)
    cols = rng.integers(0, I, nnz).astype(np.int32)
    vals = rng.normal(size=nnz).astype(np.float32)      # duplicates of (row, col) keep their input order (stable)
    for major, minor, nm, nn in ((rows, cols, U, I), (cols, rows, I, U)):
        ind, key, val = backend.csr_from_triples_host(major, minor, vals, nm, nn, sort_minor=sort_minor)
        ind0, key0, val0 = numpy_csr(major, minor, vals, nm, sort_minor)
        assert np.array_equal(ind, ind0)
        assert np.array_equal(key, key0)
        assert np.array_equal(val, val0)                  # bit-exact payload, stable order among equal keys


def test_data_layer_uses_device_sort(cuda_lib):
    """buffalo.data's csr_from_triples (MatrixMarket / Stream ingest) routes large inputs through the device sort."""
    from buffalo_b200.data import base
    rng = np.random.default_rng(3)
    n = base.DEVICE_SORT_MIN_NNZ + 1000
    rows = rng.integers(0, 20000, n)
    cols = rng.integers(0, 3000, n)
    vals = rng.integers(1, 6, n).astype(np.float32)
    got = base.csr_from_triples(rows, cols, vals, 20000)
    want = numpy_csr(rows, cols, vals, 20000, True)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("power", [0, 1, 2])
def test_popularity_table(cuda_lib, power):
    from buffalo_b200 import backend
    rng = np.random.default_rng(9)
    I = 7000
    keys = (rng.zipf(1.3, 300000) % I).astype(np.int32)
    got = backend.popularity_table_host(keys, I, power)
    table = np.bincount(keys, minlength=I).astype(np.int64)
    table **= power                                       # bpr.py:108
    assert np.array_equal(got, np.cumsum(table))

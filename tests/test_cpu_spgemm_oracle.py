"""The sequential sparse x sparse restatement (tests/spgemm_oracle.py), the bit-identity target of the GPU tests, against
scipy and against exact arithmetic."""
from fractions import Fraction

import numpy as np
import pytest
import scipy.sparse as sp

from tests import spgemm_oracle as so


def rand_csr(m, k, density, seed, empty_rows=0.0):
    rng = np.random.default_rng(seed)
    a = sp.random(m, k, density=density, format="csr", random_state=rng, dtype=np.float32)
    a.data = (rng.standard_normal(a.nnz)).astype(np.float32)
    if empty_rows > 0 and m > 0:
        keep = (rng.random(m) >= empty_rows).astype(np.float32)
        a = sp.diags(keep) @ a
        a.eliminate_zeros()
    a.sort_indices()
    return a.tocsr()


def check_against_scipy(A, B):
    rp, col, val = so.spgemm(A.indptr, A.indices, A.data, B.indptr, B.indices, B.data, B.shape[1])
    # structural pattern from |A| @ |B| with positive values (scipy drops numeric zeros of A @ B itself)
    pat = (abs(A).astype(np.float64) @ abs(B).astype(np.float64)).tocsr()
    pat.sort_indices()
    assert np.array_equal(rp, pat.indptr) and np.array_equal(col, pat.indices)
    exact = (A.astype(np.float64) @ B.astype(np.float64)).tocsr()
    bound = pat.copy()
    got = sp.csr_matrix((val.astype(np.float64), col, rp), shape=pat.shape)
    diff = abs(got - exact).tocsr()
    # fp32 accumulation: error within a few ulps of the sum of |terms| (not of the possibly cancelling result)
    if pat.nnz:
        r, c = pat.nonzero()
        d, s = np.asarray(diff[r, c]).ravel(), np.asarray(bound[r, c]).ravel()
        assert (d <= 1e-5 * s + 1e-30).all()
    return rp, col, val


@pytest.mark.parametrize("m,k,n,density,seed", [(40, 30, 50, 0.1, 0), (200, 120, 90, 0.03, 1), (7, 300, 5, 0.2, 2),
                                                (150, 150, 150, 0.05, 3)])
def test_oracle_matches_scipy_rectangular(m, k, n, density, seed):
    A, B = rand_csr(m, k, density, seed), rand_csr(k, n, density, seed + 100)
    check_against_scipy(A, B)


def test_oracle_empty_rows_empty_product_and_k1():
    A = rand_csr(80, 60, 0.08, 4, empty_rows=0.4)
    B = rand_csr(60, 70, 0.08, 5, empty_rows=0.4)
    assert (np.diff(A.indptr) == 0).any() and (np.diff(B.indptr) == 0).any()
    check_against_scipy(A, B)
    # empty product: A's columns hit only empty rows of B
    Bz = sp.csr_matrix((np.ones(3, np.float32), np.array([0, 1, 2]), np.array([0, 0, 3])), shape=(2, 3))
    Az = sp.csr_matrix((np.ones(4, np.float32), np.zeros(4, np.int32), np.array([0, 1, 2, 3, 4])), shape=(4, 2))
    rp, col, val = check_against_scipy(Az, Bz)
    assert rp[-1] == 0 and col.size == 0
    # k = 1: an outer product
    A1, B1 = rand_csr(30, 1, 0.5, 6), rand_csr(1, 40, 0.5, 7)
    rp, col, val = check_against_scipy(A1, B1)
    assert rp[-1] == np.count_nonzero(np.diff(A1.indptr)) * B1.nnz


def test_structural_zero_is_kept():
    A = sp.csr_matrix(np.array([[1.0, 1.0]], np.float32))
    B = sp.csr_matrix(np.array([[2.0], [-2.0]], np.float32))
    rp, col, val = so.spgemm(A.indptr, A.indices, A.data, B.indptr, B.indices, B.data, 1)
    assert list(rp) == [0, 1] and list(col) == [0] and val[0] == 0.0


def test_fmaf_is_correctly_rounded():
    rng = np.random.default_rng(9)
    a = (rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 30, 4000)).astype(np.float32)
    b = (rng.standard_normal(4000) * 2.0 ** rng.integers(-30, 30, 4000)).astype(np.float32)
    c = (rng.standard_normal(4000) * 2.0 ** rng.integers(-60, 60, 4000)).astype(np.float32)
    c[:1000] = -(a[:1000].astype(np.float64) * b[:1000]).astype(np.float32)   # near-cancelling sums
    got = so.fmaf(a, b, c)
    for i in range(a.size):
        exact = Fraction(float(a[i])) * Fraction(float(b[i])) + Fraction(float(c[i]))
        r = np.float32(float(exact))          # may double-round: check the neighbours against the exact value
        cands = [np.nextafter(r, np.float32(-np.inf)), r, np.nextafter(r, np.float32(np.inf))]
        best = min(cands, key=lambda v: (abs(Fraction(float(v)) - exact), int(np.float32(v).view(np.int32)) & 1))
        assert got[i] == best, (a[i], b[i], c[i])


def test_coalesce_sums_duplicates_in_input_order():
    row, col = np.array([1, 0, 1, 1, 0]), np.array([2, 1, 2, 0, 1])
    val = np.array([1.0, 2.0, 3.0, 4.0, 5.0], np.float32)
    rp, c, v = so.coalesce(row, col, val, 2, 3)
    assert list(rp) == [0, 1, 3] and list(c) == [1, 0, 2] and list(v) == [7.0, 4.0, 4.0]

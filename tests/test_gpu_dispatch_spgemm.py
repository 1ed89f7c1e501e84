"""Every tier edge of the sparse x sparse product (cogdl_b200/csrc/spgemm.cu) and its value gradients, one row of
tests/dispatch_table.py SPGEMM_TABLE each.  For every row:

- The product still reaches the edges the row names (tests/spgemm_oracle.py edges(), on the row's numpy builder).
- Count phase through the C ABI: rowptrC and nnz equal the sequential oracle's (tests/spgemm_oracle.py), and the
  tier populations and tier lists that spg_classify_kernel leaves in the scratch equal the host restatement of the
  classifier (spgemm_oracle.classify).  The call records the count name.
- Forward through spspmm: pattern and values bit-identical to the oracle (test_gpu_spspmm.run_and_check), recording
  the fill name.  Exact cancellations give +0.0, subnormal products are kept (no flush to zero), and products with a
  -0.0 factor add +0.0 or -0.0 exactly as the fp32 fused multiply-add does.
- Count and fill once more with every scratch byte set to 0xFF before each phase: the same rowptrC, columns and value
  bits.  No tier may rely on zeroed scratch (the bitmap slots are zeroed only by the blocks that have rows).
- Backward through autograd three times, for dA only, dB only and both, each recording its own name.  Every input
  entry's gradient (a duplicated entry's: its merged slot's) must be bit-identical to spgemm_oracle.spgemm_bwd, the
  kernels' order: one warp per entry, lane l chaining acc = fmaf(x, y, acc) over the terms l, l + 32, ... from +0,
  then v = v + v[lane ^ off] for off = 16, 8, 4, 2, 1 and lane 0's value.  And that emulation must be within a bound
  of an fp64 scipy restatement, dA = (dC B^T) at A's pattern and dB = (A^T dC) at B's, so that it cannot share a
  mistake with the kernels:

      |dX - dX64| <= gamma_{ceil(d/32) + 5} sum|t| + (d + 32) 2^-150 + d 2^-52 sum|t|,   gamma_n = n u / (1 - n u)

  for an entry of d terms t (d: the length of its B row for dA, of its A column for dB), u = 2^-24.  Each fmaf
  rounds once, fl(x y + acc) = (x y + acc)(1 + delta) + eta with |delta| <= u and |eta| <= 2^-150 (half the spacing
  of subnormals; delta = 0 where eta is not), and each of the butterfly's five levels of additions rounds once more.
  A term reaches lane 0 through at most ceil(d/32) fmas of its lane and five additions, so the relative part is
  gamma_{ceil(d/32)+5} sum|t|.  Lane 0's result depends on d fmas and 31 additions, each adding one eta, which the
  later roundings scale by at most 1 + gamma (< 1 + 1/(d + 31) here), hence (d + 32) 2^-150.  The fp64 sum of d
  exact products adds at most d 2^-53 sum|t|; the bound allows twice that.
"""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests import graphs
from tests import spgemm_oracle as so
from tests.dispatch_table import SPG_COUNT, SPG_DA, SPG_DA_DB, SPG_DB, SPG_FILL, SPGEMM_TABLE
from tests.gpu_util import T, dev
from tests.test_gpu_spspmm import run_and_check, to_dev

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24


def raw_product(dev, a, b, m, k, n, dirty):
    """cogdl_b200_spgemm_count then _fill_f32 on the merged CSRs a = (rowptr, col, val) and b.  The scratch is zeroed
    once, or (dirty) set to 0xFF bytes before each phase.  Returns (rowptrC, nnz, colC, valC, count's recorded name,
    fill's, the tier lists the count's classifier left in the scratch (None when m = 0))."""
    from cogdl_b200 import _cabi
    from cogdl_b200.structure import _ptr, _stream

    lib = _cabi.load()
    rpA, cA, vA = T(a[0].astype(np.int32), dev), T(a[1], dev), T(a[2], dev)
    rpB, cB, vB = T(b[0].astype(np.int32), dev), T(b[1], dev), T(b[2], dev)
    nbytes = int(lib.cogdl_b200_spgemm_scratch_bytes(m, k, n))
    scratch = torch.full((nbytes,), 0xFF if dirty else 0, dtype=torch.uint8, device=dev)
    assert scratch.data_ptr() % 256 == 0
    rowptr = torch.full((m + 1,), -7, dtype=torch.int32, device=dev)
    nnz = ctypes.c_int64(-1)
    _cabi.call("cogdl_b200_spgemm_count", _ptr(rpA), _ptr(cA), m, k, _ptr(rpB), _ptr(cB), k, n, _ptr(rowptr),
               ctypes.byref(nnz), _ptr(scratch), nbytes, _stream(dev))
    count_name = _cabi.last_kernel()
    lists = None
    if m > 0:
        # carve(): list_n [3] at the scratch's first 256-byte boundary, then the warp, block and bitmap lists of m rows
        ints = scratch[:256 + 12 * m].view(torch.int32).cpu().numpy()
        lists = [np.sort(ints[64 + t * m: 64 + t * m + ints[t]]) if 0 <= ints[t] <= m else ints[t] for t in range(3)]
    if dirty:
        scratch.fill_(0xFF)
    col = torch.full((nnz.value,), -1, dtype=torch.int32, device=dev)
    val = torch.full((nnz.value,), float("nan"), dtype=torch.float32, device=dev)
    _cabi.call("cogdl_b200_spgemm_fill_f32", _ptr(rpA), _ptr(cA), _ptr(vA), m, k, _ptr(rpB), _ptr(cB), _ptr(vB), k, n,
               _ptr(rowptr), _ptr(col), _ptr(val), _ptr(scratch), nbytes, _stream(dev))
    return (rowptr.cpu().numpy(), nnz.value, col.cpu().numpy(), val.cpu().numpy(), count_name, _cabi.last_kernel(),
            lists)


def autograd_grads(dev, A, B, m, k, n, g, want_a, want_b):
    """spspmm with gradients for the inputs asked for, then backward with dC = g: (names recorded, dA, dB) per input
    entry (None where not asked for).  The names are read by hooks on the inputs' gradients: the backward runs on
    autograd's device thread, and cogdl_b200_last_kernel() is kept per thread."""
    import cogdl_b200
    from cogdl_b200 import _cabi

    ia, xa = to_dev(*A, dev)
    ib, xb = to_dev(*B, dev)
    names = []
    for x, want in ((xa, want_a), (xb, want_b)):
        if want:
            x.requires_grad_(True)
            x.register_hook(lambda grad: names.append(_cabi.last_kernel()))
    _, val = cogdl_b200.spspmm(ia, xa, ib, xb, m, k, n)
    val.backward(T(g, dev))
    grad = lambda x, want: x.grad.cpu().numpy() if want else None  # noqa: E731
    return names, grad(xa, want_a), grad(xb, want_b)


def fp64_grads(a, b, m, k, n, rp, col, g):
    """(dA, sum|terms| of dA, dB, sum|terms| of dB) at the merged patterns, in fp64 with scipy."""
    def csr(x, shape, absolute=False):
        v = np.asarray(x[2], np.float64)
        return sp.csr_matrix((np.abs(v) if absolute else v, x[1].copy(), x[0].copy()), shape=shape)

    def at(M, rows, cols):
        return np.asarray(M[rows, cols]).ravel() if rows.size else np.zeros(0)

    rowA = np.repeat(np.arange(m), np.diff(a[0]))
    rowB = np.repeat(np.arange(k), np.diff(b[0]))
    out = []
    for absolute in (False, True):
        Am, Bm, G = csr(a, (m, k), absolute), csr(b, (k, n), absolute), csr((rp, col, g), (m, n), absolute)
        out.append((at((G @ Bm.T).tocsr(), rowA, a[1]), at((Am.T @ G).tocsr(), rowB, b[1])))
    return out[0][0], out[1][0], out[0][1], out[1][1]


def gamma(n):
    return n * U32 / (1 - n * U32)


def slots(row, col, n_cols):
    """The merged CSR slot of every COO input entry (spgemm_oracle.coalesce's order: by row, then column)."""
    key = np.asarray(row, np.int64) * max(n_cols, 1) + np.asarray(col, np.int64)
    return np.unique(key, return_inverse=True)[1].ravel()


@pytest.mark.parametrize("c", SPGEMM_TABLE, ids=lambda c: c.id)
def test_spgemm_row(dev, c, record_property):
    A, B, m, k, n = graphs.spgemm_case(c.name)
    a, b = so.coalesce(*A, m, k), so.coalesce(*B, k, n)
    rp, col, val = so.spgemm(*a, *b, n)
    _, tier = so.classify(a[0], a[1], b[0], n)
    missing = sorted(set(c.edges) - so.edges(A, B, m, k, n))
    assert not missing, f"{c.id}: the product no longer reaches {missing}"

    # count and fill through the C ABI, on zeroed and on 0xFF scratch
    for dirty in (False, True):
        rowptr, nnz, colC, valC, count_name, fill_name, lists = raw_product(dev, a, b, m, k, n, dirty)
        what = f"{c.id} ({'0xFF' if dirty else 'zeroed'} scratch)"
        assert count_name == SPG_COUNT and fill_name == SPG_FILL, (what, count_name, fill_name)
        assert np.array_equal(rowptr, rp) and nnz == col.size, f"{what}: rowptrC differs from the oracle"
        if lists is not None:
            for t, name in enumerate(so.TIERS):
                want = np.flatnonzero(tier == t)
                assert np.array_equal(lists[t], want), \
                    f"{what}: {name} tier holds {np.size(lists[t])} rows, the classifier's restatement {want.size}"
        assert np.array_equal(colC, col), f"{what}: columns differ from the oracle"
        assert np.array_equal(valC.view(np.int32), val.view(np.int32)), \
            f"{what}: values differ from the oracle at {np.flatnonzero(valC.view(np.int32) != val.view(np.int32))[:8]}"

    # forward through spspmm
    from cogdl_b200 import _cabi

    run_and_check(A, B, m, k, n, dev)
    assert _cabi.last_kernel() == SPG_FILL

    # backward: the kernels' order bit for bit, and that order within the bound of fp64
    g = np.random.default_rng(1).standard_normal(col.size).astype(np.float32)
    emu_a, emu_b = so.spgemm_bwd(*a, *b, rp, col, g)
    ref_a, abs_a, ref_b, abs_b = fp64_grads(a, b, m, k, n, rp, col, g)
    d_a = np.diff(b[0])[a[1]]                                     # terms of a dA entry: its B row's length
    d_b = np.bincount(a[1], minlength=k)[np.repeat(np.arange(k), np.diff(b[0]))]   # of a dB entry: A column's
    worst = 0.0
    for what, emu, ref, tsum, d in (("dA", emu_a, ref_a, abs_a, d_a), ("dB", emu_b, ref_b, abs_b, d_b)):
        bound = gamma((d + 31) // 32 + 5) * tsum + (d + 32) * 2.0 ** -150 + d * 2.0 ** -52 * tsum
        err = np.abs(emu.astype(np.float64) - ref)
        bad = np.flatnonzero(~(err <= bound))
        assert bad.size == 0, (f"{c.id}: {what} emulation off fp64 at {bad[:8]}: {emu[bad[:4]]} vs {ref[bad[:4]]}, "
                               f"bound {bound[bad[:4]]}")
        if err.size:
            worst = max(worst, float(np.max(err / bound)))
    record_property("bwd_error_over_bound", worst)
    sa, sb = slots(A[0], A[1], k), slots(B[0], B[1], n)
    for want_a, want_b, name in ((True, False, SPG_DA), (False, True, SPG_DB), (True, True, SPG_DA_DB)):
        names, ga, gb = autograd_grads(dev, A, B, m, k, n, g, want_a, want_b)
        assert names == [name] * (want_a + want_b), f"{c.id}: the backward recorded {names!r}, not {name!r}"
        for what, got, emu, sl in (("dA", ga, emu_a, sa), ("dB", gb, emu_b, sb)):
            if got is None:
                continue
            diff = np.flatnonzero(got.view(np.int32) != emu[sl].view(np.int32))
            assert diff.size == 0, (f"{c.id} ({name}): {what} differs from the kernels' order at input entries "
                                    f"{diff[:8]}: {got[diff[:4]]} vs {emu[sl][diff[:4]]}")

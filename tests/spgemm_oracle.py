"""Sequential Gustavson restatement of the sparse x sparse product in the kernel's order -- test infrastructure.

C = A.B for int32 CSR A, B with ascending unique columns per row: for each row i, A's entries in CSR order, for each
k B_k's entries in CSR order, acc[i, j] = fmaf(a_ik, b_kj, acc[i, j]) from 0.  The columns of row i come out ascending.
Vectorised over all output slots at once (step r applies every slot's r-th product), with a correctly rounded fp32
fused multiply-add: the fp32 product is exact in fp64, the fp64 sum is made exact with TwoSum and rounded to odd, and
rounding that to fp32 is the correctly rounded fma (53 >= 24 + 2 bits).
"""
import numpy as np


def fmaf(a, b, c):
    """Correctly rounded fp32 a * b + c, elementwise (finite inputs, no overflow)."""
    p = a.astype(np.float64) * b.astype(np.float64)
    c = c.astype(np.float64)
    s = p + c
    bp = s - c
    err = (p - bp) + (c - (s - bp))            # s + err == p + c exactly
    odd = (s.view(np.int64) & 1) == 1
    toward = np.where(err > 0, np.inf, -np.inf)
    s = np.where((err != 0) & ~odd, np.nextafter(s, toward), s)
    return s.astype(np.float32)


def spgemm(rpA, colA, valA, rpB, colB, valB, n):
    """(rowptrC, colC, valC) of C = A.B; A is (len(rpA)-1) x (len(rpB)-1), B has n columns."""
    rpA, colA, rpB, colB = (np.asarray(x, np.int64) for x in (rpA, colA, rpB, colB))
    valA, valB = np.asarray(valA, np.float32), np.asarray(valB, np.float32)
    m = rpA.size - 1
    degB = np.diff(rpB)
    rowA = np.repeat(np.arange(m), np.diff(rpA))
    reps = degB[colA]                                    # products of every A entry
    pa = np.repeat(np.arange(colA.size), reps)           # products in (row, A order, B order)
    start = np.repeat(rpB[colA], reps)
    within = np.arange(pa.size) - np.repeat(np.cumsum(reps) - reps, reps)
    pb = start + within
    prow, pcol = rowA[pa], colB[pb]
    key = prow * max(n, 1) + pcol
    order = np.argsort(key, kind="stable")               # by output slot, (A order, B order) inside a slot
    key_s = key[order]
    new = np.ones(key_s.size, bool)
    new[1:] = key_s[1:] != key_s[:-1]
    slot = np.cumsum(new) - 1
    nnz = int(slot[-1]) + 1 if slot.size else 0
    first = np.flatnonzero(new)
    rank = np.arange(key_s.size) - first[slot] if slot.size else slot
    acc = np.zeros(nnz, np.float32)
    a_s, b_s = valA[pa[order]], valB[pb[order]]
    for r in range(int(rank.max()) + 1 if rank.size else 0):
        sel = rank == r
        acc[slot[sel]] = fmaf(a_s[sel], b_s[sel], acc[slot[sel]])
    rowC = prow[order][new]
    colC = pcol[order][new].astype(np.int32)
    rowptrC = np.zeros(m + 1, np.int64)
    np.cumsum(np.bincount(rowC, minlength=m), out=rowptrC[1:])
    return rowptrC, colC, acc


def coalesce(row, col, val, m, k):
    """(rowptr, col, val) of a COO with duplicates summed in input order (fp32), columns ascending in each row."""
    row, col = np.asarray(row, np.int64), np.asarray(col, np.int64)
    val = np.asarray(val, np.float32)
    key = row * max(k, 1) + col
    order = np.argsort(key, kind="stable")
    key_s = key[order]
    new = np.ones(key_s.size, bool)
    new[1:] = key_s[1:] != key_s[:-1]
    slot = np.cumsum(new) - 1
    out = np.zeros(int(new.sum()), np.float32)
    first = np.flatnonzero(new)
    rank = np.arange(key_s.size) - first[slot] if slot.size else slot
    for r in range(int(rank.max()) + 1 if rank.size else 0):
        sel = rank == r
        out[slot[sel]] = out[slot[sel]] + val[order][sel] if r else val[order][sel]
    urow = row[order][new]
    rowptr = np.zeros(m + 1, np.int64)
    np.cumsum(np.bincount(urow, minlength=m), out=rowptr[1:])
    return rowptr, col[order][new].astype(np.int32), out

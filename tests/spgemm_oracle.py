"""Sequential Gustavson restatement of the sparse x sparse product in the kernel's order -- test infrastructure.

C = A.B for int32 CSR A, B with ascending unique columns per row: for each row i, A's entries in CSR order, for each
k B_k's entries in CSR order, acc[i, j] = fmaf(a_ik, b_kj, acc[i, j]) from 0.  The columns of row i come out ascending.
Vectorised over all output slots at once (step r applies every slot's r-th product), with a correctly rounded fp32
fused multiply-add: the fp32 product is exact in fp64, the fp64 sum is made exact with TwoSum and rounded to odd, and
rounding that to fp32 is the correctly rounded fma (53 >= 24 + 2 bits).

Also the kernels' tier classifier on the host (classify), the tier edges a product reaches (edges, for
tests/dispatch_table.py SPGEMM_TABLE), and the value gradients in the backward kernels' order (spgemm_bwd).
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


def products(colA, rpB):
    """(pa, pb, within): the A and B entry of every product a_ik b_kj in (row, A order, B order), and the product's
    position in B_k (0 .. deg_B(k) - 1)."""
    colA, rpB = np.asarray(colA, np.int64), np.asarray(rpB, np.int64)
    reps = np.diff(rpB)[colA]                            # products of every A entry
    pa = np.repeat(np.arange(colA.size), reps)
    within = np.arange(pa.size) - np.repeat(np.cumsum(reps) - reps, reps)
    return pa, np.repeat(rpB[colA], reps) + within, within


def spgemm(rpA, colA, valA, rpB, colB, valB, n):
    """(rowptrC, colC, valC) of C = A.B; A is (len(rpA)-1) x (len(rpB)-1), B has n columns."""
    rpA, colA, rpB, colB = (np.asarray(x, np.int64) for x in (rpA, colA, rpB, colB))
    valA, valB = np.asarray(valA, np.float32), np.asarray(valB, np.float32)
    m = rpA.size - 1
    rowA = np.repeat(np.arange(m), np.diff(rpA))
    pa, pb, _ = products(colA, rpB)
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


# ------------------------------------------------------------------ the tiers of spgemm.cu, restated on the host
WARP_CAP, BLOCK_CAP = 256, 4096           # SPG_WARP_CAP, SPG_BLOCK_CAP
NUM_SMS, WARPS = 132, 8                   # NUM_SMS (common.cuh), SPG_WARPS
TIERS = ("warp", "block", "bitmap")
# rows a tier's launch takes before its grid-stride loop comes round again: NUM_SMS * 8 blocks of 8 warps, NUM_SMS * 2
# blocks, SPG_LARGE_SLOTS = NUM_SMS bitmap slots
GRID_ROWS = {"warp": NUM_SMS * 8 * WARPS, "block": NUM_SMS * 2, "bitmap": NUM_SMS}
# hash tables of 2 * CAP slots; a wrap-around row has CAP columns that all hash into the table's last TAIL slots
HASH_TAIL = {"warp": (2 * WARP_CAP, 8), "block": (2 * BLOCK_CAP, 64)}
BWD_TERMS = (1, 31, 32, 33, 65, 2000)     # terms of one backward entry: one lane, 31 and 32 lanes, a second and a third
                                          # iteration, and 63 iterations of which the last is half-full


def classify(rpA, colA, rpB, n):
    """spg_classify_kernel: (sum, tier) of every row i of C = A.B, sum = sum_{k in A_i} deg_B(k) and the tier from
    bound = min(sum, n): -1 (nothing to do) for 0, 0 (warp) up to WARP_CAP, 1 (block) up to BLOCK_CAP, 2 (bitmap)."""
    rpA, colA, rpB = (np.asarray(x, np.int64) for x in (rpA, colA, rpB))
    m = rpA.size - 1
    rowA = np.repeat(np.arange(m), np.diff(rpA))
    s = np.bincount(rowA, weights=np.diff(rpB)[colA], minlength=m).astype(np.int64)
    bound = np.minimum(s, n)
    return s, np.select([bound == 0, bound <= WARP_CAP, bound <= BLOCK_CAP], [-1, 0, 1], 2)


def hash_slot(j, ts):
    """spg_hash<TS>: the high log2(TS) bits of j * 0x9E3779B1 mod 2^32."""
    h = (np.asarray(j, np.uint64) * np.uint64(0x9E3779B1)) & np.uint64(0xFFFFFFFF)
    return (h >> np.uint64(32 - (int(ts).bit_length() - 1))).astype(np.int64)


def edges(A, B, m, k, n):
    """The (tier, edge) pairs that C = A.B of the COO inputs A = (row, col, val) (m x k) and B (k x n) reaches, on the
    merged CSRs.  tests/dispatch_table.py SPGEMM_TABLE names the ones each row is built for."""
    (ra, _, _), (rb, _, _) = A, B
    pa, qa, wa = coalesce(*A, m, k)
    pb, qb, wb = coalesce(*B, k, n)
    rp, col, val = spgemm(pa, qa, wa, pb, qb, wb, n)
    s, tier = classify(pa, qa, pb, n)
    degA, c = np.diff(pa), np.diff(rp)
    rowC = np.repeat(np.arange(m), c)
    tierC = tier[rowC]
    out = set()

    def holds(cols, what):
        """some row of `what` holds all of `cols`"""
        return bool(np.any((np.bincount(rowC, weights=np.isin(col, cols), minlength=m) == len(cols)) & what))

    # rows with nothing to do, and degenerate shapes
    if np.any(degA == 0):
        out.add(("empty", "A row without entries"))
    if np.any((degA > 0) & (s == 0)):
        out.add(("empty", "A row meeting only empty B rows"))
    shape = {"m = 0": m == 0 < min(k, n) and rb.size > 0,
             "k = 0": k == 0 < min(m, n),
             "n = 0": n == 0 < min(m, k) and ra.size > 0,
             "A without entries": min(m, k, n) > 0 and ra.size == 0 < rb.size,
             "B without entries": min(m, k, n) > 0 and rb.size == 0 < ra.size,
             "m, k, n distinct, every tier": len({m, k, n}) == 3 and {0, 1, 2} <= set(tier.tolist())}
    out |= {("shape", e) for e, hit in shape.items() if hit}
    # distinct counts at and past each cap, with distinct count = bound (disjoint B rows)
    for v, t in ((1, "warp"), (255, "warp"), (256, "warp"), (257, "block"), (4095, "block"), (4096, "block"),
                 (4097, "bitmap")):
        if np.any((c == s) & (c == v)):
            out.add((t, f"{v} columns"))
    # bounds over a cap with a tiny distinct count
    bound = np.minimum(s, n)
    for b, v, t in ((256, 1, "warp"), (300, 2, "block"), (5000, 3, "bitmap")):
        if np.any((bound == b) & (c == v)):
            out.add((t, f"bound {b}, {v} columns"))
    # full tables whose columns all hash into the last slots: probes wrap past the end
    for t, (ts, tail) in HASH_TAIL.items():
        early = np.bincount(rowC, weights=hash_slot(col, ts) < ts - tail, minlength=m)
        if np.any((tier == TIERS.index(t)) & (c == ts // 2) & (early == 0)):
            out.add((t, "hash wrap-around"))
    # the bound capped by n
    if 0 < n <= WARP_CAP and np.any((c == n) & (s > BLOCK_CAP)):
        out.add(("warp", "n <= 256, full row"))
    if n == BLOCK_CAP and np.any((c == n) & (s > BLOCK_CAP)):
        out.add(("block", "n = 4096, full row"))
    # the bitmap: a full row, the last partial word, exactly 256 words and one scan carry
    big = tier == 2
    if np.any(big & (c == n)):
        out.add(("bitmap", "all n columns"))
    if n % 32 == 1 and holds([0, 31, 32, 63, 64, n - 1], big):
        out.add(("bitmap", "n = 32w + 1"))
    for w in (8192, 8193):
        if n == w and holds([0, n - 1], big):
            out.add(("bitmap", f"n = {w}"))
    # grid-stride loops: more rows than the launch has warps, blocks or bitmap slots
    for t, rows in GRID_ROWS.items():
        if np.sum(tier == TIERS.index(t)) > rows:
            out.add((t, "grid loop"))
    # values, each in a row of every tier: an exact cancellation (+0.0 from normal terms), subnormal outputs, outputs
    # whose every product has a -0.0 factor (+0.0)
    if m and rowC.size:
        ppa, ppb, _ = products(qa, pb)
        rowA = np.repeat(np.arange(m), degA)
        slot = np.searchsorted(rowC * max(n, 1) + col, rowA[ppa] * max(n, 1) + qb[ppb])
        terms = np.bincount(slot, weights=np.abs(wa[ppa].astype(np.float64) * wb[ppb]), minlength=col.size)
        negz = (np.signbit(wa[ppa]) & (wa[ppa] == 0)) | (np.signbit(wb[ppb]) & (wb[ppb] == 0))
        only_negz = np.bincount(slot, weights=~negz, minlength=col.size) == 0
        pos0 = val.view(np.uint32) == 0
        flags = {"exact cancellation": pos0 & (terms >= 2.0 ** -126),
                 "subnormal": (val != 0) & (np.abs(val) < 2.0 ** -126),
                 "-0.0 factors": pos0 & only_negz}
        for e, f in flags.items():
            if all(np.any(f & (tierC == t)) for t in range(3)):
                out.add(("values", e))
    # the backward: terms of a dA entry (its B row's length) and of a dB entry (its A column's length), duplicates
    dA_terms = set(np.diff(pb)[qa].tolist())
    dB_terms = set(np.bincount(qa, minlength=k)[np.repeat(np.arange(k), np.diff(pb))].tolist())
    for t, seen in (("dA", dA_terms), ("dB", dB_terms)):
        out |= {(t, f"{d} terms") for d in BWD_TERMS if d in seen}
    if ra.size > qa.size:
        out.add(("dA", "duplicate entries"))
    if rb.size > qb.size:
        out.add(("dB", "duplicate entries"))
    return out


# ------------------------------------------------------------------ the backward in the kernels' order
def _warp_sums(entry, t, x, y, count):
    """One warp per entry: lane t % 32 chains acc = fmaf(x, y, acc) over the entry's terms t = lane, lane + 32, ...
    from +0, then v = v + v[lane ^ off] for off = 16, 8, 4, 2, 1; lane 0's value of every entry."""
    acc = np.zeros((count, 32), np.float32)
    lane, rnd = t % 32, t // 32
    order = np.argsort(rnd, kind="stable")
    ends = np.searchsorted(rnd[order], np.arange(int(rnd.max()) + 2 if rnd.size else 1))
    for r in range(ends.size - 1):
        sel = order[ends[r]:ends[r + 1]]
        e, ln = entry[sel], lane[sel]
        acc[e, ln] = fmaf(x[sel], y[sel], acc[e, ln])
    for off in (16, 8, 4, 2, 1):
        acc = acc + acc[:, np.arange(32) ^ off]
    return acc[:, 0]


def spgemm_bwd(rpA, colA, valA, rpB, colB, valB, rpC, colC, dC):
    """(dA, dB) as spg_dA_kernel and spg_dB_kernel compute them on the merged CSRs: dA[p = (i, k)] over B_k's entries
    q in CSR order, b_q dC[i, col_B(q)]; dB[q = (k, j)] over column k of A in row order, a_p dC[row(p), j]."""
    rpA, colA, rpB, colB, rpC, colC = (np.asarray(x, np.int64) for x in (rpA, colA, rpB, colB, rpC, colC))
    valA, valB, dC = (np.asarray(x, np.float32) for x in (valA, valB, dC))
    m, kb = rpA.size - 1, rpB.size - 1
    rowA = np.repeat(np.arange(m), np.diff(rpA))
    rowB = np.repeat(np.arange(kb), np.diff(rpB))
    keyC = (np.repeat(np.arange(m), np.diff(rpC)) << 31) + colC

    def dc(i, j):
        pos = np.searchsorted(keyC, (i << 31) + j)
        assert np.array_equal(keyC[pos], (i << 31) + j), "a product outside C's pattern"
        return dC[pos]

    pa, pb, t = products(colA, rpB)
    dA = _warp_sums(pa, t, valB[pb], dc(rowA[pa], colB[pb]), colA.size)
    at = np.lexsort((rowA, colA))                         # A's transpose: by column, rows ascending
    colptr = np.zeros(kb + 1, np.int64)
    np.cumsum(np.bincount(colA, minlength=kb), out=colptr[1:])
    qb, s, t = products(rowB, colptr)
    p = at[s]
    dB = _warp_sums(qb, t, valA[p], dc(rowA[p], colB[qb]), colB.size)
    return dA, dB

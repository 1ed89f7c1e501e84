"""Seeded test graphs (numpy, int32 CSR) shared by the oracle and GPU parity tests."""
import numpy as np


def random_csr(n, e, seed=0, n_cols=None, hub=None, empty_rows=0.0):
    """Random CSR with multinomial degrees.  hub=(row, degree) plants one heavy row (so the hub
    plan's chunking and in-order combination are exercised); empty_rows = fraction forced to 0."""
    rng = np.random.default_rng(seed)
    n_cols = n if n_cols is None else n_cols
    p = rng.random(n) ** 3 + 1e-3
    if empty_rows > 0:
        p[rng.random(n) < empty_rows] = 0
    p /= p.sum()
    deg = rng.multinomial(e, p) if e > 0 else np.zeros(n, np.int64)
    if hub is not None:
        deg[hub[0]] = hub[1]
    rowptr = np.zeros(n + 1, np.int32)
    rowptr[1:] = np.cumsum(deg)
    colind = rng.integers(0, n_cols, int(rowptr[-1])).astype(np.int32)
    return rowptr, colind


CASES = {
    # name: (n, e, kwargs)
    "tiny": (7, 20, {}),
    "empty_graph": (5, 0, {}),
    "ragged": (300, 2000, {"empty_rows": 0.3}),
    "hub": (400, 3000, {"hub": (17, 1500)}),          # 1500 > chunk 256 -> 6 chunks
    "two_hubs": (1000, 8000, {"hub": (999, 700), "empty_rows": 0.1}),
    "rect": (200, 1500, {"n_cols": 350}),
}


def case(name, seed=0):
    n, e, kw = CASES[name]
    rp, ci = random_csr(n, e, seed=seed, **kw)
    n_cols = kw.get("n_cols", n)
    return rp, ci, n_cols


def boundary_csr(C, seed=0):
    """Square CSR whose rows sit on the boundaries of a hub plan with C-edge chunks (not in CASES: the parity tests
    parametrised over CASES do not grow).  Returns (rowptr, colind, n_cols) like case().

    Rows, in order (a hub row ends a run of short rows, so the runs after hubs start fresh windows):
      0, 1, C - 1, C       the largest non-hub row fills a tile exactly when C * H is the tile size
      C + 1                a hub whose last chunk has one edge
      40 x 1               a full 32-row window of one-edge rows and a remainder of 8
      2C                   a hub of full chunks
      9, 7, 6, 4, 3, 2, 1  descending degrees in one window: the degree sort reverses them
      129 C + 5            a hub of 130 chunks: at H = 1 the statistics merge loop (128 chunks a pass) runs twice
      2, 0, 0, 0, 1, 3     empty rows inside a run of short rows
      then C, 2, C - 1, 5, 0 and 40 random degrees in [0, min(C, 16))."""
    rng = np.random.default_rng(seed)
    deg = [0, 1, C - 1, C, C + 1] + [1] * 40 + [2 * C, 9, 7, 6, 4, 3, 2, 1, 129 * C + 5, 2, 0, 0, 0, 1, 3]
    deg += [C, 2, C - 1, 5, 0] + list(rng.integers(0, min(C, 16), 40))
    n = len(deg)
    rowptr = np.zeros(n + 1, np.int32)
    rowptr[1:] = np.cumsum(deg)
    colind = rng.integers(0, n, int(rowptr[-1])).astype(np.int32)
    return rowptr, colind, n


def boundary_csc(C, seed=0):
    """The transpose of boundary_csr(C), as a CSR: its COLUMNS have the boundary degrees, so a backward that walks the
    transpose (under the transpose's own hub plan) meets them.  Its rows are the random columns of boundary_csr: the
    129 C + 5 hub spreads over every row, so rows with more than C edges occur here too.  Returns (rowptr, colind, n)."""
    rp, ci, n = boundary_csr(C, seed)
    rows = np.repeat(np.arange(n), np.diff(rp))
    order = np.lexsort((rows, ci))                   # by column, then row: CSR order of the transpose
    rowptr = np.zeros(n + 1, np.int32)
    rowptr[1:] = np.cumsum(np.bincount(ci, minlength=n))
    return rowptr, rows[order].astype(np.int32), n


# ------------------------------------------------------------------ sparse x sparse products at spgemm.cu's tier edges
# Each builder returns (A, B, m, k, n): COO inputs (row int64, col int64, val fp32) in a random order, A m x k and B
# k x n.  B rows whose columns must all be distinct in a product (distinct count = bound) are disjoint.
def _coo(lists, rng, vals=None):
    """COO of row i holding the columns lists[i] (and the values vals[i]; standard normal if None), shuffled."""
    row = np.repeat(np.arange(len(lists)), [len(x) for x in lists]).astype(np.int64)
    col = np.concatenate([np.asarray(x, np.int64) for x in lists] + [np.zeros(0, np.int64)])
    if vals is None:
        val = rng.standard_normal(row.size).astype(np.float32)
    else:
        val = np.concatenate([np.asarray(v, np.float32) for v in vals] + [np.zeros(0, np.float32)])
    p = rng.permutation(row.size)
    return row[p], col[p], val[p]


def _disjoint(degs, n, rng):
    """Column lists of the given lengths, pairwise disjoint, drawn at random from n columns."""
    perm = rng.permutation(n)
    ends = np.cumsum(degs)
    return [np.sort(perm[e - d:e]) for d, e in zip(degs, ends)]


def _some(n, d, rng, also=()):
    """d random columns of n, plus the columns `also`."""
    return np.union1d(rng.choice(n, d, replace=False), np.asarray(also, np.int64))


def _product(a, b, k, n, rng, va=None, vb=None):
    return _coo(a, rng, va), _coo(b, rng, vb), len(a), k, n


def _counts(degs, a, rng):
    """Disjoint B rows of the lengths degs, A rows a (lists of B rows), 7 columns no row reaches."""
    n = sum(degs) + 7
    return _product(a, _disjoint(degs, n, rng), len(degs), n, rng)


def _wrap(ts, tail, parts, rng):
    """The first ts / 2 columns that hash into the last `tail` of ts slots, split over `parts` B rows; row 0 of A
    takes them all, row 1 some, row 2 one of them and a row of 300 other columns; n = the largest column + 1."""
    from tests.spgemm_oracle import hash_slot

    j = np.arange(ts * ts // tail, dtype=np.int64)      # about twice the columns needed
    cols = j[hash_slot(j, ts) >= ts - tail][:ts // 2]
    n = int(cols[-1]) + 1
    b = [np.sort(x) for x in np.array_split(rng.permutation(cols), parts)]
    b.append(rng.choice(np.setdiff1d(np.arange(n), cols), 300, replace=False))
    return _product([list(range(parts)), list(range(0, parts, 3)), [parts, 1]], b, parts + 1, n, rng)


def _capped(n, full, a_full, rng):
    """n columns, `full` B rows holding all of them, then rows of 3000, 2000, 100 and 30 random columns; A rows a_full
    (over the full rows) first, then [full, full + 1] and [full + 2, full + 3]."""
    b = [np.arange(n)] * full + [_some(n, min(d, n), rng) for d in (3000, 2000, 100, 30)]
    return _product(a_full + [[full, full + 1], [full + 2, full + 3]], b, full + 4, n, rng)


def _bitmap_words(n, rng):
    """n columns: rows of 3000 random columns with column 0, with column n - 1, the lower and upper half of n."""
    h = n // 2
    b = [_some(n, 3000, rng, [0]), _some(n, 3000, rng, [n - 1]), np.arange(h), np.arange(h, n)]
    return _product([[0, 1], [2, 3], [1, 3], [0]], b, 4, n, rng)


def _grid_loops(rng):
    """More rows in every tier than its launch has row slots: 140 bitmap rows (two of 40 B rows of 2100-2600 columns
    each), 300 block rows (two of 60 B rows of 150-400), 9000 warp rows (one to three of 1000 B rows of 1-60), in a
    random row order; n = 9000."""
    n = 9000
    wide = [_some(n, int(d), rng) for d in rng.integers(2100, 2601, 40)]
    mid = [_some(n, int(d), rng) for d in rng.integers(150, 401, 60)]
    small = [_some(n, int(d), rng) for d in rng.integers(1, 61, 1000)]

    def pairs(count, lo, hi):
        ij = np.array([(i, j) for i in range(lo, hi) for j in range(i + 1, hi)])
        return [list(p) for p in ij[rng.choice(len(ij), count, replace=False)]]

    a = pairs(140, 0, 40) + pairs(300, 40, 100)
    a += [list(rng.choice(np.arange(100, 1100), int(d), replace=False)) for d in rng.integers(1, 4, 9000)]
    a = [a[i] for i in rng.permutation(len(a))]
    return _product(a, wide + mid + small, 1100, n, rng)


def _value_rows(kind, rng):
    """One row per tier (B rows of 100, 1000 and 4500 columns, n = 10000), each over three B rows P, Q, P2:
      cancel     P2 = P with negated values, A's values on P and P2 equal and every product exact (small dyadic
                 values): the columns outside Q sum to exactly +0.0 (Q lies between P and P2 in A's row)
      subnormal  P's values and A's on P of order 2^-70 (products near 2^-140), Q's values subnormal (2^-130)
      negzero    A's value on P is -0.0, a quarter of P's and Q's values are -0.0: columns outside Q have only
                 -0.0 products."""
    n = 10000
    g = lambda size: rng.standard_normal(size).astype(np.float32)  # noqa: E731
    a, b, va, vb = [], [], [], []
    for t, (d, q) in enumerate(((100, 50), (1000, 300), (4500, 1000))):
        P, Q = _some(n, d, rng), _some(n, q, rng)
        b += [P, Q, P]
        vp, vq, ap, aq = g(d), g(q), g(1)[0], g(1)[0]
        if kind == "cancel":
            vp = (rng.integers(1, 65, d) * rng.choice([-1, 1], d) / 4).astype(np.float32)
            ap = np.float32(rng.choice([-3, -1.5, -1, -0.5, 0.5, 1, 1.5, 3]))
            a.append([3 * t, 3 * t + 1, 3 * t + 2])
            va.append([ap, aq, ap])
            vb += [vp, vq, -vp]
            continue
        if kind == "subnormal":
            ap, vp, vq = ap * 2.0 ** -70, vp * 2.0 ** -70, vq * 2.0 ** -130
        else:
            ap = -0.0
            vp[rng.random(d) < 0.25] = -0.0
            vq[rng.random(q) < 0.25] = -0.0
        a.append([3 * t, 3 * t + 1])
        va.append([ap, aq])
        vb += [vp, vq, g(d)]
    return _product(a, b, len(b), n, rng, va, vb)


def _bwd_terms(d, rng):
    """Backward entries of d terms: B row 0 holds d columns and A column 0 three entries (dA), A column 1 d entries and
    B row 1 three columns (dB); column / row 2 hold a few more."""
    m, n = d + 4, d + 7
    rows = [[] for _ in range(m)]
    for i in (0, 1, 2):
        rows[i].append(0)
    for i in rng.choice(m, d, replace=False):
        rows[i].append(1)
    for i in rng.choice(m, 5, replace=False):
        rows[i].append(2)
    b = [_some(n, d, rng), _some(n, 3, rng), _some(n, 4, rng)]
    return _product(rows, b, 3, n, rng)


def _bwd_duplicates(rng):
    """A (80 x 60) and B (60 x 90) of 600 random entries each, 150 of them given a second copy and 30 a third."""
    out = []
    for r, c in ((80, 60), (60, 90)):
        row, col = rng.integers(0, r, 600), rng.integers(0, c, 600)
        row = np.concatenate([row, row[:150], row[:30]])
        col = np.concatenate([col, col[:150], col[:30]])
        out.append((row, col, rng.standard_normal(row.size).astype(np.float32)))
    return out[0], out[1], 80, 60, 90


def _random_rows(k, n, lens, degs, rng):
    """A rows of `lens` random B rows, B rows of `degs` random columns."""
    return _product([rng.choice(k, int(x), replace=False) for x in lens], [_some(n, int(d), rng) for d in degs], k,
                    n, rng)


SPGEMM_CASES = {
    # rows without work, degenerate shapes
    "empty-rows": lambda r: _product([[0, 1, 2], [], [0, 4], [3], [5, 6, 7], []],
                                     [[], [], [], []] + [_some(50, 8, r) for _ in range(4)], 8, 50, r),
    "m0": lambda r: _random_rows(5, 7, [], [3, 0, 5, 1, 7], r),
    "k0": lambda r: _product([[]] * 5, [], 0, 7, r),
    "n0": lambda r: _product([[0, 2], [], [1, 2, 3], [3], [0]], [[]] * 4, 4, 0, r),
    "A-empty": lambda r: _product([[]] * 6, [_some(7, 3, r) for _ in range(5)], 5, 7, r),
    "B-empty": lambda r: _product([[0, 2], [], [1, 2, 3], [4], [0], [1]], [[]] * 5, 5, 7, r),
    "rect": lambda r: _random_rows(130, 6000,[1, 20, 60] + list(r.integers(1, 61, 47)),
                                   r.integers(40, 201, 130), r),
    # the warp tier: 512-slot tables
    "warp-counts": lambda r: _counts([1, 255, 256, 100, 155, 3], [[0], [1], [2], [3, 5], [4, 3, 0], []], r),
    "warp-bound256-c1": lambda r: _product([list(range(256)), list(range(200)), list(range(257)), [257, 258]],
                                           [[7]] * 256 + [[8]] + [_some(300, 20, r) for _ in range(2)], 259, 300, r),
    "warp-hash-wrap": lambda r: _wrap(512, 8, 4, r),
    "warp-n-capped": lambda r: _capped(200, 25, [list(range(25)), [0, 1]], r),
    # the block tier: 8192-slot tables
    "block-counts": lambda r: _counts([257, 4095, 4096, 2000, 2096, 1, 2094],
                                      [[0], [1], [2], [3, 4], [3, 5, 6], [6, 0]], r),
    "block-bound300-c2": lambda r: _product([list(range(150)), list(range(128)), [150, 151]],
                                            [[3, 250]] * 150 + [_some(400, 30, r) for _ in range(2)], 152, 400, r),
    "block-hash-wrap": lambda r: _wrap(8192, 64, 16, r),
    "block-n-capped": lambda r: _capped(4096, 3, [[0, 1, 2], [1]], r),
    # the bitmap tier: n columns in 32-bit words
    "bitmap-counts": lambda r: _counts([4097, 4096, 1, 2000, 2097, 3000], [[0], [1, 2], [3, 4], [1], [5, 3]], r),
    "bitmap-bound5000-c3": lambda r: _product([list(range(2500)), list(range(1200)), [0]],
                                              [sorted({q % 3, (q + 1) % 3}) for q in range(2500)], 2500, 6000, r),
    "bitmap-full": lambda r: _product([[0, 1], [0], [2], [3, 2]],
                                      [np.arange(3000), np.arange(2000, 5000), np.arange(5000), _some(5000, 50, r)],
                                      4, 5000, r),
    "bitmap-n32w+1": lambda r: _product([[0, 1], [1], [0]],
                                        [_some(6401, 4200, r, [0, 31, 32, 63, 64, 6400]), _some(6401, 300, r)], 2,
                                        6401, r),
    "bitmap-n8192": lambda r: _bitmap_words(8192, r),
    "bitmap-n8193": lambda r: _bitmap_words(8193, r),
    # every tier's grid-stride loop
    "grid-loops": _grid_loops,
    # values
    "cancel": lambda r: _value_rows("cancel", r),
    "subnormal": lambda r: _value_rows("subnormal", r),
    "negzero": lambda r: _value_rows("negzero", r),
    # the backward
    **{f"bwd-{d}": (lambda r, d=d: _bwd_terms(d, r)) for d in (1, 31, 32, 33, 65, 2000)},
    "bwd-duplicates": _bwd_duplicates,
}


def spgemm_case(name, seed=0):
    """(A, B, m, k, n) of a sparse x sparse product case (SPGEMM_CASES)."""
    return SPGEMM_CASES[name](np.random.default_rng(seed))

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

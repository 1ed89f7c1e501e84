"""Row ends of the row-stream SpMM's segments (stream.cuh, stream_range_lean): the column-panel passes find the rows
whose last edge falls inside a 32-edge slab from rowptr with a row cursor, the one-pass form from edge_row.  These
graphs put row ends where that is easy to get wrong: empty rows at the start and end of the graph and of segments and
runs of them longer than a slab, rows ending on slab boundaries, more than 32 rows ending inside one slab, one-row
segments, hub rows next to empty rows.

Every panel count must give bitwise the output of the single-pass kernel, rows the hub plan does not split must be
bitwise equal to the oracle, split rows within float rounding of it, and the plan's arrival counters must be left
at zero.
"""
import numpy as np
import pytest
import torch

import oracle
from tests.gpu_util import bits, dev

pytestmark = pytest.mark.gpu

CHUNK = 64


def from_degrees(deg, seed):
    deg = np.asarray(deg, dtype=np.int64)
    rp = np.zeros(deg.size + 1, np.int32)
    rp[1:] = np.cumsum(deg)
    n_cols = max(deg.size, 1)
    ci = np.random.default_rng(seed).integers(0, n_cols, int(rp[-1])).astype(np.int32)
    return rp, ci, n_cols


def graph(name):
    rng = np.random.default_rng(11)
    if name == "empty_runs":          # empty rows first and last, and runs of 1, 31, 32, 33 and 70 in between
        deg = [0] * 40
        for run in (1, 31, 32, 33, 70, 5):
            deg += list(rng.integers(1, 20, 7)) + [0] * run
        deg += list(rng.integers(1, 40, 30)) + [0] * 45
    elif name == "slab_aligned":      # row ends on multiples of 32 edges, and one edge either side of them
        deg = [32] * 20 + [16, 16] * 5 + [8] * 12 + [31, 1, 33, 31] * 6 + [32, 0, 32, 0, 0, 32] * 4
    elif name == "unit_rows":         # 40+ rows end inside one slab: 1-edge rows, some with empty rows between
        deg = [1] * 100 + [1, 0] * 50 + [2, 0, 0] * 30 + [1] * 33
    elif name == "hubs":              # hub rows (> CHUNK edges) between empty rows and short rows
        deg = [0] * 3 + [500] + [0] * 40 + [3, 1, 0, 65] + [0] * 33 + [700, 2] + list(rng.integers(0, 12, 200)) + [64, 0, 300]
    else:                             # mixed: random degrees with half of the rows empty
        deg = np.where(rng.random(2000) < 0.5, 0, rng.integers(1, 90, 2000))
    return from_degrees(deg, seed=len(name))


GRAPHS = ["empty_runs", "slab_aligned", "unit_rows", "hubs", "mixed"]
# panel counts the SpMM accepts at each width (a panel is 32, 64 or 128 floats); F = 9 takes the scalar lean loop
WIDTHS = {9: [1], 40: [1], 64: [1, 2], 128: [1, 2, 4], 256: [1, 2, 4]}


@pytest.mark.parametrize("name", GRAPHS)
@pytest.mark.parametrize("seg_cost", [None, 1, 4096])   # default segments, one row per segment, long segments
@pytest.mark.parametrize("F", sorted(WIDTHS))
@pytest.mark.parametrize("weighted", [True, False])
def test_row_ends_from_rowptr(dev, name, seg_cost, F, weighted):
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import spmm_raw
    from cogdl_b200.structure import CSRStructure

    rp, ci, n_cols = graph(name)
    rng = np.random.default_rng(5)
    X = rng.standard_normal((n_cols, F)).astype(np.float32)
    val = rng.random(ci.shape[0]).astype(np.float32) if weighted else None
    ref = oracle.spmm_csr(rp, ci, val, X)
    st = CSRStructure(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), n_cols=n_cols, chunk_edges=CHUNK,
                      seg_cost=seg_cost)
    plan = st.plan
    assert plan.n_segs > 0
    if seg_cost == 1:
        segs = plan.segs.view(-1, 2).cpu().numpy()
        assert (segs[:, 1] - segs[:, 0] == 1).any(), "no one-row segment"
    x_d = torch.from_numpy(X).to(dev)
    v_d = None if val is None else torch.from_numpy(val).to(dev)
    deg = np.diff(rp)
    unsplit = deg <= CHUNK
    scale = np.abs(ref).max(axis=1, keepdims=True) + 1e-30

    y1 = spmm_raw(st, v_d, x_d, panels=1)
    assert "stream_kernel" in _cabi.last_kernel(), _cabi.last_kernel()
    for P in WIDTHS[F]:
        y = spmm_raw(st, v_d, x_d, panels=P)
        note = _cabi.last_kernel()
        assert (f",panels={P}" in note) if P > 1 else ("panels=" not in note), note
        assert torch.equal(bits(y), bits(y1)), f"panels={P} differs from the single-pass kernel ({note})"
        yn = y.cpu().numpy()
        assert np.array_equal(yn[unsplit], ref[unsplit]), f"panels={P}: unsplit rows differ from the oracle ({note})"
        assert not yn[deg == 0].any(), "empty rows must be zero"
        assert (np.abs(yn - ref) / scale).max() <= 1e-5, f"panels={P}: split rows differ from the oracle ({note})"
        assert int(plan.counters.abs().sum()) == 0, "arrival counters must be left zero"

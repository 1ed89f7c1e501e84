"""Every kernel compiled into genconv_edge.o has a row in tests/genconv_edge_table.py that the GPU suite runs
(test_gpu_genconv_edge.py), and every kernel the table names is compiled, checked on a machine without a GPU."""
import re

from tests.genconv_edge_table import (DS, FS, GE_BWD_BLOCKS, GE_WARPS, MAX_D, TABLE, TILE_FS, required_special_forms,
                                      special_form, wide_csr)
from tests.test_cpu_kernel_inventory import assert_table_covers, canonical


def note_of(sym):
    """The name cogdl_b200_last_kernel() records for a demangled genconv_edge.o kernel symbol."""
    if re.match(r"cogdl_b200::genconv_edge_dw_reduce_kernel\(", sym):
        return "cogdl_b200::genconv_edge_dw_reduce_kernel"
    m = re.match(r"void cogdl_b200::genconv_edge_(fwd|bwd)_kernel<\(int\)([14]), \(int\)(\d+)(?:, \(bool\)([01]))?>", sym)
    assert m, f"no last_kernel() name is known for {sym!r}: add it to note_of() and a row to the table"
    op, w, dm, q = m.groups()
    v = "float4" if w == "4" else "float"
    if op == "fwd":
        return f"cogdl_b200::genconv_edge_fwd_kernel<{v},DM={dm},{'Q' if q == '1' else 'no_Q'}>"
    return f"cogdl_b200::genconv_edge_bwd_kernel<{v},DM={dm}>"


def test_genconv_edge_table_covers_every_compiled_kernel():
    table = {k for c in TABLE for k in canonical(c.kernel)}
    assert_table_covers("genconv_edge", note_of, table, "tests/genconv_edge_table.py")


def test_genconv_edge_rows_are_distinct_and_cover_the_shapes():
    ids = [c.id for c in TABLE]
    assert len(ids) == len(set(ids))
    for op in ("fwd", "bwd"):
        rows = [c for c in TABLE if c.op == op]
        assert set(FS) <= {c.F for c in rows} and set(DS) <= {c.D for c in rows}
        assert {1, MAX_D} <= {c.D for c in rows}
        assert {"hub", "two_hubs", "ragged", "rect", "empty_graph"} <= {c.graph for c in rows}
        assert any(not c.aligned for c in rows) and any(c.F > 128 for c in rows)
    assert {c.want for c in TABLE if c.op == "bwd"} == {"dx_dw", "dx", "dw"}


def test_genconv_edge_rows_cover_every_special_form():
    """The exact family's beta sweep (cancelling pre-activations included), no hub plan, the boundary-degree graphs,
    the misaligned partial scratch, a partial last tile among several and the wide grid each have exactly one row per
    instantiation they apply to, so removing any of those rows fails here."""
    forms = [special_form(c) for c in TABLE if special_form(c) is not None]
    required = required_special_forms()
    missing = sorted(required - set(forms), key=str)
    assert not missing, "special forms without a row in tests/genconv_edge_table.py:\n" + "\n".join(
        f"  {f}" for f in missing)
    extra = sorted(set(forms) - required, key=str)
    assert not extra, f"rows in special forms no check asks for: {extra}"
    dup = sorted({f for f in forms if forms.count(f) > 1}, key=str)
    assert not dup, f"several rows of one special form: {dup}"


def test_wide_graph_outgrows_the_backward_grid():
    """The wide graph's transpose has more work items than the backward's 8 x GE_BWD_BLOCKS warps even before its hub
    chunks are counted, and the boundary rows sit on a hub plan's chunk edges."""
    import numpy as np

    rp, ci, n = wide_csr()
    assert n > GE_WARPS * GE_BWD_BLOCKS
    assert np.bincount(ci, minlength=n).max() > 16            # hub columns at chunk 16: dX merges, then more items
    assert all(c.chunk in (16, 64) for c in TABLE if c.graph.startswith("bounds"))
    assert {c.F for c in TABLE if special_form(c) and special_form(c)[0] == "tile"} == set(TILE_FS)


def test_note_of_maps_genconv_edge_symbols():
    assert note_of("void cogdl_b200::genconv_edge_fwd_kernel<(int)4, (int)8, (bool)1>(cogdl_b200::GeFwdParams)") == \
        "cogdl_b200::genconv_edge_fwd_kernel<float4,DM=8,Q>"
    assert note_of("void cogdl_b200::genconv_edge_bwd_kernel<(int)1, (int)16>(cogdl_b200::GeBwdParams)") == \
        "cogdl_b200::genconv_edge_bwd_kernel<float,DM=16>"
    assert note_of("cogdl_b200::genconv_edge_dw_reduce_kernel(const float *, int, long, float *)") == \
        "cogdl_b200::genconv_edge_dw_reduce_kernel"

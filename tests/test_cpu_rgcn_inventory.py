"""Every kernel compiled into rgcn.o has a row in tests/rgcn_table.py that the GPU suite runs (test_gpu_rgcn.py), and
every kernel the table names is compiled, checked on a machine without a GPU."""
import re

from tests.rgcn_table import BASIS_TILE, BS, FS, TABLE, TS
from tests.test_cpu_kernel_inventory import assert_table_covers


def note_of(sym):
    """The name cogdl_b200_last_kernel() records for a demangled rgcn.o kernel symbol."""
    m = re.match(r"void cogdl_b200::(rgcn_fanout_kernel|rgcn_edge_dot_kernel)<(float4|float)(?:, \(bool\)([01]))?>", sym)
    assert m, f"no last_kernel() name is known for {sym!r}: add it to note_of() and a row to the table"
    name, vec, per_basis = m.groups()
    return f"cogdl_b200::{name}<{vec}{',per_basis' if per_basis == '1' else ''}>"


def test_rgcn_table_covers_every_compiled_kernel():
    assert_table_covers("rgcn", note_of, {c.kernel for c in TABLE}, "tests/rgcn_table.py")


def test_rgcn_rows_are_distinct_and_cover_the_shapes():
    ids = [c.id for c in TABLE]
    assert len(ids) == len(set(ids))
    for op in ("aggr", "per_basis", "dot"):
        rows = [c for c in TABLE if c.op == op]
        assert set(FS) <= {c.F for c in rows} and set(BS) <= {c.B for c in rows} and set(TS) <= {c.T for c in rows}
        assert {BASIS_TILE, BASIS_TILE + 1} <= {c.B for c in rows}
        assert {"hub", "two_hubs", "ragged", "bounds"} <= {c.graph for c in rows}
        assert any(not c.aligned for c in rows)


def test_note_of_maps_rgcn_symbols():
    assert note_of("void cogdl_b200::rgcn_fanout_kernel<float4, (bool)0>(cogdl_b200::RgcnParams)") == \
        "cogdl_b200::rgcn_fanout_kernel<float4>"
    assert note_of("void cogdl_b200::rgcn_fanout_kernel<float, (bool)1>(cogdl_b200::RgcnParams)") == \
        "cogdl_b200::rgcn_fanout_kernel<float,per_basis>"
    assert note_of("void cogdl_b200::rgcn_edge_dot_kernel<float4>(cogdl_b200::RgcnParams)") == \
        "cogdl_b200::rgcn_edge_dot_kernel<float4>"

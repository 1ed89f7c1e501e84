"""Every kernel compiled into label_prop.o has a row in tests/label_prop_table.py that the GPU suite runs
(test_gpu_label_prop.py), and every kernel the table names is compiled, checked on a machine without a GPU.  The
symbols are mapped to their recorded names by test_cpu_kernel_inventory.py's note_of()."""
from tests.label_prop_table import TABLE
from tests.test_cpu_kernel_inventory import assert_table_covers, canonical, note_of


def test_label_prop_table_covers_every_compiled_kernel():
    table = {k for c in TABLE for k in canonical(c.kernel)}
    assert_table_covers("label_prop", note_of, table, "tests/label_prop_table.py")


def test_label_prop_rows_are_distinct_and_cover_every_epilogue():
    ids = [c.id for c in TABLE]
    assert len(ids) == len(set(ids))
    assert all(c.z for c in TABLE if c.pin), "a pinned row is Z's row"
    assert {(c.clamp, c.pin) for c in TABLE} == {(True, True), (True, False), (False, True), (False, False)}
    assert {(c.z, c.row_scale) for c in TABLE} == {(True, True), (True, False), (False, True), (False, False)}
    assert {1, 7, 16, 40, 47, 64, 128} <= {c.F for c in TABLE}
    assert {2, 4} <= {c.panels for c in TABLE}
    assert {"none", "chunks", "default"} == {c.plan for c in TABLE}
    assert any(not c.aligned for c in TABLE)
    assert {(c.clamp, c.pin) for c in TABLE if c.graph == "bounds"} == {(True, True), (True, False), (False, True),
                                                                         (False, False)}
    for kernel in {k for c in TABLE for k in canonical(c.kernel)}:
        rows = [c for c in TABLE if kernel in canonical(c.kernel)]
        assert any(c.clamp or c.pin for c in rows), kernel


def test_note_of_maps_label_prop_symbols():
    assert note_of("void cogdl_b200::stream_kernel<float4, (int)1, (int)1, (bool)0, (int)0, (int)4, (int)4, (bool)0, "
                   "(bool)0, (bool)0, (int)2>(cogdl_b200::StreamParams)") == \
        "cogdl_b200::stream_labelprop_kernel<float4,NV=1,weighted,SRC_ONE,U=4,MINB=4>"
    assert note_of("void cogdl_b200::spmm_kernel<float, (int)32, (int)4, (bool)0, (int)2>(cogdl_b200::SpmmParams)") \
        == "cogdl_b200::spmm_labelprop_kernel<float,GROUP=32,NV=4,unweighted>"

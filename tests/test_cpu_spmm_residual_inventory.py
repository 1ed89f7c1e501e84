"""Every kernel compiled into spmm_residual.o has a row in tests/spmm_residual_table.py that the GPU suite runs
(test_gpu_spmm_residual.py), and every kernel the table names is compiled, checked on a machine without a GPU.  The
kernel entry points are read from the object and mapped to the string their launchers record for
cogdl_b200_last_kernel() by test_cpu_kernel_inventory.py."""
from tests.spmm_residual_table import TABLE
from tests.test_cpu_kernel_inventory import assert_table_covers, canonical, note_of


def test_residual_table_covers_every_compiled_kernel():
    table = {k for c in TABLE for k in canonical(c.kernel)}
    assert_table_covers("spmm_residual", note_of, table, "tests/spmm_residual_table.py")


def test_residual_rows_are_distinct_and_cover_both_epilogue_inputs():
    ids = [c.id for c in TABLE]
    assert len(ids) == len(set(ids))
    for kernel in {k for c in TABLE for k in canonical(c.kernel)}:
        rows = [c for c in TABLE if kernel in canonical(c.kernel)]
        assert any(c.z for c in rows) or any(c.row_scale for c in rows), kernel
    assert {(c.z, c.row_scale) for c in TABLE} == {(True, True), (True, False), (False, True), (False, False)}
    assert {1, 7, 16, 40, 64, 128, 256} <= {c.F for c in TABLE}
    assert {2, 4} <= {c.panels for c in TABLE}
    assert {"none", "chunks", "default"} == {c.plan for c in TABLE}
    assert any(not c.aligned for c in TABLE) and any(c.graph == "bounds" for c in TABLE)


def test_note_of_maps_residual_symbols():
    assert note_of("void cogdl_b200::stream_kernel<float4, (int)1, (int)1, (bool)0, (int)0, (int)4, (int)4, (bool)0, "
                   "(bool)0, (bool)0, (int)1>(cogdl_b200::StreamParams)") == \
        "cogdl_b200::stream_residual_kernel<float4,NV=1,weighted,SRC_ONE,U=4,MINB=4>"
    assert note_of("void cogdl_b200::spmm_kernel<float, (int)32, (int)4, (bool)0, (int)1>(cogdl_b200::SpmmParams)") \
        == "cogdl_b200::spmm_residual_kernel<float,GROUP=32,NV=4,unweighted>"

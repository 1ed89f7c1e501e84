"""Every kernel compiled into gin.o and spmm_accum.o has a row in tests/gin_grand_table.py that the GPU suite runs
(test_gpu_gin_grand.py), and every kernel the table names is compiled, checked on a machine without a GPU.  The symbols
are mapped to their recorded names by test_cpu_kernel_inventory.py's note_of()."""
from tests.gin_grand_table import TABLE
from tests.test_cpu_kernel_inventory import assert_table_covers, canonical, note_of


def _check(obj, epi):
    table = {k for c in TABLE if c.epi == epi for k in canonical(c.kernel)}
    compiled = assert_table_covers(obj, note_of, table, "tests/gin_grand_table.py")
    assert all(f"_{epi}_kernel<" in n for n in compiled), sorted(compiled)


def test_gin_table_covers_every_compiled_kernel():
    _check("gin", "dcoef")


def test_accum_table_covers_every_compiled_kernel():
    _check("spmm_accum", "accum")


def test_gin_grand_rows_are_distinct_and_cover_every_epilogue_form():
    ids = [c.id for c in TABLE]
    assert len(ids) == len(set(ids))
    dc = [c for c in TABLE if c.epi == "dcoef"]
    ac = [c for c in TABLE if c.epi == "accum"]
    assert {(c.z, c.row_scale) for c in dc} == {(True, True), (True, False), (False, True), (False, False)}
    assert {(c.last, c.in_place) for c in ac} == {(True, True), (True, False), (False, True), (False, False)}
    assert {False, True} == {c.row_scale for c in ac}
    for rows in (dc, ac):
        assert {1, 7, 16, 40, 47, 64, 128, 256} <= {c.F for c in rows}
        assert {2, 4} <= {c.panels for c in rows}
        assert {"none", "chunks", "default"} == {c.plan for c in rows}
        assert any(not c.aligned for c in rows) and any(c.graph == "bounds" for c in rows)


def test_note_of_maps_gin_grand_symbols():
    assert note_of("void cogdl_b200::stream_kernel<float4, (int)1, (int)1, (bool)0, (int)0, (int)4, (int)4, (bool)0, "
                   "(bool)0, (bool)0, (int)4>(cogdl_b200::StreamParams)") == \
        "cogdl_b200::stream_accum_kernel<float4,NV=1,weighted,SRC_ONE,U=4,MINB=4>"
    assert note_of("void cogdl_b200::spmm_kernel<float, (int)32, (int)4, (bool)0, (int)3>(cogdl_b200::SpmmParams)") \
        == "cogdl_b200::spmm_dcoef_kernel<float,GROUP=32,NV=4,unweighted>"

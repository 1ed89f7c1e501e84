"""Every kernel compiled into simple_hgn.o has a row in tests/hgn_table.py that the GPU suite runs
(test_gpu_simple_hgn.py), and every kernel the table names is compiled, checked on a machine without a GPU.  The symbols
are mapped to their recorded names by test_cpu_kernel_inventory.py's note_of()."""
from tests.hgn_table import MAX_TABLE, TABLE, form_key
from tests.test_cpu_kernel_inventory import assert_table_covers, note_of


def table_kernels():
    names = set()
    for c in TABLE:
        for mode in (2, 3):
            names.add(c.kernel(mode))
            if c.stats(mode):
                names.add(c.stats(mode))
    return names


def test_hgn_table_covers_every_typed_kernel():
    compiled = assert_table_covers("simple_hgn", note_of, table_kernels(), "tests/hgn_table.py")
    assert all(n.startswith("cogdl_b200::hgn_") for n in compiled), sorted(compiled)


def test_hgn_rows_are_distinct_and_cover_the_shapes():
    ids = [c.id for c in TABLE]
    assert len(ids) == len(set(ids))
    assert {1, 2, 8} <= {c.H for c in TABLE}
    assert {1, 5} <= {c.T for c in TABLE} and any(c.T * c.H == MAX_TABLE for c in TABLE)
    graphs = {"tiny", "empty_graph", "ragged", "hub", "two_hubs", "rect", "bounds", "bounds_t"}
    assert graphs <= {c.graph for c in TABLE}
    assert {(r, p) for c in TABLE for r, p in [(c.res, c.p)]} == {(False, 0.0), (False, 0.5), (True, 0.0), (True, 0.5)}


def test_hgn_rows_cover_every_launch_form():
    """Every launch form (the main kernel at each tile, the warp and the generic kernel) has rows, so its forward also
    runs without the attention output (test_row_against_fp64 repeats every row's forward that way), and one row whose
    backward walks boundary-degree columns (bounds_t); one row blends with alpha = 1.  Removing any bounds_t row fails
    here."""
    forms = {form_key(c) for c in TABLE}
    assert forms == {"main-512", "main-1024", "main-2048", "warp", "generic"}, forms
    bounds_t = sorted(form_key(c) for c in TABLE if c.graph == "bounds_t")
    assert bounds_t == sorted(["main-512", "main-512", "main-1024", "main-2048", "warp", "generic"]), bounds_t
    assert {1, 8, 16, 3} <= {c.H for c in TABLE if c.graph == "bounds_t"}
    assert any(c.alpha == 1.0 and c.res for c in TABLE)


def test_note_of_maps_hgn_symbols():
    assert note_of("void cogdl_b200::es_main_kernel<(int)2, (int)512, (bool)1, (bool)1, (bool)0>(cogdl_b200::EsParams)") \
        == "cogdl_b200::hgn_main_kernel<MODE=2,CAP=512,DROP>"
    assert note_of("void cogdl_b200::es_warp_kernel<(int)2, (bool)0, (bool)1, (bool)1>(cogdl_b200::EsParams)") == \
        "cogdl_b200::hgn_warp_kernel<MODE=2,MIX>"
    assert note_of("void cogdl_b200::es_stats_kernel<(int)3, (bool)1, (bool)1>(cogdl_b200::EsParams)") == \
        "cogdl_b200::hgn_stats_kernel<MODE=3>"

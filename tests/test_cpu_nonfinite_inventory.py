"""tests/nonfinite_table.py against include/cogdl_b200.h, without a GPU: every entry point that takes a float operand has
a non-finite row, an exemption or a pending entry with its reason, and no row that alone covers an entry goes missing."""
import pytest

from tests import nonfinite_table as NT
from tests.graphs import CASES
from tests.test_cpu_large_offset_inventory import HEADER, dense_entries


def check_inventory(text):
    covered = {c.entry for c in NT.TABLE}
    missing = dense_entries(text) - covered - set(NT.EXEMPT) - set(NT.NOT_COVERED)
    assert not missing, f"entry points with a float operand and no non-finite row or reason: {sorted(missing)}"


def test_every_float_entry_point_has_a_row_or_a_reason():
    check_inventory(open(HEADER).read())
    for reason in list(NT.EXEMPT.values()) + list(NT.NOT_COVERED.values()):
        assert reason.strip()
    covered = {c.entry for c in NT.TABLE}
    assert not (set(NT.EXEMPT) & covered) and not (set(NT.NOT_COVERED) & covered) and not (set(NT.EXEMPT) & set(NT.NOT_COVERED))


def test_a_new_entry_point_without_a_row_fails():
    text = open(HEADER).read() + "\nCOGDL_B200_API int cogdl_b200_fake_f32(const float *X, float *Y, int64_t n);\n"
    with pytest.raises(AssertionError, match="cogdl_b200_fake_f32"):
        check_inventory(text)


def test_every_named_entry_is_in_the_header():
    text = open(HEADER).read()
    dense = dense_entries(text)
    for entry in {c.entry for c in NT.TABLE} | set(NT.NOT_COVERED):
        assert entry in dense, f"{entry}: not an entry point of the header with a float operand"
    for entry in NT.EXEMPT:
        assert f"COGDL_B200_API int {entry}(" in text, f"{entry}: not an entry point of the header"


# Every row id.  A row that goes missing from the table fails here, even when its entry point keeps other rows.
ROW_IDS = {
    "disen_route_fwd-overflow-K3F6",
    "edge_softmax-logits-H1",
    "edge_softmax-logits-H4",
    "edge_softmax_bwd-grad_out-H4",
    "edge_softmax_bwd-saved-H4",
    "gat_attn_bwd-grad_out-H4",
    "gat_attn_bwd-saved-H4",
    "gat_attn_bwd_dropout-grad_out-H4",
    "gat_attn_bwd_dropout-saved-H4",
    "gcn_fused-features-K128",
    "gcn_fused-overflow-K128",
    "genconv_edge_fwd-features-F67",
    "hgn_attn-logits-H4",
    "hgn_attn_bwd-grad_out-H4",
    "hgn_attn_bwd-saved-H4",
    "mhspmm-attention-H4F11",
    "mhspmm_dropout-attention-H4F11",
    "residual-Z-F67",
    "residual_dcoef-b_dev-F67",
    "sage_fused-max-features-K128",
    "sage_fused-mean-features-K128",
    "sage_fused-sum-features-K128",
    "scatter_max-features-F67",
    "scatter_max_bwd-grad_out-F67",
    "sddmm-features-F67",
    "softmax_aggr_bwd-grad_out-F67",
    "softmax_aggr_bwd-overflow-F67",
    "softmax_aggr_fwd-edge_term-F67",
    "softmax_aggr_fwd-features-F67",
    "softmax_aggr_fwd-overflow-F67",
    "spmm-features-F67",
    "spmm-weights-F67",
    "spmm_f16-overflow-F66",
}


def test_no_row_is_dropped():
    ids = [c.id for c in NT.TABLE]
    assert len(ids) == len(set(ids)), "duplicate row ids"
    missing = ROW_IDS - set(ids)
    assert not missing, f"rows removed from the table: {sorted(missing)}"
    assert set(ids) == ROW_IDS, f"new rows, add them to ROW_IDS: {sorted(set(ids) - ROW_IDS)}"


def test_dropping_a_sole_row_fails():
    sole = [c for c in NT.TABLE if sum(d.entry == c.entry for d in NT.TABLE) == 1]
    assert sole
    for c in sole:
        saved = NT.TABLE[:]
        try:
            NT.TABLE.remove(c)
            with pytest.raises(AssertionError, match=c.entry):
                check_inventory(open(HEADER).read())
        finally:
            NT.TABLE[:] = saved


@pytest.mark.parametrize("c", NT.TABLE, ids=lambda c: c.id)
def test_row_shape(c):
    fixed = c.entry in ("cogdl_b200_gcn_fused_f32", "cogdl_b200_sage_fused_f32")   # K = 128 is the only width
    if not fixed and c.entry != "cogdl_b200_edge_softmax_fwd_f32":
        assert c.F % 4 != 0, f"{c.id}: F = {c.F} has no F % 4 tail"
    assert c.graph == "bounds" or c.graph in CASES

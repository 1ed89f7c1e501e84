"""tests/large_offset_table.py against include/cogdl_b200.h, without a GPU: every entry point that takes a dense float
operand has a large-offset row or an exemption with its reason, and every row's shape does what its role says."""
import os
import re

import pytest

from tests import large_offset_table as LT

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HEADER = os.path.join(ROOT, "include", "cogdl_b200.h")


def dense_entries(text):
    """Names of the COGDL_B200_API functions returning int whose parameters include a float, half (void *) or packed
    byte operand."""
    out = set()
    for m in re.finditer(r"COGDL_B200_API\s+int\s+(cogdl_b200_\w+)\s*\(([^;]*)\)\s*;", text):
        name, params = m.group(1), m.group(2)
        if re.search(r"\bfloat\s*\*|\bvoid\s*\*|\buint8_t\s*\*", params):
            out.add(name)
    return out


def test_header_parse_finds_the_known_entries():
    names = dense_entries(open(HEADER).read())
    assert {"cogdl_b200_spmm_csr_f32_ex", "cogdl_b200_spmm_csr_f16", "cogdl_b200_gat_fwd_f32",
            "cogdl_b200_actnn_unpack_f32"} <= names


def check_inventory(text):
    covered = {c.entry for c in LT.TABLE}
    missing = dense_entries(text) - covered - set(LT.EXEMPT)
    assert not missing, f"entry points with a dense operand and no large-offset row or exemption: {sorted(missing)}"


def test_every_dense_entry_point_has_a_row_or_a_reason():
    check_inventory(open(HEADER).read())
    for reason in LT.EXEMPT.values():
        assert reason.strip()
    assert not (set(LT.EXEMPT) & {c.entry for c in LT.TABLE})


def test_a_new_entry_point_without_a_row_fails():
    text = open(HEADER).read() + "\nCOGDL_B200_API int cogdl_b200_fake_f32(const float *X, float *Y, int64_t n);\n"
    with pytest.raises(AssertionError, match="cogdl_b200_fake_f32"):
        check_inventory(text)


def test_every_table_row_entry_is_in_the_header():
    dense = dense_entries(open(HEADER).read())
    for entry in {c.entry for c in LT.TABLE}:
        assert entry in dense, f"{entry}: not an entry point of the header with a dense operand"


# Every row id.  A row that goes missing from the table fails here, even when its entry point keeps other rows.
ROW_IDS = {
    "accum-F124",
    "accum-last-F300-chunks",
    "actnn-dropout",
    "actnn-dropout_bwd",
    "actnn-minmax",
    "actnn-pack",
    "actnn-relu",
    "actnn-relu_bwd",
    "actnn-unpack",
    "actnn-unpack-packed-2^32",
    "comp_aggr-gather-F300",
    "comp_aggr-store-F300",
    "dcoef-F252",
    "disen_route_fwd-store-K3d32",
    "edge_colsum-edge",
    "edge_softmax_bwd",
    "edge_softmax_fwd",
    "gat_attn_bwd-edge",
    "gat_attn_bwd_dropout-edge",
    "gat_fwd",
    "gat_fwd_dropout",
    "gather_rows",
    "gcn_fused-gather-K128",
    "gcn_fused-store-K128",
    "genconv_edge_bwd-tstore-F300",
    "genconv_edge_fwd-edge-D8",
    "genconv_edge_fwd-gather-F300",
    "hgn_attn-edge",
    "hgn_attn_bwd-edge",
    "label_prop-F124",
    "mhsddmm-edge",
    "mhsddmm-gather-H4F75",
    "mhspmm-gather-H4F75",
    "mhspmm-perm-edge",
    "mhspmm-store-H4F75",
    "mhspmm_dropout-perm-edge",
    "residual-F124",
    "residual-F300-none",
    "rgcn_aggr-gather-F300",
    "rgcn_aggr-partials-B8F128",
    "rgcn_aggr-per_basis-B2F150",
    "rgcn_aggr-store-B2F150",
    "rgcn_edge_dot-edge-B8",
    "rgcn_edge_dot-gather-F300",
    "sage_fused-gather-K128",
    "sage_fused-store-K128",
    "scatter_max-gather-F300",
    "scatter_max-store-F300",
    "scatter_max_bwd-gather-F300",
    "sddmm-gather-F300",
    "softmax_aggr_bwd-tstore-F300",
    "softmax_aggr_fwd-edge-F8",
    "softmax_aggr_fwd-gather-F300",
    "spmm-gather-lean-F124",
    "spmm-gather-panels3-F192",
    "spmm-gather-row-chunks-F37",
    "spmm-gather-row-none-F300",
    "spmm-gather-stream-nv2-F252",
    "spmm-partials-F3703",
    "spmm-store-lean-F124",
    "spmm-store-panels3-F192",
    "spmm-store-row-chunks-F300",
    "spmm-store-row-chunks-F37",
    "spmm-store-row-none-F300",
    "spmm-store-stream-nv2-F252",
    "spmm_2src-gather-F124",
    "spmm_2src-store-F124",
    "spmm_f16-gather-F300",
    "spmm_f16-store-F300",
    "spmm_peers-gather-F124",
    "spmm_peers-store-F124",
    "spmm_plain-gather-F124",
    "spmm_plain-store-F124",
}


def test_no_row_is_dropped():
    ids = [c.id for c in LT.TABLE]
    assert len(ids) == len(set(ids)), "duplicate row ids"
    missing = ROW_IDS - set(ids)
    assert not missing, f"rows removed from the table: {sorted(missing)}"
    assert set(ids) == ROW_IDS, f"new rows, add them to ROW_IDS: {sorted(set(ids) - ROW_IDS)}"


@pytest.mark.parametrize("c", LT.TABLE, ids=lambda c: c.id)
def test_row_shape(c):
    assert c.crossing_elems > LT.B31, f"{c.id}: the {c.operand} operand has {c.crossing_elems} elements"
    if c.wrap:
        assert c.crossing_elems > LT.B32, f"{c.id}: marked for the unsigned wrap, {c.crossing_elems} elements"
    S = c.samples
    assert c.straddle in S, f"{c.id}: S misses the straddling index {c.straddle}"
    assert c.straddle * c.width <= LT.B31 < (c.straddle + 1) * c.width
    assert c.bytes_needed <= LT.MAX_BYTES, f"{c.id}: {c.bytes_needed} bytes"
    assert c.kernel, f"{c.id}: no kernel string"
    if c.role in ("gather", "tstore", "store", "epilogue", "elements") and c.entry not in LT.FIXED_WIDTH:
        assert LT.B31 % c.width != 0, f"{c.id}: the width divides 2^31, so no row straddles the boundary"


def test_wrap_rows():
    wrap = {(c.entry, c.dtype) for c in LT.TABLE if c.wrap}
    assert ("cogdl_b200_spmm_csr_f16", "f16") in wrap
    assert ("cogdl_b200_actnn_unpack_f32", "u8") in wrap
    assert any(c.wrap and c.entry == "cogdl_b200_spmm_csr_f32_ex" and "stream_kernel" in c.kernel for c in LT.TABLE)


def test_every_spmm_form_has_a_gather_and_a_store_row():
    spmm = [c for c in LT.TABLE if c.entry == "cogdl_b200_spmm_csr_f32_ex"]
    forms = {
        "row/none": lambda c: "spmm_kernel<" in c.kernel and c.plan == "none",
        "row/chunks": lambda c: "spmm_kernel<" in c.kernel and c.plan == "chunks",
        "lean stream": lambda c: "stream_kernel<float4,NV=1," in c.kernel and "prefetch" not in c.kernel,
        "general stream": lambda c: "stream_kernel<" in c.kernel and "NV=1," not in c.kernel,
        "panels": lambda c: ",panels=" in c.kernel,
    }
    for form, is_form in forms.items():
        for role in ("gather", "store"):
            assert any(is_form(c) and c.role == role for c in spmm), f"no {role} row for the SpMM {form} form"
    for role in ("gather", "store"):
        assert any(c.entry == "cogdl_b200_spmm_csr_f16" and c.role == role for c in LT.TABLE)
    assert any(c.role == "partials" for c in LT.TABLE)


def test_largest_row():
    assert LT.LARGEST.bytes_needed == max(c.bytes_needed for c in LT.TABLE)

"""One row per non-finite case: an entry point of include/cogdl_b200.h run with NaN, +-Inf or overflowing values in one
operand role, on a graph whose hub plan cuts rows into chunks at every chunk size the plan forms use.

Each row names the entry point, the operand that carries the values, the graph (tests/graphs.boundary_csr at the plan's
chunk, or a graphs.CASES name) and F (with an F % 4 tail where the entry takes any F).  Where the values go, per family:
  features / logits  the first, a middle and the last chunk of the largest hub row, a one-edge row, the first and the
                     last column, a whole (row, head) of NaN logits, a +Inf logit
  edge weights       NaN and Inf weights on hub and short rows, and an edge of weight exactly 0 pointing at an Inf
                     feature (0 * Inf is NaN: no path may skip a zero weight)
  overflow           finite operands whose row sums pass the type's largest finite value (fp16 past 65504; the fused
                     layers' aggregated rows past the bf16 overflow threshold 0x1.fefp127), or whose fp32 softmax logits
                     are +-Inf (GENConv's beta m, DisenGCN's q . c / tau) on the first edge of a hub chunk, of a short
                     row and of a one-edge row
  grad_out / saved   a backward's incoming gradient, or the forward tensor it saved (softmax y, signed attention),
                     at the same sites, with a zero attention against an Inf gradient and NaN / Inf on dropped entries
  b_dev              a device scalar coefficient (GIN's learnable epsilon) that has diverged
tests/test_gpu_nonfinite.py runs every row under the plan forms PLAN_FORMS (the fused layers, which need the row-stream
form, under the default plans only; the SpMM rows also under forced panel counts)
against the fp64 composition of the same formula: the NaN mask and the +-Inf positions and signs must match exactly,
finite elements stay within the family's bound.  tests/test_cpu_nonfinite_inventory.py checks, without a GPU, that every
entry point of the header that takes a float operand has a row or an entry in EXEMPT or NOT_COVERED with its reason.
Plain Python, no torch.
"""
from dataclasses import dataclass

# (name, chunk edges, seg_cost): plan none, chunks only, the default plan at chunk 16 and at chunk 64
PLAN_FORMS = (("none", 0, None), ("chunks16", 16, 0), ("default16", 16, None), ("default64", 64, None))
SPMM_PANELS = (1, 3, 6)       # forced column panel counts of the fp32 SpMM features row on the default plans, at F = 192
PANEL_F = 192                 # (one pass, then panels of 64 and 32 floats: bitwise equal whatever the count)


@dataclass(frozen=True)
class NCase:
    name: str
    entry: str              # the C entry point (cogdl_b200_*)
    operand: str            # features | edge weights | logits | attention | Z | grad_out | saved | b_dev | overflow
    graph: str              # "bounds" (boundary_csr at the plan's chunk) or a graphs.CASES name
    F: int                  # features (per head)
    H: int = 1
    K: int = 1              # DisenGCN channels (F = K * d, d a power of two)

    @property
    def id(self):
        return self.name


TABLE = [
    NCase("spmm-features-F67", "cogdl_b200_spmm_csr_f32_ex", "features", "bounds", 67),
    NCase("spmm-weights-F67", "cogdl_b200_spmm_csr_f32_ex", "edge weights", "bounds", 67),
    NCase("spmm_f16-overflow-F66", "cogdl_b200_spmm_csr_f16", "overflow", "bounds", 66),
    NCase("residual-Z-F67", "cogdl_b200_spmm_residual_f32", "Z", "bounds", 67),
    NCase("sddmm-features-F67", "cogdl_b200_sddmm_csr_f32", "features", "bounds", 67),
    NCase("mhspmm-attention-H4F11", "cogdl_b200_mhspmm_f32", "attention", "bounds", 11, H=4),
    NCase("scatter_max-features-F67", "cogdl_b200_scatter_max_fwd_f32", "features", "bounds", 67),
    NCase("edge_softmax-logits-H4", "cogdl_b200_edge_softmax_fwd_f32", "logits", "bounds", 1, H=4),
    NCase("edge_softmax-logits-H1", "cogdl_b200_edge_softmax_fwd_f32", "logits", "bounds", 1, H=1),
    NCase("softmax_aggr_fwd-features-F67", "cogdl_b200_softmax_aggr_fwd_f32", "features", "bounds", 67),
    NCase("softmax_aggr_fwd-edge_term-F67", "cogdl_b200_softmax_aggr_fwd_f32", "edge term", "bounds", 67),
    NCase("softmax_aggr_fwd-overflow-F67", "cogdl_b200_softmax_aggr_fwd_f32", "overflow", "bounds", 67),
    NCase("softmax_aggr_bwd-grad_out-F67", "cogdl_b200_softmax_aggr_bwd_f32", "grad_out", "bounds", 67),
    NCase("softmax_aggr_bwd-overflow-F67", "cogdl_b200_softmax_aggr_bwd_f32", "overflow", "bounds", 67),
    NCase("genconv_edge_fwd-features-F67", "cogdl_b200_genconv_edge_fwd_f32", "features", "bounds", 67),
    NCase("gcn_fused-features-K128", "cogdl_b200_gcn_fused_f32", "features", "bounds", 128),
    NCase("gcn_fused-overflow-K128", "cogdl_b200_gcn_fused_f32", "overflow", "bounds", 128),
    NCase("sage_fused-sum-features-K128", "cogdl_b200_sage_fused_f32", "features", "bounds", 128),
    NCase("sage_fused-mean-features-K128", "cogdl_b200_sage_fused_f32", "features", "bounds", 128),
    NCase("sage_fused-max-features-K128", "cogdl_b200_sage_fused_f32", "features", "bounds", 128),
    NCase("residual_dcoef-b_dev-F67", "cogdl_b200_spmm_residual_dcoef_f32", "b_dev", "bounds", 67),
    NCase("mhspmm_dropout-attention-H4F11", "cogdl_b200_mhspmm_dropout_f32", "attention", "bounds", 11, H=4),
    NCase("scatter_max_bwd-grad_out-F67", "cogdl_b200_scatter_max_bwd_f32", "grad_out", "bounds", 67),
    NCase("edge_softmax_bwd-grad_out-H4", "cogdl_b200_edge_softmax_bwd_f32", "grad_out", "bounds", 1, H=4),
    NCase("edge_softmax_bwd-saved-H4", "cogdl_b200_edge_softmax_bwd_f32", "saved", "bounds", 1, H=4),
    NCase("gat_attn_bwd-grad_out-H4", "cogdl_b200_gat_attn_bwd_f32", "grad_out", "bounds", 1, H=4),
    NCase("gat_attn_bwd-saved-H4", "cogdl_b200_gat_attn_bwd_f32", "saved", "bounds", 1, H=4),
    NCase("gat_attn_bwd_dropout-grad_out-H4", "cogdl_b200_gat_attn_bwd_dropout_f32", "grad_out", "bounds", 1, H=4),
    NCase("gat_attn_bwd_dropout-saved-H4", "cogdl_b200_gat_attn_bwd_dropout_f32", "saved", "bounds", 1, H=4),
    NCase("hgn_attn-logits-H4", "cogdl_b200_hgn_attn_f32", "logits", "bounds", 1, H=4),
    NCase("hgn_attn_bwd-grad_out-H4", "cogdl_b200_hgn_attn_bwd_f32", "grad_out", "bounds", 1, H=4),
    NCase("hgn_attn_bwd-saved-H4", "cogdl_b200_hgn_attn_bwd_f32", "saved", "bounds", 1, H=4),
    NCase("disen_route_fwd-overflow-K3F6", "cogdl_b200_disen_route_fwd_f32", "overflow", "bounds", 6, K=3),
]

# Entry points whose operands no non-finite value can reach: integer only, or the value reaches only an index.
EXEMPT = {
    "cogdl_b200_spgemm_count": "sparse x sparse structure: integer indices only",
    "cogdl_b200_csr2csc": "integer only",
    "cogdl_b200_coo2csr_index": "integer only",
    "cogdl_b200_narrow_i64_i32": "integer only",
    "cogdl_b200_sample_adj_count": "sampler: integer indices only",
    "cogdl_b200_sample_adj_fill": "sampler: integer indices only",
    "cogdl_b200_subgraph_count": "sampler: integer indices only",
    "cogdl_b200_subgraph_fill": "sampler: integer indices only",
    "cogdl_b200_hub_plan_count": "integer only, reads rowptr",
    "cogdl_b200_hub_plan_fill": "integer only, reads rowptr",
    "cogdl_b200_edge_rows": "integer only",
    "cogdl_b200_actnn_bits": "returns EINVAL for a non-finite C before any kernel runs (DESIGN.md, actnn)",
}

# Entry points that take a float operand and are outside this table's scope: no non-finite row yet (follow-up work).
# Each is checked per element against fp64 on finite inputs by the suite its reason names; the inventory test lists
# them apart from EXEMPT so that they are not mistaken for coverage.  An entry that gains a row must leave NOT_COVERED.
NOT_COVERED = {
    "cogdl_b200_spmm_csr_f32": "finite rows in tests/dispatch_table.py; the same stream kernels as spmm-features-F67",
    "cogdl_b200_spmm_csr_f32_2src": "finite rows in tests/dispatch_table.py",
    "cogdl_b200_spmm_csr_f32_peers": "finite rows in tests/dispatch_table.py",
    "cogdl_b200_spmm_accum_f32": "finite rows in tests/gin_grand_table.py",
    "cogdl_b200_label_prop_f32": "finite rows in tests/label_prop_table.py; the clamp's NaN rule is pinned in tests/test_gpu_label_prop.py",
    "cogdl_b200_mhsddmm_f32": "finite rows in tests/dispatch_table.py",
    "cogdl_b200_gat_fwd_f32": "finite and -inf rows in tests/dispatch_table.py",
    "cogdl_b200_gat_fwd_dropout_f32": "finite rows in tests/dispatch_table.py",
    "cogdl_b200_edge_colsum_f32": "finite rows in tests/dispatch_table.py",
    "cogdl_b200_gather_rows_f32": "a copy: moves bits, no arithmetic",
    "cogdl_b200_genconv_edge_bwd_f32": "finite rows in tests/genconv_edge_table.py",
    "cogdl_b200_disen_route_bwd_f32": "finite rows in tests/dispatch_table.py",
    "cogdl_b200_comp_aggr_f32": "finite rows in tests/dispatch_table.py",
    "cogdl_b200_rgcn_aggr_f32": "finite rows in tests/rgcn_table.py",
    "cogdl_b200_rgcn_edge_dot_f32": "finite rows in tests/rgcn_table.py",
    "cogdl_b200_spgemm_fill_f32": "finite rows in tests/graphs.SPGEMM_CASES",
    "cogdl_b200_spgemm_bwd_f32": "finite rows in tests/graphs.SPGEMM_CASES",
    "cogdl_b200_actnn_minmax_f32": "a NaN is left out of the group range (DESIGN.md, actnn); finite rows in "
                                   "tests/test_gpu_actnn.py",
    "cogdl_b200_actnn_pack_f32": "a NaN packs to a finite code (DESIGN.md, actnn); finite rows in tests/test_gpu_actnn.py",
    "cogdl_b200_actnn_unpack_f32": "finite rows in tests/test_gpu_actnn.py",
    "cogdl_b200_actnn_relu_fwd_f32": "finite rows in tests/test_gpu_actnn.py",
    "cogdl_b200_actnn_relu_bwd_f32": "finite rows in tests/test_gpu_actnn.py",
    "cogdl_b200_actnn_dropout_fwd_f32": "finite rows in tests/test_gpu_actnn.py",
    "cogdl_b200_actnn_dropout_bwd_f32": "finite rows in tests/test_gpu_actnn.py",
}

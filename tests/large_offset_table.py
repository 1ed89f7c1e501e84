"""One row per large-offset case: an entry point of include/cogdl_b200.h run with one dense operand of more than 2^31
elements, so that every index into it past element 2^31 needs 64-bit arithmetic (DESIGN.md section 2).

Each row names the entry point, the operand that crosses the boundary and its role, the shape, the plan form and the
exact cogdl_b200_last_kernel() string, and derives from the shape the bytes the case allocates.  The shapes are thin:
only the operand under test is large.
  gather   an input read through colind (or through perm): a few hundred rows whose edges point at the columns of a
           band at the top of X, at the column whose row straddles element 2^31, at columns 0 and 1 and, for the 2^32
           rows, at the columns an unsigned 32-bit wrap aliases onto
  store    a row-indexed output: n_rows just past 2^31 / F, every row empty except a band at the top (unsplit rows,
           hub rows, empty rows) and the straddling row, so the row store, the hub-merge store and the empty-row fill
           all write past 2^31
  epilogue a row-indexed operand of an SpMM epilogue (Z, row_scale, ACC, ACC_in, Xn) on the store graph
  edge     an [nnz, H] tensor with nnz * H past 2^31 (H = 8, nnz just past 2^28 on ~4000 rows)
  tstore   the output of a backward that runs over the transpose of a gather graph (dX [n_cols, F]), with X beside it
  partials the hub plan's per-chunk scratch with n_chunks * F past 2^31
  elements an element-wise [N, D] operand (activation compression) with N * D past 2^31
  packed   the 8-bit packed input of the actnn unpack: D = 1 padded to 256 bytes a row, so the packed bytes pass 2^32
           while the fp32 output stays small
An offset in [2^31, 2^32) that is computed in unsigned 32-bit arithmetic still comes out right, so the rows marked
`wrap` go past 2^32 elements.

tests/test_gpu_large_offsets.py runs every row; tests/test_cpu_large_offset_inventory.py checks, without a GPU, that
every entry point of the header that takes a dense float operand has a row or an exemption with its reason, and that
every row's shape does what its role says.  Plain Python, no torch.
"""
from dataclasses import dataclass

from tests.dispatch_table import half_k, spmm_k, stream_k
from tests.gin_grand_table import epi_name
from tests.label_prop_table import labelprop_name
from tests.spmm_residual_table import residual_name

B31 = 2 ** 31
B32 = 2 ** 32
GIB = 2 ** 30
MAX_BYTES = 20 * GIB          # no case allocates more (LARGEST below)
CHUNK = 64                    # hub chunk edges of every plan here
SLOPE = 0.2

# gather graphs: GATHER_ROWS rows with degrees cycling through DEGREES (0: empty, > CHUNK: hub rows)
GATHER_ROWS = 512
DEGREES = (0, 1, 2, 3, 5, 8, 31, 32, 33, 64, 65, 130, 200)
BAND = 64                     # columns (gather) or rows (store) past the boundary at the top of the operand
LOW = (0, 1, 2, 3)            # low indices every sample holds

# edge graph: EDGE_FULL rows of EDGE_DEG edges (the first EDGE_SHIFT short, so that no row boundary falls on edge
# 2^28), then the tail rows, whose edges all lie past nnz * H = 2^31 for H = 8
EDGE_H = 8
EDGE_FULL = 4096
EDGE_DEG = 65536
EDGE_SHIFT = 5
EDGE_TAIL = (40, 0, 1, 2, 3, 5, 8, 31, 32, 33, 64, 65, 100, 129, 1000, 3000, 70000)
EDGE_F = 4                    # feature width of the [n, H, F] operands of the edge cases (kept small)

# partials graph: PART_ROWS hub rows of LCase.part_deg edges each (F = PART_F for the SpMM)
PART_F = 3703
PART_ROWS = 8


def ceil_div(a, b):
    return -(-a // b)


def edge_degrees():
    return [EDGE_DEG - EDGE_SHIFT] + [EDGE_DEG] * (EDGE_FULL - 1) + list(EDGE_TAIL)


@dataclass(frozen=True)
class LCase:
    name: str
    entry: str              # the C entry point (cogdl_b200_*)
    operand: str            # the operand that crosses 2^31 elements
    role: str               # gather | store | epilogue | edge | partials | elements
    dtype: str              # f32 | f16 (the crossing operand's element type; u8 for a packed actnn input)
    F: int                  # features (per head); the row width D for `elements`
    kernel: str             # exact cogdl_b200_last_kernel() after the call
    H: int = 1
    plan: str = "default"   # none | chunks | default, as in dispatch_table.Case
    panels: int = 0         # column panels passed to the SpMM (0: the library's choice)
    wrap: bool = False      # the crossing operand has more than 2^32 elements (catches unsigned 32-bit wraps)
    weighted: bool = True
    n_big: int = 1          # tensors of the crossing operand's size held at once (inputs aliased where the entry allows)
    nnz_arrays: int = 0     # [nnz] int32 / fp32 arrays beyond colind and edge_row (etype, w) of the edge and partials rows
    transpose: bool = False  # the call runs over the cached transpose (rowptr, rowind, perm built by csr2csc)

    @property
    def id(self):
        return self.name

    @property
    def esize(self):
        return {"f32": 4, "f16": 2, "u8": 1}[self.dtype]

    @property
    def width(self):
        """Elements per index of the crossing operand (a row of X or Y, an edge's heads, a chunk's partial)."""
        if self.role == "packed":
            return self.packed_row
        if self.role in ("gather", "tstore", "store", "epilogue", "partials"):
            return self.F * self.H
        return self.H if self.role == "edge" else self.F

    @property
    def limit(self):
        return B32 if self.wrap else B31

    # ---- shapes
    @property
    def n_cols(self):
        if self.role in ("gather", "tstore"):
            return ceil_div(self.limit, self.width) + BAND
        if self.role == "edge":
            return len(edge_degrees())
        return 256

    @property
    def n_rows(self):
        if self.role in ("store", "epilogue"):
            return ceil_div(self.limit, self.width) + BAND
        if self.role in ("gather", "tstore"):
            return GATHER_ROWS
        if self.role == "edge":
            return len(edge_degrees())
        if self.role == "partials":
            return PART_ROWS
        if self.role == "packed":
            return ceil_div(self.limit, self.packed_row) + BAND
        return ceil_div(self.limit, self.F) + BAND      # elements: N rows of D

    @property
    def nnz(self):
        if self.role == "edge":
            return sum(edge_degrees())
        if self.role == "partials":
            return PART_ROWS * self.part_deg
        if self.role in ("elements", "packed"):
            return 0
        return sum(DEGREES[i % len(DEGREES)] for i in range(self.n_rows if self.role in ("gather", "tstore")
                                                           else BAND + 1))

    @property
    def part_deg(self):
        """Edges of each hub row of a partials row: enough chunks that n_chunks * width passes 2^31."""
        return ceil_div(B31 // self.width + 1, PART_ROWS) * CHUNK

    @property
    def n_chunks(self):
        return PART_ROWS * self.part_deg // CHUNK if self.role == "partials" else 0

    @property
    def packed_row(self):
        """Bytes of one packed row at 8 bits: the row width D zero-padded to a multiple of the group size (256)."""
        return ceil_div(self.F, 256) * 256

    @property
    def crossing_elems(self):
        if self.role == "packed":
            return self.n_rows * self.packed_row
        n = {"gather": self.n_cols, "tstore": self.n_cols, "store": self.n_rows, "epilogue": self.n_rows,
             "edge": self.nnz, "partials": self.n_chunks, "elements": self.n_rows}[self.role]
        return n * self.width

    @property
    def straddle(self):
        """Index (column, row, edge, chunk slot) whose run of `width` elements holds element 2^31."""
        return B31 // (self.packed_row if self.role == "packed" else self.width)

    @property
    def samples(self):
        """The sampled indices S along the crossing dimension: the band past the boundary, the straddling index, the
        indices a 32-bit wrap aliases onto and a few low ones."""
        n = self.crossing_elems // self.width
        s = set(range(n - BAND, n)) | {self.straddle} | set(LOW)
        if self.role == "edge":
            s |= set(range(self.straddle, n))     # every edge past the boundary: the whole tail
        if self.wrap:
            s.add(B32 // self.width)
        for i in list(s):
            if i * self.width >= B32:
                s.add((i * self.width - B32) // self.width)
        if self.role in ("edge", "partials"):
            return sorted(s)
        return sorted(i for i in s if i < n)

    @property
    def big_tensors(self):
        """(name, bytes) of every tensor of more than 64 MiB the case holds at once."""
        cross = self.crossing_elems * self.esize
        t = [(self.operand, cross)] + [("operand of the same size", cross)] * (self.n_big - 1)
        if self.role in ("store", "epilogue"):
            t.append(("rowptr", 4 * self.n_rows))
        if self.role == "tstore":
            t += [("rowptr of the transpose", 4 * self.n_cols), ("X", self.n_cols * self.width * 4)]
        if self.role in ("edge", "partials") and self.entry != "cogdl_b200_gather_rows_f32":
            t += [("colind", 4 * self.nnz), ("edge_row", 4 * self.nnz)] + [("[nnz] array", 4 * self.nnz)] * \
                self.nnz_arrays
        if self.entry == "cogdl_b200_gather_rows_f32":
            t.append(("perm", 4 * self.nnz))
        if self.transpose and self.role == "edge":
            t += [("rowind, perm", 8 * self.nnz), ("csr2csc workspace", 12 * self.nnz)]
        if self.entry == "cogdl_b200_scatter_max_fwd_f32" and self.role == "store":
            t.append(("argmax", cross))
        if self.role == "elements" and ("relu" in self.entry or "dropout" in self.entry):
            t.append(("mask", self.crossing_elems // 8))
        if self.role == "packed":
            t.append(("x", self.n_rows * self.F * 4))
        return [(k, b) for k, b in t if b > 64 * 2 ** 20]

    @property
    def bytes_needed(self):
        return sum(b for _, b in self.big_tensors)


# cogdl_b200_gather_rows_f32 and cogdl_b200_edge_colsum_f32 record no kernel string
NO_KERNEL = "(no kernel string recorded)"
ES = "cogdl_b200::es_stats_kernel<MODE={m}> + cogdl_b200::es_main_kernel<MODE={m},CAP=512,WARPS=8{d}>"


def _w(w):
    return "weighted" if w else "unweighted"


LEAN = stream_k("float4", 1, "weighted", "SRC_ONE", 4, 5, False)           # F = 124: 31 float4, one per lane
NV2 = stream_k("float4", 2, "weighted", "SRC_ONE", 4, 1, True)             # F = 252: 63 float4, two per lane
PANEL3 = stream_k("float2", 1, "weighted", "SRC_ONE", 8, 5, True, 3)       # F = 192 in three 64-float panels
ROW300 = spmm_k("float4", 32, 2, True)                                     # F = 300: row kernel, two column tiles
ROW37 = spmm_k("float", 32, 2, True)                                       # F = 37: scalar row kernel
LEAN2 = stream_k("float4", 1, "weighted", "SRC_TWO", 4, 5, False)          # the two-source form at F = 124
LEANP = stream_k("float4", 1, "weighted", "SRC_PEERS", 4, 5, False)        # the peer form at F = 124
MH_STREAM = "cogdl_b200::stream_kernel<float,NV=1,multihead,SRC_ONE,U=8,MINB=3,prefetch> block=128"   # H*F = 300
COMP_NV2 = "cogdl_b200::stream_kernel<float4,NV=2,comp_mult,SRC_ONE,U=2,MINB=1,prefetch> block=128"
ES3_DROP = ("cogdl_b200::es_stats_kernel<MODE=3,DROP> + cogdl_b200::es_main_kernel<MODE=3,CAP=512,WARPS=8,DROP> "
            "cp.async.bulk tiles")
# the hub rows' SpMM, then the fused tile kernel (tile width = Fout rounded up: 64 for Fout = 16 .. 64, 128 above)
FUSED = "cogdl_b200::fg::fused_layer_kernel<{}, 2 groups x tile 64x{}, K=128, bf16x3 split, wgmma m64n32k16>"
FIXED_WIDTH = ("cogdl_b200_gcn_fused_f32", "cogdl_b200_sage_fused_f32")     # K = 128 is the only width they take


def _spmm(side):
    C = lambda name, F, kernel, **kw: LCase(f"spmm-{side}-{name}", "cogdl_b200_spmm_csr_f32_ex",  # noqa: E731
                                            "X" if side == "gather" else "Y", side, "f32", F, kernel, **kw)
    rows = [
        C("row-none-F300", 300, ROW300, plan="none", panels=1),
        C("row-chunks-F37", 37, ROW37, plan="chunks", panels=1),
        C("lean-F124", 124, LEAN, panels=1, wrap=side == "gather"),
        C("stream-nv2-F252", 252, NV2, panels=1),
        C("panels3-F192", 192, PANEL3, panels=3),
    ]
    if side == "store":
        rows.append(C("row-chunks-F300", 300, ROW300, plan="chunks", panels=1))
    return rows


TABLE = _spmm("gather") + _spmm("store") + [
    LCase("spmm-partials-F3703", "cogdl_b200_spmm_csr_f32_ex", "partials", "partials", "f32", PART_F,
          spmm_k("float", 32, 4, False), plan="chunks", panels=1, weighted=False),
    LCase("spmm_f16-gather-F300", "cogdl_b200_spmm_csr_f16", "X", "gather", "f16", 300, half_k(True, True), wrap=True),
    LCase("spmm_f16-store-F300", "cogdl_b200_spmm_csr_f16", "Y", "store", "f16", 300, half_k(True, True)),
    LCase("residual-F124", "cogdl_b200_spmm_residual_f32", "Z", "epilogue", "f32", 124, residual_name(LEAN), panels=1,
          n_big=2),
    LCase("residual-F300-none", "cogdl_b200_spmm_residual_f32", "Z", "epilogue", "f32", 300, residual_name(ROW300),
          plan="none", panels=1, n_big=2),
    LCase("label_prop-F124", "cogdl_b200_label_prop_f32", "Z", "epilogue", "f32", 124,
          labelprop_name(residual_name(LEAN)), panels=1, n_big=2),
    LCase("dcoef-F252", "cogdl_b200_spmm_residual_dcoef_f32", "Z", "epilogue", "f32", 252,
          epi_name(residual_name(NV2), "dcoef"), panels=1, n_big=2),
    LCase("accum-F124", "cogdl_b200_spmm_accum_f32", "ACC", "epilogue", "f32", 124,
          epi_name(residual_name(LEAN), "accum"), panels=1, n_big=2),
    LCase("accum-last-F300-chunks", "cogdl_b200_spmm_accum_f32", "ACC_in", "epilogue", "f32", 300,
          epi_name(residual_name(ROW300), "accum"), plan="chunks", panels=1, n_big=2),
    LCase("sddmm-gather-F300", "cogdl_b200_sddmm_csr_f32", "D2", "gather", "f32", 300,
          "cogdl_b200::sddmm_kernel<float4,GROUP=32,SUB=32,NV=4>"),
    LCase("scatter_max-gather-F300", "cogdl_b200_scatter_max_fwd_f32", "X", "gather", "f32", 300,
          "cogdl_b200::scatter_max_fwd_kernel<float4,GROUP=32,NV=2>", plan="chunks"),
    LCase("scatter_max-store-F300", "cogdl_b200_scatter_max_fwd_f32", "out", "store", "f32", 300,
          "cogdl_b200::scatter_max_fwd_kernel<float4,GROUP=32,NV=2>", plan="chunks"),
    LCase("scatter_max_bwd-gather-F300", "cogdl_b200_scatter_max_bwd_f32", "gx", "gather", "f32", 300,
          "cogdl_b200::scatter_max_bwd_kernel", plan="chunks"),
    # edge-aligned [nnz, H] tensors
    LCase("edge_softmax_fwd", "cogdl_b200_edge_softmax_fwd_f32", "in/out", "edge", "f32", 1,
          ES.format(m=0, d="") + " cp.async.bulk tiles", H=EDGE_H, n_big=2),
    LCase("edge_softmax_bwd", "cogdl_b200_edge_softmax_bwd_f32", "y/g/gin", "edge", "f32", 1,
          ES.format(m=1, d="") + " cp.async.bulk tiles", H=EDGE_H, n_big=2),
    LCase("gat_fwd", "cogdl_b200_gat_fwd_f32", "att_out", "edge", "f32", EDGE_F,
          ES.format(m=2, d="") + " + cogdl_b200::mhspmm_kernel<float4,GROUP=8,no_perm>", H=EDGE_H),
    LCase("gat_fwd_dropout", "cogdl_b200_gat_fwd_dropout_f32", "att_out", "edge", "f32", EDGE_F,
          ES.format(m=2, d=",DROP") + " + cogdl_b200::mhspmm_kernel<float4,GROUP=8,no_perm,drop>", H=EDGE_H),
    LCase("gather_rows", "cogdl_b200_gather_rows_f32", "in/out", "edge", "f32", 1, NO_KERNEL, H=EDGE_H, n_big=2),
    LCase("spmm_plain-gather-F124", "cogdl_b200_spmm_csr_f32", "X", "gather", "f32", 124, LEAN),
    LCase("spmm_plain-store-F124", "cogdl_b200_spmm_csr_f32", "Y", "store", "f32", 124, LEAN),
    LCase("spmm_2src-gather-F124", "cogdl_b200_spmm_csr_f32_2src", "X1", "gather", "f32", 124, LEAN2),
    LCase("spmm_2src-store-F124", "cogdl_b200_spmm_csr_f32_2src", "Y", "store", "f32", 124, LEAN2),
    LCase("spmm_peers-gather-F124", "cogdl_b200_spmm_csr_f32_peers", "peer shard", "gather", "f32", 124, LEANP),
    LCase("spmm_peers-store-F124", "cogdl_b200_spmm_csr_f32_peers", "Y", "store", "f32", 124, LEANP),
    LCase("mhspmm-gather-H4F75", "cogdl_b200_mhspmm_f32", "feat", "gather", "f32", 75, MH_STREAM, H=4),
    LCase("mhspmm-store-H4F75", "cogdl_b200_mhspmm_f32", "out", "store", "f32", 75, MH_STREAM, H=4),
    LCase("mhspmm-perm-edge", "cogdl_b200_mhspmm_f32", "att", "edge", "f32", EDGE_F, "cogdl_b200::mhspmm_kernel<float4,GROUP=8,perm>", H=EDGE_H, transpose=True),
    LCase("mhspmm_dropout-perm-edge", "cogdl_b200_mhspmm_dropout_f32", "att", "edge", "f32", EDGE_F, "cogdl_b200::mhspmm_kernel<float4,GROUP=8,perm,drop>", H=EDGE_H,
          transpose=True),
    LCase("mhsddmm-gather-H4F75", "cogdl_b200_mhsddmm_f32", "feat", "gather", "f32", 75, "cogdl_b200::sddmm_kernel<float,GROUP=32,SUB=32,NV=4>", H=4),
    LCase("mhsddmm-edge", "cogdl_b200_mhsddmm_f32", "out", "edge", "f32", EDGE_F, "cogdl_b200::sddmm_kernel<float4,GROUP=8,SUB=1,NV=1>", H=EDGE_H),
    LCase("gat_attn_bwd-edge", "cogdl_b200_gat_attn_bwd_f32", "att/d_att/d_edge", "edge", "f32", 1, ES.format(m=3, d="") + " cp.async.bulk tiles", H=EDGE_H,
          n_big=2),
    LCase("gat_attn_bwd_dropout-edge", "cogdl_b200_gat_attn_bwd_dropout_f32", "att/d_att/d_edge", "edge", "f32", 1,
          ES3_DROP, H=EDGE_H, n_big=2),
    LCase("edge_colsum-edge", "cogdl_b200_edge_colsum_f32", "e", "edge", "f32", 1, NO_KERNEL, H=EDGE_H, transpose=True),
    LCase("softmax_aggr_fwd-gather-F300", "cogdl_b200_softmax_aggr_fwd_f32", "X", "gather", "f32", 300, "cogdl_b200::softmax_aggr_fwd_kernel<float4,no_edge_term,Q>"),
    LCase("softmax_aggr_fwd-edge-F8", "cogdl_b200_softmax_aggr_fwd_f32", "edge_term", "edge", "f32", 1, "cogdl_b200::softmax_aggr_fwd_kernel<float4,edge_term,no_Q>", H=8),
    LCase("softmax_aggr_bwd-tstore-F300", "cogdl_b200_softmax_aggr_bwd_f32", "dX", "tstore", "f32", 300, "cogdl_b200::softmax_aggr_bwd_kernel<float4,no_edge_term>"),
    LCase("genconv_edge_fwd-gather-F300", "cogdl_b200_genconv_edge_fwd_f32", "X", "gather", "f32", 300, "cogdl_b200::genconv_edge_fwd_kernel<float4,DM=8,Q>"),
    LCase("genconv_edge_fwd-edge-D8", "cogdl_b200_genconv_edge_fwd_f32", "attr", "edge", "f32", 1, "cogdl_b200::genconv_edge_fwd_kernel<float4,DM=8,no_Q>", H=8),
    LCase("genconv_edge_bwd-tstore-F300", "cogdl_b200_genconv_edge_bwd_f32", "dX", "tstore", "f32", 300, "cogdl_b200::genconv_edge_bwd_kernel<float4,DM=8>"),
    LCase("disen_route_fwd-store-K3d32", "cogdl_b200_disen_route_fwd_f32", "q=c/out", "store", "f32", 96, "cogdl_b200::disen_route_fwd_kernel<float4,GROUP=32>", n_big=2),
    LCase("comp_aggr-gather-F300", "cogdl_b200_comp_aggr_f32", "A", "gather", "f32", 300, COMP_NV2),
    LCase("comp_aggr-store-F300", "cogdl_b200_comp_aggr_f32", "Y", "store", "f32", 300, COMP_NV2),
    LCase("rgcn_aggr-gather-F300", "cogdl_b200_rgcn_aggr_f32", "X", "gather", "f32", 300, "cogdl_b200::rgcn_fanout_kernel<float4> block=128"),
    LCase("rgcn_aggr-per_basis-B2F150", "cogdl_b200_rgcn_aggr_f32", "X [*, B, F]", "gather", "f32", 150, "cogdl_b200::rgcn_fanout_kernel<float,per_basis> block=128", H=2),
    LCase("rgcn_aggr-store-B2F150", "cogdl_b200_rgcn_aggr_f32", "Y [n, B, F]", "store", "f32", 150, "cogdl_b200::rgcn_fanout_kernel<float> block=128", H=2),
    LCase("rgcn_aggr-partials-B8F128", "cogdl_b200_rgcn_aggr_f32", "partials", "partials", "f32", 128, "cogdl_b200::rgcn_fanout_kernel<float4> block=128", H=8,
          nnz_arrays=2),
    LCase("rgcn_edge_dot-gather-F300", "cogdl_b200_rgcn_edge_dot_f32", "X", "gather", "f32", 300, "cogdl_b200::rgcn_edge_dot_kernel<float4> block=128"),
    LCase("rgcn_edge_dot-edge-B8", "cogdl_b200_rgcn_edge_dot_f32", "P [nnz, B]", "edge", "f32", 1, "cogdl_b200::rgcn_edge_dot_kernel<float4> block=128", H=8,
          nnz_arrays=1),
    LCase("hgn_attn-edge", "cogdl_b200_hgn_attn_f32", "att_out/mix_out", "edge", "f32", 1, "cogdl_b200::hgn_stats_kernel<MODE=2> + cogdl_b200::hgn_main_kernel<MODE=2,CAP=512>", H=EDGE_H, n_big=2,
          nnz_arrays=1),
    LCase("hgn_attn_bwd-edge", "cogdl_b200_hgn_attn_bwd_f32", "att/d_mix/d_edge", "edge", "f32", 1, "cogdl_b200::hgn_stats_kernel<MODE=3> + cogdl_b200::hgn_main_kernel<MODE=3,CAP=512,DROP> cp.async.bulk tiles", H=EDGE_H,
          n_big=2, nnz_arrays=1),
    LCase("gcn_fused-gather-K128", "cogdl_b200_gcn_fused_f32", "X", "gather", "f32", 128, LEAN + " + " + FUSED.format("gcn", 64)),
    LCase("gcn_fused-store-K128", "cogdl_b200_gcn_fused_f32", "out/hub_agg", "store", "f32", 128, LEAN + " + " + FUSED.format("gcn", 128), n_big=2),
    LCase("sage_fused-gather-K128", "cogdl_b200_sage_fused_f32", "X", "gather", "f32", 128,
          LEAN + " + " + FUSED.format("sage-sum", 64)),
    LCase("sage_fused-store-K128", "cogdl_b200_sage_fused_f32", "hub_agg", "store", "f32", 128,
          LEAN + " + " + FUSED.format("sage-sum", 64)),
    LCase("actnn-minmax", "cogdl_b200_actnn_minmax_f32", "x", "elements", "f32", 300, "actnn_minmax<256>"),
    LCase("actnn-pack", "cogdl_b200_actnn_pack_f32", "x", "elements", "f32", 300, "actnn_pack<256>"),
    LCase("actnn-unpack", "cogdl_b200_actnn_unpack_f32", "out", "elements", "f32", 300, "actnn_unpack<256>", n_big=2),
    LCase("actnn-unpack-packed-2^32", "cogdl_b200_actnn_unpack_f32", "packed", "packed", "u8", 1, "actnn_unpack<256>",
          wrap=True),
    LCase("actnn-relu", "cogdl_b200_actnn_relu_fwd_f32", "x/y", "elements", "f32", 300, "actnn_relu_fwd", n_big=2),
    LCase("actnn-relu_bwd", "cogdl_b200_actnn_relu_bwd_f32", "g/gx", "elements", "f32", 300, "actnn_relu_bwd", n_big=2),
    LCase("actnn-dropout", "cogdl_b200_actnn_dropout_fwd_f32", "x/y", "elements", "f32", 300, "actnn_dropout_fwd", n_big=2),
    LCase("actnn-dropout_bwd", "cogdl_b200_actnn_dropout_bwd_f32", "g/gx", "elements", "f32", 300,
          "actnn_dropout_bwd", n_big=2),
]

LARGEST = max(TABLE, key=lambda c: c.bytes_needed)

# Entry points with no dense float operand a large-offset case could reach.
EXEMPT = {
    "cogdl_b200_spgemm_count": "sparse x sparse: no dense operand, and nnz < 2^31 by contract",
    "cogdl_b200_spgemm_fill_f32": "sparse x sparse: values are nnz-indexed, and nnz < 2^31 by contract",
    "cogdl_b200_spgemm_bwd_f32": "sparse x sparse: values are nnz-indexed, and nnz < 2^31 by contract",
    "cogdl_b200_csr2csc": "integer only, nnz < 2^31 by contract",
    "cogdl_b200_coo2csr_index": "integer only, int64 throughout",
    "cogdl_b200_narrow_i64_i32": "integer only, one int64 index per element",
    "cogdl_b200_sample_adj_count": "sampler: int64 indices throughout",
    "cogdl_b200_sample_adj_fill": "sampler: int64 indices; the int32 assoc is bounded by an explicit n_batch + n_edges guard",
    "cogdl_b200_subgraph_count": "sampler: int64 indices throughout",
    "cogdl_b200_subgraph_fill": "sampler: int64 indices; the int32 assoc is bounded by an explicit guard",
    "cogdl_b200_actnn_bits": "N < 2^28 by contract; its keys are indexed N * 7 < 2^31",
    "cogdl_b200_hub_plan_count": "integer only, reads rowptr",
    "cogdl_b200_hub_plan_fill": "integer only, reads rowptr",
    "cogdl_b200_edge_rows": "integer only, nnz < 2^31 by contract",
    "cogdl_b200_disen_route_bwd_f32": "every dense operand is [n, F] on a square structure (q, c, G, out, g_u, dq, dc); "
                                      "even with q = c and G = out aliased, five of them past 2^31 fp32 elements are "
                                      "43 GB, over the 20 GiB one case may hold on a shared GPU.  The forward's row "
                                      "(disen_route_fwd-store-K3d32) covers the same [n, F] row indexing",
}

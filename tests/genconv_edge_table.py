"""One row per case of the GENConv edge-encoder kernels (cogdl_b200/csrc/genconv_edge.cu): the forward
cogdl_b200_genconv_edge_fwd_f32 with and without Q, and the backward cogdl_b200_genconv_edge_bwd_f32 with dX, dW or
both, across row widths F (scalar, one float4 tile, two tiles, a partial last tile), feature counts D (each side of
the 8-weight instantiation, and 16), the hub / empty-row / rectangular graphs, the boundary-degree graphs of a hub plan
(boundary_csr for the forward, boundary_csc for the backward, whose transpose has the boundary degrees), no hub plan, a
16-edge chunk, an unaligned x, a plan partial scratch 4 bytes off 16-byte alignment, and a graph with more work items
than the backward's fixed grid has warps.  `kernel` is the name cogdl_b200_last_kernel() records for the row.  The
rows must name every kernel compiled into genconv_edge.o and no other, and cover every special form of
special_form() (tests/test_cpu_genconv_edge_inventory.py).

Two input families (tests/test_gpu_genconv_edge.py): "general" (attr ~ U[0, 1), W ~ N(0, 1/D)) and "exact" (attr in
{-2..2}, W a power of two times multiples of 1/8, so attr @ W.T is exact in fp32, with one pre-activation per column
that cancels to exactly 0).  Plain Python, no torch."""
from dataclasses import dataclass

MAX_D = 16               # GE_MAX_D of genconv_edge.cu
DM_SMALL = 8             # D <= 8 runs the 8-weight instantiation, 9..16 the 16-weight one
GE_WARPS = 8             # warps per block of the backward
GE_BWD_BLOCKS = 2 * 132  # the backward's fixed grid on an H100 (2 x NUM_SMS)
FS = (7, 16, 64, 128, 256)
DS = (1, 3, 8, 9, 16)
BETAS = (0.0, 0.5, 4.0, 20.0, -2.0)   # the exact family's sweep: none, moderate, large, larger, negative
TILE_FS = (260, 37)                   # 65 float4 vectors / 37 floats: several 32-vector tiles, the last partial


def wide_csr():
    """More backward work items (transpose columns + hub chunks at chunk 16) than GE_WARPS x GE_BWD_BLOCKS = 2112
    warps: every warp takes a second item.  Not in tests/graphs.CASES, whose parity tests would grow."""
    from tests.graphs import random_csr

    rp, ci = random_csr(6000, 50000, seed=3, hub=(5, 4000))
    return rp, ci, 6000


@dataclass(frozen=True)
class Row:
    id: str
    op: str                  # "fwd" or "bwd"
    F: int
    D: int
    graph: str               # a tests/graphs.py case, "bounds" / "bounds_t" (boundary_csr / _csc) or "wide"
    chunk: int = 0           # 0: the default chunk
    want_q: bool = False     # fwd: beta needs grad
    want: str = "dx_dw"      # bwd: "dx_dw", "dx" or "dw"
    aligned: bool = True
    beta: float = 1.3
    family: str = "general"  # "general" or "exact"
    plan: bool = True        # False: chunk_edges = 0, no hub plan
    partials_offset: int = 0  # bytes the plan's partial scratch is moved off 16-byte alignment (C entry point)

    @property
    def vec(self):
        return self.F % 4 == 0 and self.aligned and not self.partials_offset

    @property
    def kernel(self):
        v = "float4" if self.vec else "float"
        dm = DM_SMALL if self.D <= DM_SMALL else MAX_D
        if self.op == "fwd":
            return f"cogdl_b200::genconv_edge_fwd_kernel<{v},DM={dm},{'Q' if self.want_q else 'no_Q'}>"
        k = f"cogdl_b200::genconv_edge_bwd_kernel<{v},DM={dm}>"
        return k + (" + cogdl_b200::genconv_edge_dw_reduce_kernel" if "dw" in self.want else "")

    @property
    def n_tiles(self):
        fv = self.F // 4 if self.vec else self.F
        return -(-fv // 32)


def special_form(c):
    """The form a row checks beyond its instantiation, or None: ("exact", op, vector width, beta), ("noplan", op,
    width), (graph, op, width, chunk) on the boundary graphs, ("partials+4", op, want), ("tile", width) for several
    tiles with a partial last one, ("wide", want, D)."""
    v = "float4" if c.vec else "float"
    if c.family == "exact":
        return ("exact", c.op, v, c.beta)
    if not c.plan:
        return ("noplan", c.op, v)
    if c.graph in ("bounds", "bounds_t"):
        return (c.graph, c.op, v, c.chunk)
    if c.partials_offset:
        return ("partials+4", c.op, "Q" if c.want_q else c.want)
    if c.op == "bwd" and c.n_tiles > 1 and c.F % (128 if c.vec else 32):
        return ("tile", v)
    if c.graph == "wide":
        return ("wide", c.want, c.D)
    return None


def required_special_forms():
    forms = {("exact", op, v, b) for b in BETAS for op, v in (("fwd", "float4"), ("bwd", "float4"), ("bwd", "float"))}
    forms |= {("noplan", op, v) for op in ("fwd", "bwd") for v in ("float4", "float")}
    forms |= {(g, op, v, ch) for g, op in (("bounds", "fwd"), ("bounds_t", "bwd")) for v in ("float4", "float")
              for ch in (16, 64)}
    forms |= {("partials+4", "fwd", "Q"), ("partials+4", "bwd", "dx"), ("tile", "float4"), ("tile", "float")}
    forms |= {("wide", want, D) for want in ("dx_dw", "dw") for D in (3, 16)}
    return forms


def _b(beta):
    return f"b{beta:g}"


def _rows():
    rows = []
    for F in FS:
        for D in DS:
            for q in (False, True):
                rows.append(Row(f"fwd-F{F}-D{D}-{'Q' if q else 'noQ'}-two_hubs-c16", "fwd", F, D, "two_hubs", 16, q))
            for want in ("dx_dw", "dx", "dw"):
                rows.append(Row(f"bwd-F{F}-D{D}-{want}-two_hubs-c16", "bwd", F, D, "two_hubs", 16, want=want))
    for g in ("tiny", "empty_graph", "ragged", "hub", "rect"):
        for D in (3, 16):
            rows.append(Row(f"fwd-F64-D{D}-Q-{g}", "fwd", 64, D, g, want_q=True))
            rows.append(Row(f"bwd-F64-D{D}-dx_dw-{g}", "bwd", 64, D, g))
            rows.append(Row(f"bwd-F7-D{D}-dx_dw-{g}", "bwd", 7, D, g))
    for D in (8, 16):
        rows.append(Row(f"fwd-F128-D{D}-noQ-hub-unaligned", "fwd", 128, D, "hub", aligned=False))
        rows.append(Row(f"bwd-F128-D{D}-dx_dw-hub-unaligned", "bwd", 128, D, "hub", aligned=False))
    # exact family: the beta sweep, with exactly cancelling pre-activations
    for beta in BETAS:
        rows.append(Row(f"fwd-F64-D8-Q-two_hubs-c16-exact-{_b(beta)}", "fwd", 64, 8, "two_hubs", 16, True,
                        beta=beta, family="exact"))
        rows.append(Row(f"bwd-F64-D8-dx_dw-two_hubs-c16-exact-{_b(beta)}", "bwd", 64, 8, "two_hubs", 16,
                        beta=beta, family="exact"))
        rows.append(Row(f"bwd-F7-D3-dx_dw-hub-c16-exact-{_b(beta)}", "bwd", 7, 3, "hub", 16, beta=beta,
                        family="exact"))
    # no hub plan
    for F, D in ((64, 8), (7, 16)):
        rows.append(Row(f"fwd-F{F}-D{D}-Q-hub-noplan", "fwd", F, D, "hub", want_q=True, plan=False))
        rows.append(Row(f"bwd-F{F}-D{D}-dx_dw-hub-noplan", "bwd", F, D, "hub", plan=False))
    # the boundary degrees: rows of the forward, columns (transpose rows) of the backward
    for chunk in (16, 64):
        for F, D in ((64, 8), (7, 16)):
            rows.append(Row(f"fwd-F{F}-D{D}-Q-bounds-c{chunk}", "fwd", F, D, "bounds", chunk, True))
            rows.append(Row(f"bwd-F{F}-D{D}-dx_dw-bounds_t-c{chunk}", "bwd", F, D, "bounds_t", chunk))
    # plan partial scratch 4 bytes off 16-byte alignment: the scalar kernel at F % 4 == 0
    rows.append(Row("fwd-F64-D8-Q-two_hubs-c16-partials+4", "fwd", 64, 8, "two_hubs", 16, True, partials_offset=4))
    rows.append(Row("bwd-F64-D8-dx-two_hubs-c16-partials+4", "bwd", 64, 8, "two_hubs", 16, want="dx",
                    partials_offset=4))
    # several 32-vector tiles, the last one partial
    for F in TILE_FS:
        rows.append(Row(f"bwd-F{F}-D9-dx_dw-two_hubs-c16", "bwd", F, 9, "two_hubs", 16))
    # more work items than warps: dW carried across items, hub merges followed by more items, the full grid
    for D in (3, 16):
        for want in ("dx_dw", "dw"):
            rows.append(Row(f"bwd-F64-D{D}-{want}-wide-c16", "bwd", 64, D, "wide", 16, want=want))
    return rows


TABLE = _rows()

"""One row per case of the GENConv edge-encoder kernels (cogdl_b200/csrc/genconv_edge.cu): the forward
cogdl_b200_genconv_edge_fwd_f32 with and without Q, and the backward cogdl_b200_genconv_edge_bwd_f32 with dX, dW or
both, across row widths F (scalar, one float4 tile, two tiles), feature counts D (each side of the 8-weight
instantiation, and 16), the hub / empty-row / rectangular graphs, a 16-edge chunk and an unaligned x.  `kernel` is the
name cogdl_b200_last_kernel() records for the row.  The rows must name every kernel compiled into genconv_edge.o and no
other (tests/test_cpu_genconv_edge_inventory.py).  Plain Python, no torch."""
from dataclasses import dataclass

MAX_D = 16               # GE_MAX_D of genconv_edge.cu
DM_SMALL = 8             # D <= 8 runs the 8-weight instantiation, 9..16 the 16-weight one
FS = (7, 16, 64, 128, 256)
DS = (1, 3, 8, 9, 16)


@dataclass(frozen=True)
class Row:
    id: str
    op: str                  # "fwd" or "bwd"
    F: int
    D: int
    graph: str               # a tests/graphs.py case
    chunk: int = 0           # 0: the default chunk
    want_q: bool = False     # fwd: beta needs grad
    want: str = "dx_dw"      # bwd: "dx_dw", "dx" or "dw"
    aligned: bool = True

    @property
    def vec(self):
        return self.F % 4 == 0 and self.aligned

    @property
    def kernel(self):
        v = "float4" if self.vec else "float"
        dm = DM_SMALL if self.D <= DM_SMALL else MAX_D
        if self.op == "fwd":
            return f"cogdl_b200::genconv_edge_fwd_kernel<{v},DM={dm},{'Q' if self.want_q else 'no_Q'}>"
        k = f"cogdl_b200::genconv_edge_bwd_kernel<{v},DM={dm}>"
        return k + (" + cogdl_b200::genconv_edge_dw_reduce_kernel" if "dw" in self.want else "")


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
    return rows


TABLE = _rows()

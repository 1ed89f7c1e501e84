"""One row per case of the R-GCN kernels (cogdl_b200/csrc/rgcn.cu): the fan-out aggregation cogdl_b200_rgcn_aggr_f32,
its per-basis form and the edge dot cogdl_b200_rgcn_edge_dot_f32, across row widths F, basis counts B (one basis
tile, the tile, the tile + 1, two tiles), type counts T, the hub / empty-row / boundary-degree graphs and an unaligned
x.  `kernel` is the name cogdl_b200_last_kernel() records for the row.  The rows must name every kernel compiled into
rgcn.o and no other (tests/test_cpu_rgcn_inventory.py).  Plain Python, no torch."""
from dataclasses import dataclass

BASIS_TILE = 8           # RGCN_BT of rgcn.cu: bases per pass
FS = (1, 7, 16, 100, 128, 200, 256)
BS = (1, 2, 5, BASIS_TILE, BASIS_TILE + 1, 16)
TS = (1, 3, 237)


@dataclass(frozen=True)
class Row:
    id: str
    op: str                  # "aggr", "per_basis" or "dot"
    F: int
    B: int
    T: int
    graph: str               # a tests/graphs.py case, or "bounds" (boundary-degree graph under a 64-edge plan)
    aligned: bool = True

    @property
    def vec(self):
        return self.F % 4 == 0 and self.aligned

    @property
    def kernel(self):
        v = "float4" if self.vec else "float"
        if self.op == "dot":
            return f"cogdl_b200::rgcn_edge_dot_kernel<{v}>"
        return f"cogdl_b200::rgcn_fanout_kernel<{v}{',per_basis' if self.op == 'per_basis' else ''}>"


def _rows():
    rows = []
    for op in ("aggr", "per_basis", "dot"):
        for F in FS:
            for B in BS:
                rows.append(Row(f"{op}-F{F}-B{B}-T3-hub", op, F, B, 3, "hub"))
        for T in (1, 237):
            for B in (1, 5, BASIS_TILE + 1):
                rows.append(Row(f"{op}-F200-B{B}-T{T}-two_hubs", op, 200, B, T, "two_hubs"))
        for g in ("ragged", "tiny", "bounds", "rect"):
            rows.append(Row(f"{op}-F128-B5-T3-{g}", op, 128, 5, 3, g))
            rows.append(Row(f"{op}-F7-B5-T3-{g}", op, 7, 5, 3, g))
        rows.append(Row(f"{op}-F128-B5-T3-hub-unaligned", op, 128, 5, 3, "hub", aligned=False))
        rows.append(Row(f"{op}-F200-B9-T237-bounds-unaligned", op, 200, 9, 237, "bounds", aligned=False))
    return rows


TABLE = _rows()

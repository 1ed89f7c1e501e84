"""One row per case of the Simple-HGN attention kernels (cogdl_b200/csrc/simple_hgn.cu): the forward stage
cogdl_b200_hgn_attn_f32 (with and without dropout and residual attention) and its backward cogdl_b200_hgn_attn_bwd_f32,
across head counts H (the 512-, 1024- and 2048-float tiles of the segment kernel, H = 1 and head counts that take the
generic kernel), type counts T (1, 5 and the table's cap), the tests/graphs.py cases and boundary_csr, with and without
a hub plan.  "bounds_t" (boundary_csc) rows put the boundary degrees on the columns, which the backward walks: the
multi-head SpMM with permutation for d h and the column sums for d h_r meet hub columns of degree C - 1, C, C + 1, 2C
and 129C + 5.  One row blends with alpha = 1 (every gradient but those of h and res_attn exactly 0).  `kernel` is the
main kernel cogdl_b200_last_kernel() records for the row and `stats` the statistics kernel recorded before it (hub rows
under a plan).  The rows must name every kernel compiled into simple_hgn.o and no other, and every launch form must
have a bounds_t row (tests/test_cpu_hgn_inventory.py).  Plain Python, no torch."""
from dataclasses import dataclass

MAX_TABLE = 1024         # HGN_MAX_TABLE of simple_hgn.cu: T * H
CHUNK = 64               # hub chunk edges of the planned rows
HUB_GRAPHS = ("hub", "two_hubs", "bounds", "bounds_t")
ALPHA = 0.05             # weight of res_attn in the blend, unless a row says otherwise


@dataclass(frozen=True)
class Row:
    id: str
    H: int
    T: int
    graph: str               # a tests/graphs.py case, or "bounds" (boundary-degree graph under the 64-edge plan)
    plan: bool               # hub plan with row-stream segments (chunk_edges = 64), else none
    res: bool                # res_attn given (the blend)
    p: float                 # attention dropout
    alpha: float = ALPHA     # weight of res_attn (with res)

    @property
    def form(self):
        if self.H > 32 or self.H & (self.H - 1):
            return "generic"
        return "main" if self.plan and CHUNK * self.H <= 2048 else "warp"

    def kernel(self, mode):
        flags = (",DROP" if self.p > 0 or mode == 3 else "") + (",MIX" if self.res and mode == 2 else "")
        if self.form == "main":
            cap = next(c for c in (512, 1024, 2048) if CHUNK * self.H <= c)
            return f"cogdl_b200::hgn_main_kernel<MODE={mode},CAP={cap}{flags}>"
        return f"cogdl_b200::hgn_{self.form}_kernel<MODE={mode}{flags}>"

    def stats(self, mode):
        has_hub = self.graph in HUB_GRAPHS
        return f"cogdl_b200::hgn_stats_kernel<MODE={mode}>" if self.form == "main" and has_hub else None


def _rows():
    rows = []
    for H, graphs in ((8, ("hub", "two_hubs", "ragged", "tiny", "rect", "empty_graph", "bounds")), (16, ("hub",)),
                      (32, ("two_hubs",)), (2, ("hub", "ragged")), (1, ("hub", "bounds")), (3, ("ragged",)),
                      (64, ("tiny",))):
        for g in graphs:
            for plan in ((True, False) if g in ("hub", "ragged") else (True,)):
                for res in (False, True):
                    for p in (0.0, 0.5):
                        T = {8: 5, 16: 1, 32: MAX_TABLE // 32, 2: MAX_TABLE // 2, 1: 5, 3: 5, 64: MAX_TABLE // 64}[H]
                        rows.append(Row(f"H{H}-T{T}-{g}-{'plan' if plan else 'noplan'}-{'res' if res else 'nores'}-p{p}",
                                        H, T, g, plan, res, p))
    for T in (1, MAX_TABLE // 8):
        rows.append(Row(f"H8-T{T}-two_hubs-plan-res-p0.5", 8, T, "two_hubs", True, True, 0.5))
    # the backward over boundary-degree columns, one row per launch form (main at each tile, warp, generic)
    for H, plan, res, p in ((1, True, False, 0.0), (8, True, True, 0.5), (16, True, False, 0.5), (32, True, True, 0.0),
                            (8, False, False, 0.0), (3, True, True, 0.5)):
        rows.append(Row(f"H{H}-T5-bounds_t-{'plan' if plan else 'noplan'}-{'res' if res else 'nores'}-p{p}", H, 5,
                        "bounds_t", plan, res, p))
    rows.append(Row("H8-T5-hub-plan-res-p0.5-alpha1", 8, 5, "hub", True, True, 0.5, alpha=1.0))
    return rows


def form_key(c):
    """The launch form of a row: the main kernel's tile (CAP), or the warp / generic kernel."""
    if c.form == "main":
        return f"main-{next(cap for cap in (512, 1024, 2048) if CHUNK * c.H <= cap)}"
    return c.form


TABLE = _rows()

"""One row per dispatch branch of the gather kernels in spmm.cu, sddmm.cu, mhspmm.cu and scatter_max.cu.

Each row names the inputs that select a kernel instantiation (op, graph, width, alignment, plan form, weights,
perm, dropout, source form) and the exact cogdl_b200_last_kernel() string the call must record.  The GPU test
(test_gpu_dispatch.py) runs every row and checks the output against a reference; the CPU test
(test_cpu_kernel_inventory.py) checks that the rows cover every kernel compiled into those four objects, and
that every kernel named here is compiled.  Plain Python, no torch: the CPU test imports it without a GPU.
"""
from dataclasses import dataclass

# threads per block of every row-stream launch (STREAM_BLOCK, stream.cuh), appended to the stream kernels' names
STREAM_BLOCK = 128


@dataclass(frozen=True)
class Case:
    op: str                 # spmm | spmm_f16 | sddmm | mhspmm | scatter_max | scatter_max_bwd
    graph: str              # a name in tests/graphs.py CASES
    F: int                  # features per head
    kernel: str             # exact cogdl_b200_last_kernel() after the call
    H: int = 1              # heads (sddmm: H > 1 calls the multi-head SDDMM)
    aligned: bool = True    # False: the feature input is a view one element past an aligned allocation
    plan: str = "default"   # none (no hub plan) | chunks (hub chunks, seg_cost 0) | default (chunks + segments)
    chunk: int = 64         # hub chunk edges of the plan
    weighted: bool = True   # spmm / spmm_f16: edge values, or the unweighted form
    perm: bool = False      # mhspmm: the transposed pass with the attention permutation fused
    drop: bool = False      # mhspmm: attention carrying a dropout mask in its sign bit (cogdl_b200_mhspmm_dropout_f32)
    src: str = "one"        # spmm: one | two (cogdl_b200_spmm_csr_f32_2src) | peers (cogdl_b200_spmm_csr_f32_peers)
    panels: int = 0         # spmm: column panels of X (0: chosen by the library)
    partials_offset: int = 0  # bytes the plan's partial scratch starts past a 16-byte boundary

    @property
    def id(self):
        s = f"{self.op}-{self.graph}-H{self.H}F{self.F}-{self.plan}"
        if self.op in ("spmm", "spmm_f16"):
            s += "-w" if self.weighted else "-u"
        if not self.aligned:
            s += "-misaligned"
        for flag in ("perm", "drop"):
            if getattr(self, flag):
                s += "-" + flag
        if self.src != "one":
            s += "-" + self.src
        if self.panels:
            s += f"-P{self.panels}"
        if self.partials_offset:
            s += f"-partials+{self.partials_offset}"
        return s


# ------------------------------------------------------------------ kernel names, as the launchers format them
def _w(weighted):
    return "weighted" if weighted else "unweighted"


def spmm_k(vec, group, nv, weighted):
    return f"cogdl_b200::spmm_kernel<{vec},GROUP={group},NV={nv},{_w(weighted)}>"


def stream_k(vec, nv, what, src, u, minb, prefetch, panels=0):
    s = f"cogdl_b200::stream_kernel<{vec},NV={nv},{what},{src},U={u},MINB={minb}{',prefetch' if prefetch else ''}>"
    if panels > 1:
        s += f",panels={panels}"
    return s + f" block={STREAM_BLOCK}"


def half_k(weighted, vec):
    return f"cogdl_b200::spmm_half_kernel<{_w(weighted)},{'vec' if vec else 'scalar'}>"


def sddmm_k(vec, group, sub, nv):
    return f"cogdl_b200::sddmm_kernel<{vec},GROUP={group},SUB={sub},NV={nv}>"


def sddmm_stream_k(nv):
    return f"cogdl_b200::sddmm_stream_kernel<NV={nv},U={4 if nv == 1 else 2}>"


def mh_k(vec, group, perm, drop):
    return f"cogdl_b200::mhspmm_kernel<{vec},GROUP={group},{'perm' if perm else 'no_perm'}{',drop' if drop else ''}>"


def mh_stream_k(vec, perm, drop):
    what = "multihead" + ("+perm" if perm else "") + ("+drop" if drop else "")
    return stream_k(vec, 1, what, "SRC_ONE", 8, 3, True)


def smax_k(vec, group, nv):
    return f"cogdl_b200::scatter_max_fwd_kernel<{vec},GROUP={group},NV={nv}>"


def smax_stream_k(nv):
    return f"cogdl_b200::scatter_max_stream_kernel<NV={nv},U={4 if nv == 1 else 2}>"


SMAX_BWD = "cogdl_b200::scatter_max_bwd_kernel"


# ------------------------------------------------------------------ SpMM (fp32): cogdl_b200_spmm_csr_f32_ex / _2src / _peers
def _spmm_rows(w):
    S = lambda vec, nv, src, u, minb, pf, panels=0: stream_k(vec, nv, _w(w), src, u, minb, pf, panels)  # noqa: E731
    lean4 = lambda src: S("float4", 1, src, 4, 5, False)   # noqa: E731  float4, one vector per lane
    nv2_4 = lambda src: S("float4", 2, src, 4, 1, True)    # noqa: E731
    nv1_f = lambda src: S("float", 1, src, 8, 1, True)     # noqa: E731
    nv2_f = lambda src: S("float", 2, src, 4, 1, True)     # noqa: E731
    nv4_f = lambda src: S("float", 4, src, 2, 1, True)     # noqa: E731
    C = lambda graph, F, kernel, **kw: Case("spmm", graph, F, kernel, weighted=w, **kw)  # noqa: E731
    return [
        # row kernels, float4 (F % 4 == 0, aligned): GROUP = F/4 vectors rounded up to a power of two
        C("two_hubs", 4, spmm_k("float4", 1, 1, w), plan="chunks"),
        C("hub", 8, spmm_k("float4", 2, 1, w), plan="none"),
        C("two_hubs", 16, spmm_k("float4", 4, 1, w), plan="chunks"),
        C("two_hubs", 32, spmm_k("float4", 8, 1, w)),                    # 8 vectors: row kernel even with segments
        C("two_hubs", 64, spmm_k("float4", 16, 1, w), plan="chunks"),
        C("hub", 128, spmm_k("float4", 32, 1, w), plan="chunks"),
        C("two_hubs", 300, spmm_k("float4", 32, 2, w), plan="chunks"),   # 75 vectors: two column tiles
        # row kernels, float (F % 4 != 0, or a misaligned view)
        C("two_hubs", 1, spmm_k("float", 1, 1, w)),
        C("hub", 2, spmm_k("float", 2, 1, w), plan="chunks"),
        C("two_hubs", 3, spmm_k("float", 4, 1, w), plan="chunks"),
        C("two_hubs", 8, spmm_k("float", 8, 1, w), aligned=False),
        C("two_hubs", 9, spmm_k("float", 16, 1, w), plan="chunks"),
        C("hub", 17, spmm_k("float", 32, 1, w), plan="none"),
        C("two_hubs", 40, spmm_k("float", 32, 2, w), plan="chunks", aligned=False),
        C("two_hubs", 65, spmm_k("float", 32, 4, w), plan="chunks"),
        C("two_hubs", 129, spmm_k("float", 32, 4, w), plan="chunks"),   # one column past the first 128-float tile
        C("two_hubs", 1433, spmm_k("float", 32, 4, w), plan="chunks"),  # Cora's raw feature width
        C("hub", 3703, spmm_k("float", 32, 4, w), plan="none"),         # Citeseer's
        # row-stream kernels (plan with segments), float4
        C("two_hubs", 40, lean4("SRC_ONE")),
        C("two_hubs", 128, lean4("SRC_TWO"), src="two"),
        C("two_hubs", 64, lean4("SRC_PEERS"), src="peers"),
        C("two_hubs", 300, nv2_4("SRC_ONE")),
        C("two_hubs", 256, nv2_4("SRC_TWO"), src="two"),
        C("two_hubs", 260, nv2_4("SRC_PEERS"), src="peers"),
        # row-stream kernels, float; the peer form takes them only when the partial scratch is not 16-byte aligned
        C("two_hubs", 9, nv1_f("SRC_ONE")),
        C("two_hubs", 17, nv1_f("SRC_TWO"), src="two"),
        C("two_hubs", 32, nv1_f("SRC_PEERS"), src="peers", partials_offset=4),
        C("two_hubs", 33, nv2_f("SRC_ONE")),
        C("two_hubs", 64, nv2_f("SRC_TWO"), src="two", aligned=False),
        C("two_hubs", 64, nv2_f("SRC_PEERS"), src="peers", partials_offset=4),
        C("two_hubs", 1433, nv4_f("SRC_ONE")),
        C("hub", 3703, nv4_f("SRC_ONE")),
        C("two_hubs", 130, nv4_f("SRC_TWO"), src="two"),
        C("two_hubs", 128, nv4_f("SRC_PEERS"), src="peers", partials_offset=4),
        # panel form: 32-, 64- and 128-float column panels
        C("two_hubs", 64, S("float", 1, "SRC_ONE", 8, 6, True, 2), panels=2),
        C("two_hubs", 128, S("float2", 1, "SRC_ONE", 8, 5, True, 2), panels=2),
        C("two_hubs", 256, S("float4", 1, "SRC_ONE", 4, 5, True, 2), panels=2),
    ]


SPMM = _spmm_rows(True) + _spmm_rows(False)

# ------------------------------------------------------------------ SpMM (fp16 storage): cogdl_b200_spmm_csr_f16
SPMM_F16 = []
for _w_ in (True, False):
    SPMM_F16 += [
        Case("spmm_f16", "hub", 128, half_k(_w_, True), weighted=_w_),
        Case("spmm_f16", "two_hubs", 300, half_k(_w_, True), plan="none", weighted=_w_),    # three column tiles
        Case("spmm_f16", "two_hubs", 33, half_k(_w_, False), plan="chunks", weighted=_w_),
        Case("spmm_f16", "hub", 64, half_k(_w_, False), aligned=False, weighted=_w_),       # X 2 bytes past 8
        Case("spmm_f16", "two_hubs", 129, half_k(_w_, False), weighted=_w_),
    ]

# ------------------------------------------------------------------ SDDMM: cogdl_b200_sddmm_csr_f32 (H = 1) / _mhsddmm_f32
SDDMM = [
    Case("sddmm", "two_hubs", 128, sddmm_stream_k(1)),                      # 32 vectors per head, with segments
    Case("sddmm", "two_hubs", 256, sddmm_stream_k(2), H=2),                 # 64
    # (H, F) -> (GROUP, SUB, NV) of the row kernel; float4 rows first, then the same branches in float
    Case("sddmm", "two_hubs", 600, sddmm_k("float4", 32, 32, 0), plan="chunks"),
    Case("sddmm", "hub", 300, sddmm_k("float4", 32, 32, 4)),
    Case("sddmm", "two_hubs", 256, sddmm_k("float4", 32, 32, 2), plan="chunks"),
    Case("sddmm", "two_hubs", 128, sddmm_k("float4", 32, 32, 1), H=2, plan="none"),
    Case("sddmm", "two_hubs", 40, sddmm_k("float4", 32, 16, 1), H=2),
    Case("sddmm", "hub", 64, sddmm_k("float4", 16, 16, 1), plan="chunks"),
    Case("sddmm", "two_hubs", 32, sddmm_k("float4", 32, 8, 1), H=4),
    Case("sddmm", "two_hubs", 24, sddmm_k("float4", 16, 8, 1), H=3),
    Case("sddmm", "two_hubs", 20, sddmm_k("float4", 8, 8, 1)),
    Case("sddmm", "two_hubs", 16, sddmm_k("float4", 32, 4, 1), H=8),
    Case("sddmm", "hub", 12, sddmm_k("float4", 16, 4, 1), H=5),
    Case("sddmm", "two_hubs", 16, sddmm_k("float4", 8, 4, 1), H=2),
    Case("sddmm", "two_hubs", 12, sddmm_k("float4", 4, 4, 1)),
    Case("sddmm", "two_hubs", 8, sddmm_k("float4", 16, 2, 1), H=8),
    Case("sddmm", "two_hubs", 8, sddmm_k("float4", 8, 2, 1), H=6),
    Case("sddmm", "hub", 8, sddmm_k("float4", 4, 2, 1)),
    Case("sddmm", "two_hubs", 4, sddmm_k("float4", 8, 1, 1), H=8),
    Case("sddmm", "two_hubs", 4, sddmm_k("float4", 4, 1, 1), H=4),
    Case("sddmm", "two_hubs", 4, sddmm_k("float4", 2, 1, 1), H=2),
    Case("sddmm", "two_hubs", 4, sddmm_k("float4", 1, 1, 1)),
    Case("sddmm", "two_hubs", 129, sddmm_k("float", 32, 32, 0), H=2),
    Case("sddmm", "two_hubs", 65, sddmm_k("float", 32, 32, 4), H=3),
    Case("sddmm", "hub", 64, sddmm_k("float", 32, 32, 2), aligned=False),    # a float4 width, misaligned
    Case("sddmm", "two_hubs", 33, sddmm_k("float", 32, 32, 2), plan="chunks"),
    Case("sddmm", "two_hubs", 17, sddmm_k("float", 32, 32, 1)),
    Case("sddmm", "two_hubs", 9, sddmm_k("float", 32, 16, 1), H=3),
    Case("sddmm", "two_hubs", 16, sddmm_k("float", 16, 16, 1), aligned=False),
    Case("sddmm", "two_hubs", 5, sddmm_k("float", 32, 8, 1), H=4),
    Case("sddmm", "two_hubs", 7, sddmm_k("float", 16, 8, 1), H=2),
    Case("sddmm", "two_hubs", 8, sddmm_k("float", 8, 8, 1), aligned=False),
    Case("sddmm", "two_hubs", 3, sddmm_k("float", 32, 4, 1), H=8),
    Case("sddmm", "two_hubs", 4, sddmm_k("float", 16, 4, 1), H=4, aligned=False),
    Case("sddmm", "hub", 3, sddmm_k("float", 8, 4, 1), H=3),
    Case("sddmm", "two_hubs", 4, sddmm_k("float", 4, 4, 1), aligned=False),
    Case("sddmm", "two_hubs", 2, sddmm_k("float", 16, 2, 1), H=9),
    Case("sddmm", "two_hubs", 2, sddmm_k("float", 8, 2, 1), H=4),
    Case("sddmm", "two_hubs", 2, sddmm_k("float", 4, 2, 1), H=3),
    Case("sddmm", "two_hubs", 1, sddmm_k("float", 8, 1, 1), H=16),
    Case("sddmm", "two_hubs", 1, sddmm_k("float", 4, 1, 1), H=5),
    Case("sddmm", "hub", 1, sddmm_k("float", 2, 1, 1), H=2),
    Case("sddmm", "two_hubs", 1, sddmm_k("float", 1, 1, 1)),
]

# ------------------------------------------------------------------ multi-head SpMM: cogdl_b200_mhspmm_f32 / _dropout_f32
# (vec, H, F, plan, aligned) -> GROUP = H*F vectors rounded up to a power of two, at most 32; 32 with segments: row-stream
_MH_SHAPES = [
    ("float4", 1, 4, "chunks", True, 1),
    ("float4", 2, 4, "default", True, 2),
    ("float4", 3, 4, "none", True, 4),
    ("float4", 2, 16, "chunks", True, 8),
    ("float4", 8, 8, "default", True, 16),
    ("float4", 8, 16, "chunks", True, 32),
    ("float4", 3, 64, "none", True, 32),
    ("float4", 8, 128, "default", True, "stream"),
    ("float4", 3, 44, "default", True, "stream"),
    ("float", 1, 1, "chunks", True, 1),
    ("float", 2, 1, "default", True, 2),
    ("float", 1, 3, "none", True, 4),
    ("float", 3, 2, "chunks", True, 8),
    ("float", 3, 5, "default", True, 16),
    ("float", 4, 9, "chunks", True, 32),
    ("float", 8, 16, "none", False, 32),
    ("float", 8, 16, "default", False, "stream"),
    ("float", 2, 33, "default", True, "stream"),
]
MHSPMM = []
for _vec, _H, _F, _plan, _al, _g in _MH_SHAPES:
    for _perm in (False, True):
        for _drop in (False, True):
            _k = mh_stream_k(_vec, _perm, _drop) if _g == "stream" else mh_k(_vec, _g, _perm, _drop)
            # the transposed pass runs on the CSC, whose column degrees are small: 16-edge chunks still split some
            MHSPMM.append(Case("mhspmm", "two_hubs", _F, _k, H=_H, aligned=_al, plan=_plan, perm=_perm, drop=_drop,
                               chunk=16 if _perm else 64))

# ------------------------------------------------------------------ scatter_max: cogdl_b200_scatter_max_fwd_f32 / _bwd_f32
SCATTER_MAX = [
    Case("scatter_max", "two_hubs", 4, smax_k("float4", 1, 1)),
    Case("scatter_max", "hub", 8, smax_k("float4", 2, 1), plan="chunks"),
    Case("scatter_max", "two_hubs", 16, smax_k("float4", 4, 1), plan="none"),
    Case("scatter_max", "two_hubs", 32, smax_k("float4", 8, 1)),
    Case("scatter_max", "two_hubs", 64, smax_k("float4", 16, 1)),                # 16 vectors: row kernel with segments
    Case("scatter_max", "two_hubs", 128, smax_k("float4", 32, 1), plan="chunks"),
    Case("scatter_max", "two_hubs", 300, smax_k("float4", 32, 2), plan="chunks"),
    Case("scatter_max", "two_hubs", 128, smax_stream_k(1)),
    Case("scatter_max", "two_hubs", 300, smax_stream_k(2)),
    Case("scatter_max", "two_hubs", 1, smax_k("float", 1, 1)),
    Case("scatter_max", "hub", 2, smax_k("float", 2, 1), plan="chunks"),
    Case("scatter_max", "two_hubs", 3, smax_k("float", 4, 1)),
    Case("scatter_max", "two_hubs", 5, smax_k("float", 8, 1), plan="none"),
    Case("scatter_max", "two_hubs", 16, smax_k("float", 16, 1), aligned=False),
    Case("scatter_max", "two_hubs", 17, smax_k("float", 32, 1), plan="chunks"),
    Case("scatter_max", "two_hubs", 128, smax_k("float", 32, 2), aligned=False),  # no row-stream form in float
    Case("scatter_max", "hub", 1433, smax_k("float", 32, 2), plan="chunks"),
    Case("scatter_max_bwd", "two_hubs", 33, SMAX_BWD),
]

TABLE = SPMM + SPMM_F16 + SDDMM + MHSPMM + SCATTER_MAX

# Compiled instantiations no public entry point above reaches: launched only by the fused layers' hub-row pre-pass.
EXEMPT = {
    "cogdl_b200::scatter_max_stream_kernel<NV=1,U=4,values_only>":
        "smax_hub_rows_only (fused SAGE max layer): tests/test_gpu_fused_sage.py",
}

"""One row per dispatch branch of the gather kernels in spmm.cu, sddmm.cu, mhspmm.cu and scatter_max.cu, and of the
edge softmax and GAT attention kernels in edge_softmax.cu.

Each row names the inputs that select a kernel instantiation (op, graph, width, alignment, plan form, weights,
perm, dropout, source form) and the exact cogdl_b200_last_kernel() string the call must record.  The GPU test
(test_gpu_dispatch.py) runs every row and checks the output against a reference; the CPU test
(test_cpu_kernel_inventory.py) checks that the rows cover every kernel compiled into those five objects, and
that every kernel named here is compiled.  Plain Python, no torch: the CPU test imports it without a GPU.
"""
from dataclasses import dataclass

# threads per block of every row-stream launch (STREAM_BLOCK, stream.cuh), appended to the stream kernels' names
STREAM_BLOCK = 128


@dataclass(frozen=True)
class Case:
    op: str                 # spmm | spmm_f16 | sddmm | mhspmm | scatter_max | scatter_max_bwd | edge_softmax |
                            # edge_softmax_bwd | gat_fwd | gat_attn_bwd
    graph: str              # a name in tests/graphs.py CASES, or "bounds": boundary_csr(chunk)
    F: int                  # features per head
    kernel: str             # exact cogdl_b200_last_kernel() after the call
    H: int = 1              # heads (sddmm: H > 1 calls the multi-head SDDMM)
    aligned: bool = True    # False: the feature input (edge_softmax: the logits; the backwards: g) is a view one
                            # element past an aligned allocation
    plan: str = "default"   # none (no hub plan) | chunks (hub chunks, seg_cost 0) | default (chunks + segments)
    chunk: int = 64         # hub chunk edges of the plan
    weighted: bool = True   # spmm / spmm_f16: edge values, or the unweighted form
    perm: bool = False      # mhspmm: the transposed pass with the attention permutation fused
    drop: bool = False      # mhspmm: attention carrying a dropout mask in its sign bit (cogdl_b200_mhspmm_dropout_f32)
                            # gat_fwd / gat_attn_bwd: the attention-dropout entry points
    src: str = "one"        # spmm: one | two (cogdl_b200_spmm_csr_f32_2src) | peers (cogdl_b200_spmm_csr_f32_peers)
    panels: int = 0         # spmm: column panels of X (0: chosen by the library)
    partials_offset: int = 0  # bytes the plan's partial scratch starts past a 16-byte boundary
    masked: bool = False    # edge_softmax: -inf logits (leading, middle and trailing in a row, a whole first hub chunk,
                            # a (row, head) of nothing but -inf)

    @property
    def id(self):
        s = f"{self.op}-{self.graph}-H{self.H}F{self.F}-{self.plan}"
        if self.op in ES_OPS:
            s += f"-C{self.chunk}"
        if self.op in ("spmm", "spmm_f16"):
            s += "-w" if self.weighted else "-u"
        if not self.aligned:
            s += "-misaligned"
        for flag in ("perm", "drop", "masked"):
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

# ------------------------------------------------------------------ edge softmax and the GAT attention (edge_softmax.cu)
# cogdl_b200_edge_softmax_fwd_f32 (MODE 0) / _bwd_f32 (MODE 1), the attention of cogdl_b200_gat_fwd_f32 /
# _dropout_f32 (MODE 2, followed by the multi-head SpMM) and cogdl_b200_gat_attn_bwd_f32 / _dropout_f32 (MODE 3).
# With a plan that has segments and chunk_edges * H <= 2048 the main kernel runs with the smallest tile of 512, 1024
# or 2048 floats that holds chunk_edges * H, after the statistics kernel when the graph has hub rows; otherwise a warp
# per row.  Head counts that are not a power of two <= 32 take the generic kernel.
ES_OPS = ("edge_softmax", "edge_softmax_bwd", "gat_fwd", "gat_attn_bwd")
ES_WARPS = 8


def es_main(mode, cap, drop=False, bulk=False, stats=True):
    """Main kernel, staged by cp.async.bulk (bulk) or coalesced loads, preceded by the statistics kernel (stats), whose
    forward attention runs without the dropout flag."""
    s = f"cogdl_b200::es_main_kernel<MODE={mode},CAP={cap},WARPS={ES_WARPS}{',DROP' if drop else ''}>"
    s += " cp.async.bulk tiles" if bulk else ""
    if stats:
        s = f"cogdl_b200::es_stats_kernel<MODE={mode}{',DROP' if drop and mode == 3 else ''}> + " + s
    return s


def es_warp(mode, drop=False):
    return f"cogdl_b200::es_warp_kernel<MODE={mode}{',DROP' if drop else ''}>"


def es_generic(mode, drop=False):
    return f"cogdl_b200::es_generic_kernel<MODE={mode}{',DROP' if drop else ''}>"


def gat_k(attention, aggregation):
    return f"{attention} + {aggregation}"


def _es_rows(op, mode):
    """edge_softmax (MODE 0) or edge_softmax_bwd (MODE 1): the forward's logits carry -inf masks."""
    m = mode == 0
    C = lambda graph, kernel, **kw: Case(op, graph, 0, kernel, masked=m, **kw)  # noqa: E731
    return [
        C("bounds", es_main(mode, 512, bulk=True), H=8, chunk=64),
        C("bounds", es_main(mode, 512), H=8, chunk=64, aligned=False),
        C("bounds", es_main(mode, 1024, bulk=True), H=4, chunk=256),
        C("bounds", es_main(mode, 2048, bulk=True), H=32, chunk=64),
        C("bounds", es_main(mode, 2048), H=1, chunk=2048),              # H % 4 != 0: coalesced staging
        C("bounds", es_warp(mode), H=16, chunk=256),                    # 4096 floats: no tile holds a chunk
        C("bounds", es_warp(mode), H=8, chunk=64, plan="none"),
        C("bounds", es_generic(mode), H=3, chunk=64),
        C("bounds", es_generic(mode), H=6, chunk=64),
        C("bounds", es_generic(mode), H=64, chunk=64),                  # a power of two above 32
        C("ragged", es_main(mode, 512, bulk=True, stats=False), H=8, chunk=64),     # no hub rows
        # 512-float tiles on a graph with a 700-edge hub, without masks
        Case(op, "two_hubs", 0, es_main(mode, 512, bulk=True), H=8, chunk=64),
        Case(op, "two_hubs", 0, es_main(mode, 512, bulk=True), H=4, chunk=64),
    ]


EDGE_SOFTMAX = _es_rows("edge_softmax", 0) + _es_rows("edge_softmax_bwd", 1)

GAT_FWD = []
GAT_ATTN_BWD = []
for _d in (False, True):
    _S = lambda vec: mh_stream_k(vec, False, _d)  # noqa: E731
    _M = lambda vec, group: mh_k(vec, group, False, _d)  # noqa: E731
    _G = lambda graph, F, att, agg, **kw: Case("gat_fwd", graph, F, gat_k(att, agg), drop=_d, **kw)  # noqa: E731
    GAT_FWD += [
        _G("bounds", 16, es_main(2, 512, _d), _S("float4"), H=8, chunk=64),
        _G("bounds", 32, es_main(2, 1024, _d), _S("float4"), H=4, chunk=256),
        _G("bounds", 4, es_main(2, 2048, _d), _S("float4"), H=32, chunk=64),
        _G("bounds", 8, es_main(2, 2048, _d), _M("float4", 2), H=1, chunk=2048),
        _G("bounds", 8, es_warp(2, _d), _S("float4"), H=16, chunk=256),
        _G("bounds", 16, es_warp(2, _d), _M("float4", 32), H=8, chunk=64, plan="none"),
        _G("bounds", 5, es_generic(2, _d), _M("float", 16), H=3, chunk=64),
        _G("bounds", 4, es_generic(2, _d), _M("float4", 8), H=6, chunk=64),
        _G("bounds", 4, es_generic(2, _d), _S("float4"), H=64, chunk=64),
        _G("ragged", 16, es_main(2, 512, _d, stats=False), _S("float4"), H=8, chunk=64),
    ]
    _B = lambda graph, kernel, **kw: Case("gat_attn_bwd", graph, 0, kernel, drop=_d, **kw)  # noqa: E731
    GAT_ATTN_BWD += [
        _B("bounds", es_main(3, 512, _d, bulk=True), H=8, chunk=64),
        _B("bounds", es_main(3, 512, _d), H=8, chunk=64, aligned=False),
        _B("bounds", es_main(3, 1024, _d, bulk=True), H=4, chunk=256),
        _B("bounds", es_main(3, 2048, _d, bulk=True), H=32, chunk=64),
        _B("bounds", es_main(3, 2048, _d), H=1, chunk=2048),
        _B("bounds", es_warp(3, _d), H=16, chunk=256),
        _B("bounds", es_warp(3, _d), H=8, chunk=64, plan="none"),
        _B("bounds", es_generic(3, _d), H=3, chunk=64),
        _B("bounds", es_generic(3, _d), H=6, chunk=64),
        _B("bounds", es_generic(3, _d), H=64, chunk=64),
        _B("ragged", es_main(3, 512, _d, bulk=True, stats=False), H=8, chunk=64),
    ]

TABLE = SPMM + SPMM_F16 + SDDMM + MHSPMM + SCATTER_MAX + EDGE_SOFTMAX + GAT_FWD + GAT_ATTN_BWD

# Compiled instantiations no public entry point above reaches: launched only by the fused layers' hub-row pre-pass.
EXEMPT = {
    "cogdl_b200::scatter_max_stream_kernel<NV=1,U=4,values_only>":
        "smax_hub_rows_only (fused SAGE max layer): tests/test_gpu_fused_sage.py",
}

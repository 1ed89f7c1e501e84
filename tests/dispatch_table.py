"""One row per dispatch branch of the gather kernels in spmm.cu, sddmm.cu, mhspmm.cu and scatter_max.cu, and of the
edge softmax and GAT attention kernels in edge_softmax.cu.

Each row names the inputs that select a kernel instantiation (op, graph, width, alignment, plan form, weights,
perm, dropout, source form) and the exact cogdl_b200_last_kernel() string the call must record.  The GPU test
(test_gpu_dispatch.py) runs every row and checks the output against a reference; the CPU test
(test_cpu_kernel_inventory.py) checks that the rows cover every kernel compiled into those five objects, and
that every kernel named here is compiled.  Plain Python, no torch: the CPU test imports it without a GPU.

The message operators and fused layers (MESSAGE_TABLE) and the sparse x sparse product's tier edges (SPGEMM_TABLE)
follow, each with its own GPU test.
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


# ================================================================== message operators and the fused layers
# GENConv's softmax aggregation (softmax_aggr.cu), DisenGCN's routing (disen_routing.cu), CompGCN's composition
# aggregation (comp_aggr.cu) and the fused GCN / SAGE layers (fused_gcn.cu).  Run by test_gpu_dispatch_message.py.
@dataclass(frozen=True)
class MessageCase:
    op: str                 # sa_fwd | sa_bwd | disen_fwd | disen_bwd | comp | fused_gcn | fused_sage_sum | fused_sage_max
    graph: str              # "bounds": boundary_csr(chunk); "bounds_t": boundary_csc(chunk), whose transpose (walked by
                            # the backwards) has the boundary degrees; else a name in tests/graphs.py CASES
    F: int                  # features (fused layers: Fout; their input width is 128)
    kernel: str             # exact cogdl_b200_last_kernel() after the call
    plan: str = "chunks"    # none | chunks (hub chunks, no segments) | default (chunks + segments)
    chunk: int = 64         # hub chunk edges of the plan (of the transpose's too)
    aligned: bool = True    # False: the feature inputs are views one element past an aligned allocation
    partials_offset: int = 0  # bytes the plan's partial scratch starts past a 16-byte boundary
    # GENConv
    beta: float = 1.0
    edge_term: bool = False
    want_q: bool = False
    want_edge_grad: bool = True
    # DisenGCN
    K: int = 1              # channels (d = F / K)
    tau: float = 1.0
    want_saved: bool = True
    zero_norm: bool = False  # one node's channel of c is NaN, as normalising a zero-norm channel gives
    # CompGCN
    comp: str = "mult"      # mult | sub | copy
    T: int = 1              # edge types (rows of the relation table)
    # fused layers
    relu: bool = False
    bias: bool = False
    row_scale: bool = False
    weighted: bool = True

    @property
    def id(self):
        s = f"{self.op}-{self.graph}-F{self.F}-{self.plan}-C{self.chunk}"
        if self.op.startswith("sa_"):
            s += f"-beta{self.beta:g}" + ("-A" if self.edge_term else "") + ("-Q" if self.want_q else "")
            s += "" if self.want_edge_grad else "-no_dA"
        if self.op.startswith("disen"):
            s += f"-K{self.K}-tau{self.tau:g}" + ("" if self.want_saved else "-unsaved") + ("-nan" if self.zero_norm else "")
        if self.op == "comp":
            s += f"-{self.comp}-T{self.T}"
        if self.op.startswith("fused"):
            s += ("-relu" if self.relu else "") + ("-bias" if self.bias else "") + ("-rs" if self.row_scale else "")
            s += "-w" if self.weighted else "-u"
        if not self.aligned:
            s += "-misaligned"
        if self.partials_offset:
            s += f"-partials+{self.partials_offset}"
        return s

    @property
    def vec(self):
        """Vector width W of the kernel the row selects: 4 (float4) or 1."""
        return 4 if "<float4" in self.kernel.split(" + ")[-1] else 1


def sa_fwd_k(vec, edge_term, q):
    return (f"cogdl_b200::softmax_aggr_fwd_kernel<{vec},{'edge_term' if edge_term else 'no_edge_term'},"
            f"{'Q' if q else 'no_Q'}>")


def sa_bwd_k(vec, edge_term):
    return f"cogdl_b200::softmax_aggr_bwd_kernel<{vec},{'edge_term' if edge_term else 'no_edge_term'}>"


def dr_fwd_k(vec, group):
    return f"cogdl_b200::disen_route_fwd_kernel<{vec},GROUP={group}>"


def dr_bwd_k(vec, group):
    return (f"cogdl_b200::disen_route_bwd_row_kernel<{vec},GROUP={group}> + "
            f"cogdl_b200::disen_route_bwd_col_kernel<{vec},GROUP={group}>")


COMP_WHAT = {"mult": "comp_mult", "sub": "comp_sub", "copy": "weighted"}


def comp_k(vec, nv, comp):
    return stream_k(vec, nv, COMP_WHAT[comp], "SRC_ONE", 4 if nv == 1 else 2, 1, True)


FUSED_AGG = {"fused_gcn": "gcn", "fused_sage_sum": "sage-sum", "fused_sage_max": "sage-max"}


def fused_k(op, npad, hub, weighted=True, row_scale=False):
    """The fused layer; with hub rows after its pre-pass (the SpMM's hub chunks, or scatter_max's without argmax)."""
    s = (f"cogdl_b200::fg::fused_layer_kernel<{FUSED_AGG[op]}{'+row_scale' if row_scale else ''}, 2 groups x tile "
         f"64x{npad}, K=128, bf16x3 split, wgmma m64n32k16>")
    if not hub:
        return s
    pre = ("cogdl_b200::scatter_max_stream_kernel<NV=1,U=4,values_only>" if op == "fused_sage_max"
           else stream_k("float4", 1, _w(weighted), "SRC_ONE", 4, 5, False))
    return f"{pre} + {s}"


# ------------------------------------------------------------------ GENConv: cogdl_b200_softmax_aggr_fwd_f32 / _bwd_f32
# float4 iff F % 4 == 0 and every operand (the partial scratch too) is 16-byte aligned; a warp per row or hub chunk,
# 32 vectors per pass.  Betas 0, 0.5, 4 and 20 spread over the rows.
_SA = lambda F, kernel, beta, **kw: MessageCase("sa_fwd", "bounds", F, kernel, beta=beta, **kw)  # noqa: E731
SOFTMAX_AGGR = [
    _SA(64, sa_fwd_k("float4", False, False), 0.5),
    _SA(32, sa_fwd_k("float4", False, True), 4.0, want_q=True),
    _SA(128, sa_fwd_k("float4", True, False), 20.0, edge_term=True),          # 32 vectors: one full pass
    _SA(16, sa_fwd_k("float4", True, True), 0.0, edge_term=True, want_q=True),
    _SA(7, sa_fwd_k("float", False, False), 4.0),
    _SA(1, sa_fwd_k("float", False, True), 20.0, want_q=True),
    _SA(13, sa_fwd_k("float", True, False), 0.5, edge_term=True),
    _SA(31, sa_fwd_k("float", True, True), 20.0, edge_term=True, want_q=True),
    # more than 32 vectors per row: the pass loop runs 3 times, the last pass partial
    _SA(264, sa_fwd_k("float4", True, True), 4.0, edge_term=True, want_q=True),
    _SA(70, sa_fwd_k("float", True, True), 0.5, edge_term=True, want_q=True),
    # no plan: every row (the 129 C + 5 hub too) is one warp's
    _SA(128, sa_fwd_k("float4", False, False), 20.0, plan="none"),
    _SA(33, sa_fwd_k("float", False, False), 4.0, plan="none"),
    # a float4 width and aligned operands, but the partial scratch 4 bytes off: the scalar kernel
    _SA(64, sa_fwd_k("float", True, True), 4.0, edge_term=True, want_q=True, partials_offset=4),
]
_SB = lambda F, kernel, beta, **kw: MessageCase("sa_bwd", "bounds_t", F, kernel, beta=beta, **kw)  # noqa: E731
SOFTMAX_AGGR += [
    _SB(64, sa_bwd_k("float4", False), 4.0),
    _SB(128, sa_bwd_k("float4", True), 0.5, edge_term=True),
    _SB(7, sa_bwd_k("float", False), 20.0),
    _SB(33, sa_bwd_k("float", True), 0.0, edge_term=True),                     # two passes
    _SB(32, sa_bwd_k("float4", True), 20.0, edge_term=True, want_edge_grad=False),   # dA == nullptr
]

# ------------------------------------------------------------------ DisenGCN: cogdl_b200_disen_route_fwd_f32 / _bwd_f32
# F = K d; float4 iff d % 4 == 0 and the operands are aligned; GROUP = the row's vectors rounded up to a power of two,
# at most 32 (wider rows loop over 32-vector tiles); L = d / W lanes per channel reduce its dot products.
_DR_SHAPES = [   # (vec, GROUP, K, d, aligned, tau)
    ("float4", 1, 1, 4, True, 1.0),
    ("float4", 2, 2, 4, True, 0.1),
    ("float4", 4, 1, 16, True, 5.0),
    ("float4", 8, 4, 8, True, 1.0),
    ("float4", 16, 2, 32, True, 0.1),
    ("float4", 32, 8, 16, True, 5.0),
    ("float", 1, 1, 1, True, 1.0),
    ("float", 2, 1, 2, True, 0.1),
    ("float", 4, 2, 2, True, 5.0),
    ("float", 8, 8, 1, True, 1.0),
    ("float", 16, 4, 4, False, 0.1),
    ("float", 32, 8, 4, False, 5.0),
]
_DR_EXTRA = [    # GROUP = 32 with idle lanes (K = 3) and with several 32-vector tiles
    ("float4", 32, 3, 32, True, 1.0),
    ("float4", 32, 16, 32, True, 0.1),           # 128 vectors: four tiles
    ("float", 32, 3, 8, False, 1.0),
    ("float", 32, 2, 32, False, 5.0),            # 64 floats: two tiles
]
DISEN = []
for _op, _k in (("disen_fwd", dr_fwd_k), ("disen_bwd", dr_bwd_k)):
    for _vec, _g, _K, _d, _al, _tau in _DR_SHAPES + _DR_EXTRA:
        DISEN.append(MessageCase(_op, "bounds" if _op == "disen_fwd" else "bounds_t", _K * _d, _k(_vec, _g), K=_K,
                                 tau=_tau, aligned=_al))
DISEN += [
    MessageCase("disen_fwd", "bounds", 32, dr_fwd_k("float4", 8), K=4, tau=1.0, want_saved=False),
    MessageCase("disen_fwd", "bounds", 64, dr_fwd_k("float4", 16), K=2, tau=0.1, zero_norm=True),
]

# ------------------------------------------------------------------ CompGCN: cogdl_b200_comp_aggr_f32
# The row-stream kernel with a second gathered row: one vector per lane up to 32 vectors, two beyond (rows wider than
# 64 vectors loop over column tiles).  "copy" is the weighted SpMM form at the composition's U and MINB.
COMP = []
for _comp in ("mult", "sub", "copy"):
    for _vec, (_f1, _f2, _f3) in (("float4", (64, 200, 264)), ("float", (7, 50, 133))):
        COMP += [
            MessageCase("comp", "bounds", _f1, comp_k(_vec, 1, _comp), plan="default", comp=_comp, T=1),
            MessageCase("comp", "bounds", _f2, comp_k(_vec, 2, _comp), plan="default", comp=_comp, T=300),
            MessageCase("comp", "bounds", _f3, comp_k(_vec, 2, _comp), plan="default", comp=_comp, T=1),
        ]

# ------------------------------------------------------------------ fused layers: cogdl_b200_gcn_fused_f32 / _sage_fused_f32
# 400 rows: 7 tiles of 64, the last one of 16 rows.  Fout <= 64 fills a 64-row W^T, Fout > 64 a 128-row one.  Chunk 64
# makes hub rows (the pre-pass runs first); chunk 4096 leaves none.
_FUSED_SHAPES = {   # op -> rows (Npad, hub, Fout, relu, bias, row_scale, weighted)
    "fused_gcn": [(64, True, 33, True, True, False, True), (64, False, 1, False, False, False, False),
                  (128, True, 128, False, True, False, True), (128, False, 65, True, False, False, False)],
    "fused_sage_sum": [(64, True, 64, False, True, True, True), (64, False, 33, True, False, False, True),
                       (128, True, 65, True, True, False, False), (128, False, 128, False, False, True, True)],
    "fused_sage_max": [(64, True, 1, True, True, False, False), (64, False, 64, False, True, False, False),
                       (128, True, 128, True, False, False, False), (128, False, 65, False, False, False, False)],
}
FUSED = [MessageCase(_op, "hub", _fo, fused_k(_op, _np, _hub, _wt, _rs), plan="default", chunk=64 if _hub else 4096,
                     relu=_relu, bias=_b, row_scale=_rs, weighted=_wt)
         for _op, _rows in _FUSED_SHAPES.items() for _np, _hub, _fo, _relu, _b, _rs, _wt in _rows]

MESSAGE_TABLE = SOFTMAX_AGGR + DISEN + COMP + FUSED

# Compiled instantiations no row above reaches (none: the fused layers record their hub pre-pass).
EXEMPT = {}


# ================================================================== sparse x sparse product (spgemm.cu)
# cogdl_b200_spgemm_count / _fill_f32 put every output row into a tier by bound = min(sum_{k in A_i} deg_B(k), n):
# nothing to do (0), a warp with a 512-slot hash table (<= 256), a block with an 8192-slot table (<= 4096), or a
# block with a bitmap of the n columns in one of 132 global slots.  Every tier kernel and the classifier launch on every
# call and the call records one name per phase, so a row names the edges of the tiers its product reaches
# (tests/spgemm_oracle.py edges(), which test_cpu_kernel_inventory.py checks against the row's builder), and
# cogdl_b200_spgemm_bwd_f32's one-warp-per-entry reductions.  Run by test_gpu_dispatch_spgemm.py.
SPG_COUNT = "cogdl_b200::spg_count<warp=256,block=4096,bitmap>"
SPG_FILL = "cogdl_b200::spg_fill<warp=256,block=4096,bitmap>"
SPG_DA = "cogdl_b200::spg_dA_kernel"
SPG_DB = "cogdl_b200::spg_dB_kernel"
SPG_DA_DB = f"{SPG_DA} + {SPG_DB}"


@dataclass(frozen=True)
class SpgemmCase:
    name: str               # the product: tests/graphs.py spgemm_case(name)
    edges: tuple            # the (tier, edge) pairs it is built for

    @property
    def id(self):
        return f"spgemm-{self.name}"

    # what every row's calls record: count, fill, and the backward for dA, dB and both
    kernels = (SPG_COUNT, SPG_FILL, SPG_DA, SPG_DB, SPG_DA_DB)


def _spg(name, *edges):
    return SpgemmCase(name, tuple(edges))


SPGEMM_TABLE = [
    _spg("empty-rows", ("empty", "A row without entries"), ("empty", "A row meeting only empty B rows")),
    _spg("m0", ("shape", "m = 0")),
    _spg("k0", ("shape", "k = 0")),
    _spg("n0", ("shape", "n = 0")),
    _spg("A-empty", ("shape", "A without entries")),
    _spg("B-empty", ("shape", "B without entries")),
    _spg("rect", ("shape", "m, k, n distinct, every tier")),
    _spg("warp-counts", ("warp", "1 columns"), ("warp", "255 columns"), ("warp", "256 columns")),
    _spg("warp-bound256-c1", ("warp", "bound 256, 1 columns")),
    _spg("warp-hash-wrap", ("warp", "hash wrap-around")),
    _spg("warp-n-capped", ("warp", "n <= 256, full row")),
    _spg("block-counts", ("block", "257 columns"), ("block", "4095 columns"), ("block", "4096 columns")),
    _spg("block-bound300-c2", ("block", "bound 300, 2 columns")),
    _spg("block-hash-wrap", ("block", "hash wrap-around")),
    _spg("block-n-capped", ("block", "n = 4096, full row")),
    _spg("bitmap-counts", ("bitmap", "4097 columns")),
    _spg("bitmap-bound5000-c3", ("bitmap", "bound 5000, 3 columns")),
    _spg("bitmap-full", ("bitmap", "all n columns")),
    _spg("bitmap-n32w+1", ("bitmap", "n = 32w + 1")),
    _spg("bitmap-n8192", ("bitmap", "n = 8192")),
    _spg("bitmap-n8193", ("bitmap", "n = 8193")),
    _spg("grid-loops", ("warp", "grid loop"), ("block", "grid loop"), ("bitmap", "grid loop")),
    _spg("cancel", ("values", "exact cancellation")),
    _spg("subnormal", ("values", "subnormal")),
    _spg("negzero", ("values", "-0.0 factors")),
    *[_spg(f"bwd-{d}", ("dA", f"{d} terms"), ("dB", f"{d} terms")) for d in (1, 31, 32, 33, 65, 2000)],
    _spg("bwd-duplicates", ("dA", "duplicate entries"), ("dB", "duplicate entries")),
]

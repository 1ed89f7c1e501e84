"""Every gather kernel compiled into spmm.o, sddmm.o, mhspmm.o and scatter_max.o, every edge-softmax / GAT attention
kernel compiled into edge_softmax.o, every message-operator kernel of softmax_aggr.o (GENConv), disen_routing.o
(DisenGCN) and comp_aggr.o (CompGCN), every fused layer of fused_gcn.o and every tier kernel of the sparse x sparse
product in spgemm.o has a row in the dispatch table (tests/dispatch_table.py) that the GPU suite runs and checks, and
every kernel the table names is compiled.  A new dispatch branch without a test case fails here, on a machine without
a GPU.

Objects left out on purpose, none of which picks a kernel by size and all of which are checked bit for bit: actnn.o
(against the numpy restatement, test_gpu_actnn.py), sampler.o (against the oracle, test_gpu_sampler.py) and
csr_tools.o (its integer and permutation kernels checked exactly by the structure tests; its one float reduction,
cogdl_b200_edge_colsum_f32, per element against fp64 with its column-degree bound by every row of
test_gpu_simple_hgn.py::test_row_against_fp64, as d h_r, hub columns on the boundary degrees and no plan included).

The kernel entry points are read from the objects with cuobjdump and demangled with cu++filt; each instantiation
is mapped to the string its launcher records for cogdl_b200_last_kernel()."""
import os
import re
import shutil
import subprocess

import pytest

from tests import graphs
from tests import spgemm_oracle as so
from tests.dispatch_table import ES_OPS, EXEMPT, MESSAGE_TABLE, SPG_COUNT, SPG_FILL, SPGEMM_TABLE, TABLE

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OBJ_DIR = os.path.join(ROOT, "cogdl_b200", "csrc", "build")
OBJECTS = ("spmm", "sddmm", "mhspmm", "scatter_max", "edge_softmax", "softmax_aggr", "disen_routing", "comp_aggr",
           "fused_gcn", "spgemm")
ROWS = TABLE + MESSAGE_TABLE


def table_names():
    """The recorded name of every row; a sparse x sparse row's calls record several."""
    return [c.kernel for c in ROWS] + [k for c in SPGEMM_TABLE for k in c.kernels]


def _tool(name):
    for d in (os.environ.get("CUDA_HOME"), "/usr/local/cuda"):
        if d and os.access(os.path.join(d, "bin", name), os.X_OK):
            return os.path.join(d, "bin", name)
    return shutil.which(name)


def compiled_kernels(objects=OBJECTS):
    """Demangled kernel entry points (global functions) of the objects."""
    cuobjdump, cufilt = _tool("cuobjdump"), _tool("cu++filt")
    if not cuobjdump or not cufilt:
        pytest.skip("cuobjdump / cu++filt from the CUDA toolkit are not available")
    paths = [os.path.join(OBJ_DIR, f"{o}.o") for o in objects]
    missing = [p for p in paths if not os.path.exists(p)]
    if missing:
        pytest.skip(f"library objects not built (run build()): {', '.join(missing)}")
    mangled = []
    for p in paths:
        out = subprocess.run([cuobjdump, "-symbols", p], capture_output=True, text=True, check=True).stdout
        mangled += [ln.split()[-1] for ln in out.splitlines() if "STT_FUNC" in ln and "STB_GLOBAL" in ln]
    assert mangled, "no kernel symbols found"
    out = subprocess.run([cufilt], input="\n".join(mangled) + "\n", capture_output=True, text=True, check=True).stdout
    return [ln.strip() for ln in out.splitlines() if ln.strip()]


def assert_table_covers(obj, note_of, table_kernels, table_file):
    """Every kernel compiled into <obj>.o has a row in table_file, and every kernel the table names is compiled.
    note_of maps a demangled symbol to the name cogdl_b200_last_kernel() records, table_kernels is the set of names the
    table's rows record.  Returns {recorded name: symbol} of the object."""
    compiled = {note_of(s): s for s in compiled_kernels((obj,))}
    assert compiled, f"{obj}.o holds no kernels"
    untested = sorted(set(compiled) - table_kernels)
    assert not untested, f"compiled kernels without a row in {table_file}:\n" + "\n".join(
        f"  {n}   ({compiled[n]})" for n in untested)
    unknown = sorted(table_kernels - set(compiled))
    assert not unknown, "table rows name kernels that are not compiled:\n" + "\n".join(f"  {n}" for n in unknown)
    return compiled


_SRC = {0: "SRC_ONE", 1: "SRC_TWO", 2: "SRC_PEERS"}
# the SpMM row and row-stream kernels are recorded as spmm<tag>_kernel / stream<tag>_kernel, by their epilogue argument
_EPI_TAG = {0: "", 1: "_residual", 2: "_labelprop", 3: "_dcoef", 4: "_accum"}


def _args(sig):
    """Template arguments of a demangled name: 'float4', '(int)32', '(bool)1' -> 'float4', 32, True."""
    inner = sig[sig.index("<") + 1: sig.rindex(">")]
    out = []
    for a in inner.split(","):
        a = a.strip()
        m = re.fullmatch(r"\((int|bool)\)(-?\d+)", a)
        out.append(a if m is None else (int(m.group(2)) if m.group(1) == "int" else m.group(2) != "0"))
    return out


def note_of(sym):
    """The cogdl_b200_last_kernel() string of one demangled instantiation (canonical form, see canonical())."""
    if re.match(r"void cub::\w+::(DeviceScan\w*Kernel|EmptyKernel)<", sym):
        return SPG_COUNT      # spgemm.o: the count phase's scan of the row counts (cub compiles EmptyKernel beside it)
    m = re.fullmatch(r"(?:void )?cogdl_b200::((?:fg::)?\w+)(<.*>)?\(.*\)", sym)
    assert m, f"unexpected symbol {sym!r}"
    name = m.group(1)
    a = _args(m.group(2)) if m.group(2) else []
    w = lambda b: "weighted" if b else "unweighted"  # noqa: E731
    if name == "spmm_kernel":
        vec, group, nv, has_val, epi = a
        return f"cogdl_b200::spmm{_EPI_TAG[epi]}_kernel<{vec},GROUP={group},NV={nv},{w(has_val)}>"
    if name == "spmm_half_kernel":
        has_val, vec = a
        return f"cogdl_b200::spmm_half_kernel<{w(has_val)},{'vec' if vec else 'scalar'}>"
    if name == "stream_kernel":
        vec, nv, mode, perm, src, u, minb, prefetch, panel, drop, epi = a
        what = {0: "unweighted", 1: "weighted", 2: "multihead", 3: "comp_mult", 4: "comp_sub"}[mode]
        if mode == 2:
            what += ("+perm" if perm else "") + ("+drop" if drop else "")
        s = (f"cogdl_b200::stream{_EPI_TAG[epi]}_kernel<{vec},NV={nv},{what},{_SRC[src]},U={u},MINB={minb}"
             f"{',prefetch' if prefetch else ''}>")
        return s + (",panels" if panel else "")
    if name == "sddmm_kernel":
        vec, group, sub, nv = a
        return f"cogdl_b200::sddmm_kernel<{vec},GROUP={group},SUB={sub},NV={nv}>"
    if name == "sddmm_stream_kernel":
        nv, u = a
        return f"cogdl_b200::sddmm_stream_kernel<NV={nv},U={u}>"
    if name == "mhspmm_kernel":
        vec, group, perm, drop = a
        return f"cogdl_b200::mhspmm_kernel<{vec},GROUP={group},{'perm' if perm else 'no_perm'}{',drop' if drop else ''}>"
    if name == "scatter_max_fwd_kernel":
        vec, group, nv = a
        return f"cogdl_b200::scatter_max_fwd_kernel<{vec},GROUP={group},NV={nv}>"
    if name == "scatter_max_stream_kernel":
        nv, u, argmax = a
        return f"cogdl_b200::scatter_max_stream_kernel<NV={nv},U={u}{'' if argmax else ',values_only'}>"
    if name == "scatter_max_bwd_kernel":
        return "cogdl_b200::scatter_max_bwd_kernel"
    # edge softmax: TYPED kernels (Simple-HGN) are recorded as hgn_*_kernel, without the es_ names' WARPS and their
    # statistics kernel's DROP
    if name == "es_stats_kernel":
        mode, drop, typed = a
        return f"cogdl_b200::{'hgn' if typed else 'es'}_stats_kernel<MODE={mode}{',DROP' * (drop and not typed)}>"
    if name in ("es_main_kernel", "es_warp_kernel", "es_generic_kernel"):
        mode, drop, typed, mix = [a[0]] + a[-3:]
        cap = f",CAP={a[1]}{'' if typed else ',WARPS=8'}" if name == "es_main_kernel" else ""
        return (f"cogdl_b200::{name.replace('es_', 'hgn_', 1) if typed else name}<MODE={mode}{cap}"
                f"{',DROP' if drop else ''}{',MIX' if mix else ''}>")
    if name == "softmax_aggr_fwd_kernel":
        w_, has_a, want_q = a
        return (f"cogdl_b200::softmax_aggr_fwd_kernel<{'float4' if w_ == 4 else 'float'},"
                f"{'edge_term' if has_a else 'no_edge_term'},{'Q' if want_q else 'no_Q'}>")
    if name == "softmax_aggr_bwd_kernel":
        w_, has_a = a
        return f"cogdl_b200::softmax_aggr_bwd_kernel<{'float4' if w_ == 4 else 'float'},{'edge_term' if has_a else 'no_edge_term'}>"
    if name in ("disen_route_fwd_kernel", "disen_route_bwd_row_kernel", "disen_route_bwd_col_kernel"):
        w_, group = a
        return f"cogdl_b200::{name}<{'float4' if w_ == 4 else 'float'},GROUP={group}>"
    if name == "fg::fused_layer_kernel":
        agg, epi = a
        what = {(0, 0): "gcn", (0, 1): "sage-sum", (1, 1): "sage-max"}[(agg, epi)]
        return f"cogdl_b200::fg::fused_layer_kernel<{what}, 2 groups x tile 64xN, K=128, bf16x3 split, wgmma m64n32k16>"
    if name in ("spg_classify_kernel", "spg_warp_kernel", "spg_block_kernel", "spg_large_kernel"):
        return SPG_FILL if a == [True] else SPG_COUNT     # the classifier runs in both phases, first in the count
    if name in ("spg_dA_kernel", "spg_dB_kernel"):
        return f"cogdl_b200::{name}"
    raise AssertionError(f"no last_kernel() name is known for {sym!r}: add it to note_of() and a row to the table")


def canonical(note):
    """The instantiations a recorded name lists, without their launch-shape suffixes.  A note of several launches
    ('a + b': the edge-softmax statistics and main kernels, the GAT attention and aggregation, the DisenGCN row and
    column kernels, a fused layer's hub pre-pass and the layer) is split; the panel count becomes ',panels' (the
    instantiation is the same for every count), a fused layer's W^T rows '64xN' and its '+row_scale' go (one
    instantiation serves every Fout and both forms of the sum), as do ' block=N' and the staging note
    ' cp.async.bulk tiles'."""
    out = []
    for part in note.split(" + "):
        part = re.sub(r" block=\d+$", "", part)
        part = re.sub(r"(fused_layer_kernel<[\w-]+)\+row_scale,", r"\1,", part)
        part = re.sub(r" tile 64x\d+,", " tile 64xN,", part)
        part = re.sub(r" cp\.async\.bulk tiles$", "", part)
        out.append(re.sub(r",panels=\d+", ",panels", part))
    return out


def test_note_of_maps_known_symbols():
    assert note_of("void cogdl_b200::spmm_kernel<float, (int)32, (int)4, (bool)1, (int)0>(cogdl_b200::SpmmParams)") == \
        "cogdl_b200::spmm_kernel<float,GROUP=32,NV=4,weighted>"
    assert note_of("void cogdl_b200::stream_kernel<float2, (int)1, (int)0, (bool)0, (int)0, (int)8, (int)5, (bool)1, "
                   "(bool)1, (bool)0, (int)0>(cogdl_b200::StreamParams)") == \
        "cogdl_b200::stream_kernel<float2,NV=1,unweighted,SRC_ONE,U=8,MINB=5,prefetch>,panels"
    assert canonical("cogdl_b200::stream_kernel<float2,NV=1,unweighted,SRC_ONE,U=8,MINB=5,prefetch>,panels=4 block=128") \
        == ["cogdl_b200::stream_kernel<float2,NV=1,unweighted,SRC_ONE,U=8,MINB=5,prefetch>,panels"]
    assert note_of("void cogdl_b200::es_main_kernel<(int)3, (int)512, (bool)1, (bool)0, (bool)0>(cogdl_b200::EsParams)") \
        == "cogdl_b200::es_main_kernel<MODE=3,CAP=512,WARPS=8,DROP>"
    assert note_of("void cogdl_b200::es_stats_kernel<(int)2, (bool)0, (bool)0>(cogdl_b200::EsParams)") == \
        "cogdl_b200::es_stats_kernel<MODE=2>"
    assert note_of("void cogdl_b200::es_stats_kernel<(int)3, (bool)1, (bool)0>(cogdl_b200::EsParams)") == \
        "cogdl_b200::es_stats_kernel<MODE=3,DROP>"
    assert canonical("cogdl_b200::es_stats_kernel<MODE=0> + cogdl_b200::es_main_kernel<MODE=0,CAP=512,WARPS=8> "
                     "cp.async.bulk tiles") == ["cogdl_b200::es_stats_kernel<MODE=0>",
                                                "cogdl_b200::es_main_kernel<MODE=0,CAP=512,WARPS=8>"]
    assert note_of("void cogdl_b200::fg::fused_layer_kernel<(int)0, (int)1>(cogdl_b200::fg::Params)") == \
        "cogdl_b200::fg::fused_layer_kernel<sage-sum, 2 groups x tile 64xN, K=128, bf16x3 split, wgmma m64n32k16>"
    assert canonical("cogdl_b200::stream_kernel<float4,NV=1,weighted,SRC_ONE,U=4,MINB=5> block=128 + "
                     "cogdl_b200::fg::fused_layer_kernel<sage-sum+row_scale, 2 groups x tile 64x128, K=128, bf16x3 split, "
                     "wgmma m64n32k16>") == [
        "cogdl_b200::stream_kernel<float4,NV=1,weighted,SRC_ONE,U=4,MINB=5>",
        "cogdl_b200::fg::fused_layer_kernel<sage-sum, 2 groups x tile 64xN, K=128, bf16x3 split, wgmma m64n32k16>"]
    assert note_of("void cogdl_b200::stream_kernel<float, (int)2, (int)4, (bool)0, (int)0, (int)2, (int)1, (bool)1, "
                   "(bool)0, (bool)0, (int)0>(cogdl_b200::StreamParams)") == \
        "cogdl_b200::stream_kernel<float,NV=2,comp_sub,SRC_ONE,U=2,MINB=1,prefetch>"
    assert note_of("void cogdl_b200::softmax_aggr_fwd_kernel<(int)4, (bool)1, (bool)0>(cogdl_b200::SaFwdParams)") == \
        "cogdl_b200::softmax_aggr_fwd_kernel<float4,edge_term,no_Q>"
    assert note_of("void cogdl_b200::disen_route_bwd_col_kernel<(int)1, (int)16>(cogdl_b200::DrColBwdParams)") == \
        "cogdl_b200::disen_route_bwd_col_kernel<float,GROUP=16>"
    assert note_of("cogdl_b200::spg_classify_kernel(cogdl_b200::SpgParams, bool)") == SPG_COUNT
    assert note_of("void cogdl_b200::spg_block_kernel<(bool)0>(cogdl_b200::SpgParams)") == SPG_COUNT
    assert note_of("void cogdl_b200::spg_large_kernel<(bool)1>(cogdl_b200::SpgParams)") == SPG_FILL
    assert note_of("cogdl_b200::spg_dB_kernel(cogdl_b200::SpgBwdParams)") == "cogdl_b200::spg_dB_kernel"
    assert canonical("cogdl_b200::spg_dA_kernel + cogdl_b200::spg_dB_kernel") == ["cogdl_b200::spg_dA_kernel",
                                                                                  "cogdl_b200::spg_dB_kernel"]


def test_dispatch_table_covers_every_compiled_kernel():
    compiled = {}
    for sym in compiled_kernels():
        compiled.setdefault(note_of(sym), sym)
    table = {k for name in table_names() for k in canonical(name)}
    untested = sorted(set(compiled) - table - set(EXEMPT))
    assert not untested, "compiled kernels without a row in tests/dispatch_table.py:\n" + "\n".join(
        f"  {n}   ({compiled[n]})" for n in untested)
    unknown = sorted(table - set(compiled))
    assert not unknown, "table rows name kernels that are not compiled:\n" + "\n".join(f"  {n}" for n in unknown)
    stale = sorted(set(EXEMPT) - set(compiled))
    assert not stale, f"exemptions for kernels that are not compiled: {stale}"


def test_table_rows_are_distinct():
    ids = [c.id for c in ROWS + SPGEMM_TABLE]
    dup = sorted({i for i in ids if ids.count(i) > 1})
    assert not dup, f"duplicate table rows: {dup}"


def test_recorded_names_fit_the_note_buffer():
    """cogdl_b200_last_kernel() is kept in a 256-byte buffer: the longest name the table expects (a GAT forward:
    statistics + main kernel of the attention, then the row-stream aggregation; a fused layer after its hub pre-pass)
    must fit whole."""
    longest = max(table_names(), key=lambda k: len(k.encode()))
    assert len(longest.encode()) < 256, longest


_ES_OP = {0: "edge_softmax", 1: "edge_softmax_bwd", 2: "gat_fwd", 3: "gat_attn_bwd"}


def es_form(c):
    """The launch form of an edge-softmax row: op, dropout, the attention part of the recorded name (statistics kernel
    or not, cp.async.bulk or coalesced staging), and what else decides how the kernel runs: for the main kernel the
    graph (boundary degrees or a random power-law graph), one head or several, and whether a chunk fills the tile
    exactly; how a warp-kernel row got there (no plan, or no tile holds a chunk); a generic row's head count."""
    att = c.kernel.split(" + cogdl_b200::stream_kernel")[0].split(" + cogdl_b200::mhspmm_kernel")[0]
    if "es_main_kernel" in att:
        cap = int(re.search(r"CAP=(\d+)", att).group(1))
        detail = (c.graph == "bounds", c.H == 1, c.chunk * c.H == cap)
    elif "es_warp_kernel" in att:
        detail = c.plan
    else:
        detail = c.H
    return (c.op, c.drop, att, detail)


def required_es_forms():
    """Every launch form es_launch can take with the compiled instantiations, on the boundary-degree graph unless
    said otherwise: the main kernel after the statistics kernel at every tile, with several heads filling it exactly
    and with bulk staging where the mode allows it; at the 2048-float tile also one head (coalesced staging: rows are
    4 bytes apart); at the 512-float tile coalesced staging of a misaligned operand, no hub rows (a random graph),
    and for the edge softmax the random graph with a 700-edge hub with the tile filled and half filled; the warp
    kernel without a plan and when no tile holds a chunk; the generic kernel at 3 and 6 heads and at 64 (a power of
    two above 32)."""
    forms = set()
    for sym in compiled_kernels():
        m = re.fullmatch(r"(?:void )?cogdl_b200::(es_\w+)<(.*)>\(.*\)", sym)
        if not m:
            continue
        name, a = m.group(1), _args("<" + m.group(2) + ">")
        mode, drop = a[0], a[2 if name == "es_main_kernel" else 1]
        op = _ES_OP[mode]
        dn = ",DROP" if drop else ""
        if name == "es_main_kernel":
            cap = a[1]
            main = note_of(sym)
            st = f"cogdl_b200::es_stats_kernel<MODE={mode}{dn if mode == 3 else ''}> + "
            bulk = " cp.async.bulk tiles" if mode != 2 else ""
            forms.add((op, drop, st + main + bulk, (True, False, True)))
            if cap == 2048:
                forms.add((op, drop, st + main, (True, True, True)))
            if cap == 512:
                forms.add((op, drop, main + bulk, (False, False, True)))
                if mode != 2:
                    forms.add((op, drop, st + main, (True, False, True)))
                if mode in (0, 1):
                    forms.add((op, drop, st + main + bulk, (False, False, True)))
                    forms.add((op, drop, st + main + bulk, (False, False, False)))
        elif name == "es_warp_kernel":
            for route in ("none", "default"):
                forms.add((op, drop, note_of(sym), route))
        elif name == "es_generic_kernel":
            for H in (3, 6, 64):
                forms.add((op, drop, note_of(sym), H))
    return forms


def test_edge_softmax_and_gat_rows_cover_every_launch_form():
    """Every launch form has a row and every row is the only one of its form, so removing any edge-softmax row fails
    here."""
    rows = [es_form(c) for c in TABLE if c.op in ES_OPS]
    required = required_es_forms()
    missing = sorted(required - set(rows), key=str)
    assert not missing, "edge-softmax launch forms without a row in tests/dispatch_table.py:\n" + "\n".join(
        f"  {f}" for f in missing)
    extra = sorted(set(rows) - required, key=str)
    assert not extra, f"rows in launch forms the compiled kernels do not have: {extra}"
    dup = sorted({f for f in rows if rows.count(f) > 1}, key=str)
    assert not dup, f"several rows of one launch form: {dup}"


def message_form(c):
    """The launch form of a message-operator or fused-layer row: op, the instantiations it records, and what else
    decides how they run.  GENConv forward: no plan, a partial scratch off alignment, more than 32 vectors a row (several
    passes), or hub chunks; backward: with or without d edge_term.  DisenGCN: without saved state, a NaN channel, several
    32-vector tiles, idle lanes of a 32-lane group, or none of these.  CompGCN: the row's vectors (<= 32, <= 64, more:
    column tiles) and whether there is one edge type.  Fused layers: W^T rows (Npad), hub rows, row scale."""
    k = tuple(canonical(c.kernel))
    fv = c.F // c.vec
    if c.op == "sa_fwd":
        tag = "none" if c.plan == "none" else "partials+4" if c.partials_offset else "tiles" if fv > 32 else "chunks"
    elif c.op == "sa_bwd":
        tag = "chunks" if c.want_edge_grad else "no_dA"
    elif c.op in ("disen_fwd", "disen_bwd"):
        tag = ("unsaved" if not c.want_saved else "nan" if c.zero_norm else "tiles" if fv > 32 else
               "idle" if 16 < fv < 32 else "")
    elif c.op == "comp":
        tag = ("one" if fv <= 32 else "two" if fv <= 64 else "tiles", c.T == 1)
    else:    # the pre-pass of a hub row: test_fused_rows_name_their_pre_pass
        k, tag = k[-1:], (64 if c.F <= 64 else 128, " + " in c.kernel, c.row_scale)
    return (c.op, k, tag)


_FUSED_OP = {"gcn": "fused_gcn", "sage-sum": "fused_sage_sum", "sage-max": "fused_sage_max"}


def required_message_forms():
    """Every launch form the compiled message kernels and fused layers can take.  GENConv forward: every instantiation
    with hub chunks; per vector width a row without a plan, a row of several passes, and (scalar only) a row sent to
    the scalar kernel by a partial scratch 4 bytes off alignment.  Backward: every instantiation with hub chunks on the
    transpose, and the float4 edge-term kernel without d edge_term.  DisenGCN: every (kernel, W, GROUP), forward and
    backward (the backward records its row and column kernels); at GROUP 32 and both widths, idle lanes and several
    tiles; a forward without saved state and one with a NaN channel.  CompGCN: every instantiation, NV = 2 both within
    64 vectors and over several column tiles, each width and op with one edge type and with 300.  Fused layers: each
    at Npad 64 and 128, with and without hub rows; the sum of the SAGE layer with and without a row scale."""
    forms = set()
    comp = {note_of(s) for s in compiled_kernels(("comp_aggr",))}
    for sym in compiled_kernels(("softmax_aggr", "disen_routing", "comp_aggr", "fused_gcn")):
        n = note_of(sym)
        if "softmax_aggr_fwd_kernel" in n:
            forms.add(("sa_fwd", (n,), "chunks"))
            if "no_edge_term,no_Q" in n:
                forms.add(("sa_fwd", (n,), "none"))
            if ",edge_term,Q" in n:
                forms.add(("sa_fwd", (n,), "tiles"))
                if "<float," in n:
                    forms.add(("sa_fwd", (n,), "partials+4"))
        elif "softmax_aggr_bwd_kernel" in n:
            forms.add(("sa_bwd", (n,), "chunks"))
            if n.endswith("<float4,edge_term>"):
                forms.add(("sa_bwd", (n,), "no_dA"))
        elif "disen_route_bwd_col_kernel" in n:
            continue
        elif "disen_route_" in n:
            op = "disen_fwd" if "fwd" in n else "disen_bwd"
            k = (n,) if op == "disen_fwd" else (n, n.replace("bwd_row", "bwd_col"))
            forms.add((op, k, ""))
            if n.endswith("GROUP=32>"):
                forms.update({(op, k, "idle"), (op, k, "tiles")})
            if op == "disen_fwd" and n.endswith("<float4,GROUP=8>"):
                forms.add((op, k, "unsaved"))
            if op == "disen_fwd" and n.endswith("<float4,GROUP=16>"):
                forms.add((op, k, "nan"))
        elif n in comp:
            if ",NV=1," in n:
                forms.add(("comp", (n,), ("one", True)))
            else:
                forms.update({("comp", (n,), ("two", False)), ("comp", (n,), ("tiles", True))})
        elif "fused_layer_kernel" in n:
            op = _FUSED_OP[re.search(r"<([\w-]+),", n).group(1)]
            for npad in (64, 128):
                for hub in (False, True):
                    rs = op == "fused_sage_sum" and hub == (npad == 64)
                    forms.add((op, (n,), (npad, hub, rs)))
    return forms


def test_message_rows_cover_every_launch_form():
    """Every launch form of the message operators and fused layers has exactly one row, so removing any of those rows
    fails here."""
    rows = [message_form(c) for c in MESSAGE_TABLE]
    required = required_message_forms()
    missing = sorted(required - set(rows), key=str)
    assert not missing, "message launch forms without a row in tests/dispatch_table.py:\n" + "\n".join(
        f"  {f}" for f in missing)
    extra = sorted(set(rows) - required, key=str)
    assert not extra, "rows in launch forms the compiled kernels do not have:\n" + "\n".join(f"  {f}" for f in extra)
    dup = sorted({f for f in rows if rows.count(f) > 1}, key=str)
    assert not dup, f"several rows of one launch form: {dup}"


def test_fused_rows_name_their_pre_pass():
    """A fused row with hub rows names the pre-pass its layer launches (the SpMM's hub chunks, weighted iff the row has
    edge values; scatter_max's without argmax for the max layer), one without names the layer alone."""
    for c in MESSAGE_TABLE:
        if not c.op.startswith("fused"):
            continue
        parts = canonical(c.kernel)
        hub = c.chunk < 1500                      # the 400-row graph's hub has 1500 edges
        assert len(parts) == (2 if hub else 1), c.id
        if hub and c.op == "fused_sage_max":
            assert parts[0] == "cogdl_b200::scatter_max_stream_kernel<NV=1,U=4,values_only>", c.id
        elif hub:
            assert parts[0] == f"cogdl_b200::stream_kernel<float4,NV=1,{'weighted' if c.weighted else 'unweighted'}," \
                               "SRC_ONE,U=4,MINB=5>", c.id


# The edges of each tier of the sparse x sparse product, as tests/spgemm_oracle.py edges() names them.  The classifier
# owns the rows with nothing to do and the degenerate shapes; each fill kernel also owns the values its fmaf chains
# produce, in a row of every tier.
_SPG_TIERS = {"spg_classify_kernel": ("empty", "shape"), "spg_warp_kernel": ("warp",), "spg_block_kernel": ("block",),
              "spg_large_kernel": ("bitmap",), "spg_dA_kernel": ("dA",), "spg_dB_kernel": ("dB",)}
_SPG_EDGES = {
    "empty": ("A row without entries", "A row meeting only empty B rows"),
    "shape": ("m = 0", "k = 0", "n = 0", "A without entries", "B without entries", "m, k, n distinct, every tier"),
    "warp": ("1 columns", "255 columns", "256 columns", "bound 256, 1 columns", "hash wrap-around",
             "n <= 256, full row", "grid loop"),
    "block": ("257 columns", "4095 columns", "4096 columns", "bound 300, 2 columns", "hash wrap-around",
              "n = 4096, full row", "grid loop"),
    "bitmap": ("4097 columns", "bound 5000, 3 columns", "all n columns", "n = 32w + 1", "n = 8192", "n = 8193",
               "grid loop"),
    "values": ("exact cancellation", "subnormal", "-0.0 factors"),
    "dA": tuple(f"{d} terms" for d in so.BWD_TERMS) + ("duplicate entries",),
    "dB": tuple(f"{d} terms" for d in so.BWD_TERMS) + ("duplicate entries",),
}


def required_spgemm_edges():
    """The (tier, edge) pairs of every compiled tier kernel of spgemm.o.  Warp and block tiers: rows of distinct
    count 1 / 255 / 256 and 257 / 4095 / 4096 with distinct count = bound, a bound at or past the cap with 1 or 2
    columns, a full table whose columns all hash into its last slots (probes wrap to slot 0), the bound capped by
    n <= 256 and by n = 4096 with a full row, and more rows than the launch has warps or blocks.  The bitmap: 4097
    columns, bound 5000 with 3 columns, a row of all n columns, n = 32w + 1 with columns 0, 31, 32, 63, 64 and n - 1,
    n = 8192 (256 words) and 8193 (a scan carry), more rows than slots.  The backward: entries of 1, 31, 32, 33, 65
    and 2000 terms and duplicated input entries, for dA and dB."""
    req = set()
    for sym in compiled_kernels(("spgemm",)):
        m = re.fullmatch(r"(?:void )?cogdl_b200::(spg_\w+)(<.*>)?\(.*\)", sym)
        if not m:
            continue                                      # cub's scan
        assert m.group(1) in _SPG_TIERS, f"no edges are known for {sym!r}: add them here and rows to SPGEMM_TABLE"
        tiers = _SPG_TIERS[m.group(1)] + (("values",) if m.group(2) and _args(m.group(2)) == [True] else ())
        req |= {(t, e) for t in tiers for e in _SPG_EDGES[t]}
    return req


def test_spgemm_rows_cover_every_tier_edge():
    """Every tier edge has exactly one row built for it, and each row's product (rebuilt here from its numpy builder)
    reaches the edges it names, so removing any sparse x sparse row, or a builder drifting off its edge, fails here."""
    rows = [e for c in SPGEMM_TABLE for e in c.edges]
    required = required_spgemm_edges()
    missing = sorted(required - set(rows))
    assert not missing, "tier edges without a row in SPGEMM_TABLE:\n" + "\n".join(f"  {e}" for e in missing)
    extra = sorted(set(rows) - required)
    assert not extra, f"rows for edges no compiled kernel has: {extra}"
    dup = sorted({e for e in rows if rows.count(e) > 1})
    assert not dup, f"several rows for one edge: {dup}"
    for c in SPGEMM_TABLE:
        off = sorted(set(c.edges) - so.edges(*graphs.spgemm_case(c.name)))
        assert not off, f"{c.id} does not reach {off}"

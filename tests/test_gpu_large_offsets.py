"""Every row of tests/large_offset_table.py on the GPU: an entry point with one operand of more than 2^31 elements (2^32
for the `wrap` rows), checked on a sampled set S of rows, columns or edges, never on the whole tensor.

S holds every index past the boundary that the case touches, the index whose run of elements straddles element 2^31,
the indices a 32-bit wrap would alias onto and a few low ones (store side: rows the call leaves empty, which must come
back zero).  Two checks, in this order:
  1. bit-identity with a compact twin: the same entry point on a small problem that holds exactly the rows in S, with
     renumbered columns and small operands, at the same F, plan form, panels and alignment.  Both calls must record the
     row's kernel string and the sampled outputs must match bit for bit.  A row's arithmetic depends on its degree and
     its chunking, never on its position, so a wrong offset shows up as a mismatch whatever its size.  Exceptions: the
     partial sums of the hub plan are numbered by chunk slot (the twin's slots are low, which is the point: its
     partials never cross); the element-wise actnn entries and gather_rows are checked against the operand itself;
     the dropout mask of gat_fwd_dropout depends on the CSR edge position, so only |att| is compared with the twin
     and the sign bits are compared with tests/gat_dropout_ref.keep_mask at the large graph's positions.
  2. the suite's per-element fp64 bounds (tests/test_gpu_dispatch.py) on the twin's inputs, against the sampled
     outputs of the large call, for the SpMM forms and epilogues, SDDMM, scatter_max, the edge softmax and the GAT
     forward; exact equality for the actnn entries.  The other message operators and fused layers (multi-head SpMM /
     SDDMM, GAT attention backward, edge_colsum, GENConv, DisenGCN, CompGCN, R-GCN, Simple-HGN, fused GCN / SAGE) rest
     on check 1: their twins are small problems of the kind their own per-element fp64 tests cover.
Each row's worst error-to-bound ratio is printed at the end.

The GPU is shared, so: before allocating, a row compares its bytes_needed + 2 GiB with torch.cuda.mem_get_info() and
skips (both numbers in the reason) when it does not fit; one row's tensors are held at a time and freed when it ends;
inputs are filled on the device from a seeded torch.Generator, and only S and the twin's operands are copied to the
host.  The largest row is large_offset_table.LARGEST: the Simple-HGN attention, about 20.4 GB (two [nnz, 8] fp32
tensors, colind, the plan's edge_row and etype).  A failing row's frames are cleared, so its tensors are freed too.
"""
import gc
import traceback

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests import large_offset_table as LT
from tests.gpu_util import plan_structure
from tests.test_gpu_dispatch import SLOPE, TINY, U32, check_softmax, gat_logits32, softmax_bwd64

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
RATIOS = {}
MARGIN = 2 * LT.GIB


@pytest.fixture(autouse=True)
def _one_case_at_a_time():
    gc.collect()
    torch.cuda.empty_cache()
    yield
    gc.collect()
    torch.cuda.empty_cache()


def need(c):
    free, total = torch.cuda.mem_get_info()
    if c.bytes_needed + MARGIN > free:
        pytest.skip(f"{c.id}: needs {c.bytes_needed} + {MARGIN} bytes, {free} of {total} free")


def gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def normal(shape, g, dtype=torch.float32, scale=1.0):
    t = torch.empty(shape, dtype=dtype, device=DEV)
    t.normal_(0.0, scale, generator=g)
    return t


def D(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


def structure(rp, ci, n_cols, plan):
    int32 = lambda a: a if isinstance(a, torch.Tensor) else a.astype(np.int32)  # noqa: E731
    return plan_structure(int32(rp), int32(ci), n_cols, DEV, plan, LT.CHUNK)


def last_kernel():
    from cogdl_b200 import _cabi

    return _cabi.last_kernel()


def check_kernel(c, big, twin):
    assert big == twin, f"{c.id}: the large call launched {big!r}, its twin {twin!r}"
    if c.kernel == LT.NO_KERNEL:
        return
    assert big == c.kernel, f"{c.id}: launched {big!r}, the table names {c.kernel!r}"


def assert_within(got, ref, bound, what):
    err = np.abs(np.asarray(got, np.float64) - ref)
    bad = np.argwhere(~(err <= bound))
    assert bad.size == 0, (f"{what}: {len(bad)} elements outside the bound, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]!r}, ref {ref[tuple(bad[0])]!r}, bound {bound[tuple(bad[0])]!r}")
    if err.size:
        RATIOS[what] = max(RATIOS.get(what, 0.0), float(np.max(err / np.maximum(bound, 1e-300))))


def same_bits(a, b, what):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    assert a.shape == b.shape, f"{what}: shapes {a.shape} and {b.shape}"
    ua = a.view(np.uint8).reshape(a.shape[0], -1)
    ub = b.view(np.uint8).reshape(b.shape[0], -1)
    bad = np.nonzero((ua != ub).any(1))[0]
    assert bad.size == 0, f"{what}: {bad.size} sampled rows differ from the twin's, first at sample {bad[0]}"


def spmm_bound(rp, ci, val, X):
    A = sp.csr_matrix((val.astype(np.float64), ci, rp), shape=(rp.shape[0] - 1, X.shape[0]))
    A.sum_duplicates()                       # values are >= 0 here, so |A| of the sums is the sum of the |a|
    X64 = X.astype(np.float64)
    deg = np.diff(rp)[:, None]
    return A @ X64, deg * U32 * (abs(A) @ np.abs(X64)), A


# ------------------------------------------------------------------------------------------ graphs
def gather_graph(c, rng):
    """GATHER_ROWS rows whose edges point at the sampled columns (the band past the boundary, the straddling column,
    the alias columns, the low columns)."""
    deg = np.array([LT.DEGREES[i % len(LT.DEGREES)] for i in range(c.n_rows)])
    rp = np.concatenate([[0], np.cumsum(deg)]).astype(np.int64)
    cols = np.array(c.samples)
    ci = rng.choice(cols, rp[-1]).astype(np.int64)
    for k, col in enumerate(cols):             # every sampled column at least once
        ci[(k * 7) % ci.size] = col
    return rp, ci


def compact(rp, ci):
    """The twin of a gather graph: the same rows, columns renumbered over the ones used."""
    uniq, inv = np.unique(ci, return_inverse=True)
    return inv.astype(np.int64), uniq


def store_graph(c, rng):
    """n_rows just past 2^31 / F: the band at the top and the straddling row hold edges (unsplit, hub and empty rows),
    every other row is empty.  Returns (deg, rowptr, colind, S)."""
    S = np.array(c.samples)
    band = [r for r in S if r >= c.n_rows - LT.BAND or r == c.straddle]
    deg = np.zeros(c.n_rows, np.int64)
    for k, r in enumerate(band):
        deg[r] = LT.DEGREES[k % len(LT.DEGREES)]
    rp = np.concatenate([[0], np.cumsum(deg)])
    ci = rng.integers(0, c.n_cols, rp[-1])
    extra = rng.integers(LT.BAND, c.straddle, 4)               # untouched low rows
    return deg, rp, ci, np.unique(np.concatenate([S, extra]))


def twin_rows(deg, rp, S):
    """Row-subset twin: (rowptr, edge positions of the rows in S, in order)."""
    d = deg[S]
    edges = np.concatenate([np.arange(rp[r], rp[r + 1]) for r in S] + [np.zeros(0, np.int64)])
    return np.concatenate([[0], np.cumsum(d)]), edges


# ------------------------------------------------------------------------------------------ SpMM family
def _spmm_call(c, st, val, x, **ep):
    from cogdl_b200.operators import _raw
    from cogdl_b200.operators.label_prop import label_prop_raw

    e = c.entry
    if e in ("cogdl_b200_spmm_csr_f32_ex", "cogdl_b200_spmm_csr_f16"):
        return _raw.spmm_raw(st, val, x, panels=c.panels)
    if e == "cogdl_b200_spmm_residual_f32":
        return _raw.spmm_residual_raw(st, val, x, ep["z"], 0.75, -1.25, ep["rs"], panels=c.panels)
    if e == "cogdl_b200_label_prop_f32":
        return label_prop_raw(st, val, x, ep["z"], 0.75, -1.25, ep["rs"], clamp=(-1.0, 1.0), panels=c.panels)
    if e == "cogdl_b200_spmm_residual_dcoef_f32":
        return _raw.spmm_residual_dcoef_raw(st, val, x, ep["z"], 0.75, ep["b_dev"], ep["rs"], panels=c.panels)
    if e == "cogdl_b200_spmm_accum_f32":
        last = ep["acc_in"] is not None
        xn = _raw.spmm_accum_raw(st, val, x, ep["acc"], ep["acc_in"], ep["rs"], last=last, scale=0.25,
                                 panels=c.panels)
        return ep["acc"] if last else (ep["acc"], xn)
    raise AssertionError(e)


def _epilogue_ref(c, sum64, mag, rs, z, acc_in):
    """fp64 epilogue of the row sums and its bound (one rounding per epilogue operation)."""
    r = rs.astype(np.float64)[:, None]
    e = c.entry
    if e == "cogdl_b200_spmm_accum_f32":
        xn = r * sum64
        xb = r * mag + U32 * np.abs(xn)
        acc = acc_in.astype(np.float64) + xn
        ab = xb + U32 * np.abs(acc)
        if c.operand == "ACC":
            return acc, ab, xn, xb
        return 0.25 * acc, 0.25 * ab + U32 * 0.25 * np.abs(acc), None, None
    a, b = 0.75, (-1.25 if e != "cogdl_b200_spmm_residual_dcoef_f32" else 1.5)
    out = a * r * sum64 + b * z.astype(np.float64)
    bound = a * np.abs(r) * mag + 4 * U32 * (np.abs(a * r * sum64) + np.abs(b * z)) + TINY
    if e == "cogdl_b200_label_prop_f32":
        out = np.clip(out, -1.0, 1.0)
    return out, bound, None, None


def run_spmm_gather(c):
    rng = np.random.default_rng(7 + c.F)
    g = gen(11 + c.F)
    dt = torch.float16 if c.dtype == "f16" else torch.float32
    X = normal((c.n_cols, c.F), g, dt)
    rp, ci = gather_graph(c, rng)
    val = rng.random(ci.size).astype(np.float32)
    vd = D(val).to(dt)
    y = _spmm_call(c, structure(rp, ci, c.n_cols, c.plan), vd, X)
    k_big = last_kernel()
    got = y.cpu().numpy()
    ci_t, uniq = compact(rp, ci)
    X_t = X[D(uniq)].contiguous()
    del X, y
    y_t = _spmm_call(c, structure(rp, ci_t, uniq.size, c.plan), vd, X_t)
    check_kernel(c, k_big, last_kernel())
    same_bits(got, y_t.cpu().numpy(), c.id)
    Xh = X_t.cpu().numpy()
    if c.dtype == "f16":
        v16 = val.astype(np.float16)
        ref, mag, _ = spmm_bound(rp, ci_t, v16.astype(np.float32), Xh.astype(np.float32))
        assert_within(got.astype(np.float32), ref, 2.0 ** -11 * np.abs(ref) + mag + 2.0 ** -24, c.id)
    else:
        ref, mag, _ = spmm_bound(rp, ci_t, val, Xh)
        assert_within(got, ref, mag + TINY, c.id)


def run_spmm_store(c):
    rng = np.random.default_rng(17 + c.F)
    g = gen(19 + c.F)
    dt = torch.float16 if c.dtype == "f16" else torch.float32
    deg, rp, ci, S = store_graph(c, rng)
    X = normal((c.n_cols, c.F), g, dt)
    val = rng.random(ci.size).astype(np.float32)
    vd = D(val).to(dt)
    Sd = D(S)
    ep = {}
    if c.role == "epilogue":
        rs = torch.rand(c.n_rows, generator=g, device=DEV)
        ep = {"rs": rs, "z": None, "acc": None, "acc_in": None, "b_dev": torch.tensor([1.5], device=DEV)}
        if c.entry == "cogdl_b200_spmm_accum_f32":
            ep["acc" if c.operand == "ACC" else "acc_in"] = normal((c.n_rows, c.F), g)
            if c.operand == "ACC_in":
                ep["acc"] = torch.empty((c.n_rows, c.F), device=DEV)
                ep["rs"] = None
        else:
            ep["z"] = normal((c.n_rows, c.F), g)
    # the twin's row operands: the rows in S, sliced before the large call (ACC is updated in place)
    ep_t = {k: (v[Sd].contiguous() if (v is not None and k != "b_dev") else v) for k, v in ep.items()}
    if c.operand == "ACC_in":
        ep_t["acc"] = torch.empty((S.size, c.F), device=DEV)
    host = {k: (v.cpu().numpy() if v is not None and k not in ("b_dev", "acc") else None) for k, v in ep_t.items()}
    if c.operand == "ACC":
        host["acc_in"] = ep_t["acc"].cpu().numpy()          # accumulated in place: ACC's input
    st = structure(rp, ci, c.n_cols, c.plan)
    y = _spmm_call(c, st, vd, X, **ep)
    k_big = last_kernel()
    if isinstance(y, tuple):
        got = [t[Sd].cpu().numpy() for t in y]
    else:
        got = [y[Sd].cpu().numpy()]
    del y, st
    ep.clear()
    rp_t, edges = twin_rows(deg, rp, S)
    y_t = _spmm_call(c, structure(rp_t, ci[edges], c.n_cols, c.plan), vd[D(edges)], X, **ep_t)
    check_kernel(c, k_big, last_kernel())
    y_t = list(y_t) if isinstance(y_t, tuple) else [y_t]
    for k, (a, b) in enumerate(zip(got, y_t)):
        same_bits(a, b.cpu().numpy(), f"{c.id} output {k}")
    Xh = X[:].cpu().numpy().astype(np.float32)
    v = val[edges]
    if c.dtype == "f16":
        v = v.astype(np.float16).astype(np.float32)
    ref, mag, _ = spmm_bound(rp_t, ci[edges], v, Xh)
    if c.role == "store":
        bound = (2.0 ** -11 * np.abs(ref) + mag + 2.0 ** -24) if c.dtype == "f16" else mag + TINY
        assert_within(got[0].astype(np.float32), ref, bound, c.id)
        assert not got[0][deg[S] == 0].any(), f"{c.id}: an empty row is not zero"
        return
    rs = host["rs"] if host["rs"] is not None else np.ones(S.size, np.float32)
    out, bound, xn, xb = _epilogue_ref(c, ref, mag, rs, host["z"], host["acc_in"])
    if c.entry == "cogdl_b200_spmm_accum_f32" and c.operand == "ACC":
        assert_within(got[1], xn, xb + TINY, f"{c.id} Xn")
        assert_within(got[0], out, bound + TINY, f"{c.id} ACC")
    else:
        assert_within(got[0], out, bound + TINY, c.id)


def run_spmm_partials(c):
    """Eight hub rows of LCase.part_deg edges: the last rows' chunk slots put their partial sums past element 2^31 of
    the scratch.  The twin holds rows 0 and 7 alone, whose slots are low.  The SpMM at F = 3703, and R-GCN's
    aggregation at B = 8, F = 128 (partials n_chunks * B * F)."""
    from cogdl_b200.operators import _raw

    g = gen(23)
    rgcn = c.entry == "cogdl_b200_rgcn_aggr_f32"
    X = normal((c.n_cols, c.F), g)
    rp = np.arange(LT.PART_ROWS + 1, dtype=np.int64) * c.part_deg
    nnz = int(rp[-1])
    ci_d = torch.randint(0, c.n_cols, (nnz,), generator=g, device=DEV, dtype=torch.int32)
    etype = torch.randint(0, 3, (nnz,), generator=g, device=DEV, dtype=torch.int32) if rgcn else None
    w = torch.rand(nnz, generator=g, device=DEV) if rgcn else None
    coef = normal((3, c.H), g)

    def call(st, et, ww):
        if rgcn:
            return _raw.rgcn_aggr_raw(st, et, ww, coef, X)
        return _raw.spmm_raw(st, None, X, panels=c.panels)

    st = structure(rp, ci_d, c.n_cols, c.plan)
    assert st.plan.n_chunks == c.n_chunks
    y = call(st, etype, w)
    k_big = last_kernel()
    S = np.array([0, LT.PART_ROWS - 1])
    got = y[D(S)].cpu().numpy()
    del st, y
    edges = D(np.concatenate([np.arange(rp[r], rp[r + 1]) for r in S]))
    ci_t = ci_d[edges].contiguous()
    et_t = etype[edges].contiguous() if rgcn else None
    w_t = w[edges].contiguous() if rgcn else None
    del ci_d, etype, w
    rp_t = np.array([0, c.part_deg, 2 * c.part_deg])
    y_t = call(structure(rp_t, ci_t, c.n_cols, c.plan), et_t, w_t)
    check_kernel(c, k_big, last_kernel())
    same_bits(got, y_t.cpu().numpy(), c.id)
    if rgcn:
        RATIOS[c.id] = 0.0
        return
    ref, mag, _ = spmm_bound(rp_t, ci_t.cpu().numpy().astype(np.int64), np.ones(edges.numel(), np.float32),
                             X.cpu().numpy())
    assert_within(got, ref, mag + TINY, c.id)


# ------------------------------------------------------------------------------------------ SDDMM, scatter_max
def run_sddmm(c):
    from cogdl_b200.operators._raw import sddmm_raw

    rng = np.random.default_rng(29)
    g = gen(31)
    D2 = normal((c.n_cols, c.F), g)
    rp, ci = gather_graph(c, rng)
    D1 = normal((c.n_rows, c.F), g)
    out = sddmm_raw(structure(rp, ci, c.n_cols, c.plan), D1, D2)
    k_big = last_kernel()
    got = out.cpu().numpy()
    ci_t, uniq = compact(rp, ci)
    D2_t = D2[D(uniq)].contiguous()
    del D2
    out_t = sddmm_raw(structure(rp, ci_t, uniq.size, c.plan), D1, D2_t)
    check_kernel(c, k_big, last_kernel())
    same_bits(got[:, None], out_t.cpu().numpy()[:, None], c.id)
    rows = np.repeat(np.arange(c.n_rows), np.diff(rp))
    terms = D1.cpu().numpy()[rows].astype(np.float64) * D2_t.cpu().numpy()[ci_t].astype(np.float64)
    assert_within(got, terms.sum(-1), c.F * U32 * np.abs(terms).sum(-1) + TINY, c.id)


def _smax_ref(rp, ci, X):
    import oracle

    return oracle.scatter_max_fwd(rp.astype(np.int32), ci.astype(np.int32), X)


def run_scatter_max(c):
    from cogdl_b200.operators._raw import scatter_max_fwd_raw

    rng = np.random.default_rng(37)
    g = gen(41)
    if c.role == "gather":
        X = normal((c.n_cols, c.F), g, scale=4.0).round_().div_(4)          # ties: the first max wins
        rp, ci = gather_graph(c, rng)
        out, arg = scatter_max_fwd_raw(structure(rp, ci, c.n_cols, c.plan), X)
        k_big = last_kernel()
        got, got_arg = out.cpu().numpy(), arg.cpu().numpy()
        ci_t, uniq = compact(rp, ci)
        X_t = X[D(uniq)].contiguous()
        del X, out, arg
        out_t, arg_t = scatter_max_fwd_raw(structure(rp, ci_t, uniq.size, c.plan), X_t)
        check_kernel(c, k_big, last_kernel())
        same_bits(got, out_t.cpu().numpy(), c.id)
        a_t = arg_t.cpu().numpy()
        assert np.array_equal(got_arg, np.where(a_t >= 0, uniq[np.maximum(a_t, 0)], -1)), f"{c.id}: argmax"
        ref, ref_id = _smax_ref(rp, ci_t, X_t.cpu().numpy())
    else:
        deg, rp, ci, S = store_graph(c, rng)
        X = normal((c.n_cols, c.F), g, scale=4.0).round_().div_(4)
        out, arg = scatter_max_fwd_raw(structure(rp, ci, c.n_cols, c.plan), X)
        k_big = last_kernel()
        Sd = D(S)
        got, got_arg = out[Sd].cpu().numpy(), arg[Sd].cpu().numpy()
        del out, arg
        rp_t, edges = twin_rows(deg, rp, S)
        out_t, arg_t = scatter_max_fwd_raw(structure(rp_t, ci[edges], c.n_cols, c.plan), X)
        check_kernel(c, k_big, last_kernel())
        same_bits(got, out_t.cpu().numpy(), c.id)
        assert np.array_equal(got_arg, arg_t.cpu().numpy()), f"{c.id}: argmax"
        ref, ref_id = _smax_ref(rp_t, ci[edges], X.cpu().numpy())
    assert np.array_equal(got, ref) and np.array_equal(got_arg if c.role == "store" else a_t, ref_id), \
        f"{c.id}: not the exact maximum / first argmax"
    RATIOS[c.id] = 0.0


def run_scatter_max_bwd(c):
    """gx [n_src, F] with n_src just past 2^31 / F: argmax points at the sampled columns, every (column, feature) at
    most once, so that the kernel's atomic adds land on zeros and the twin's result is bit-identical."""
    from cogdl_b200.operators._raw import scatter_max_bwd_raw

    g = gen(47)
    cols = np.array(c.samples)
    n = cols.size
    arg = cols[(np.arange(n)[:, None] + np.arange(c.F)[None, :]) % n].astype(np.int32)
    arg[::7, ::3] = -1
    grad = normal((n, c.F), g)
    gx = scatter_max_bwd_raw(grad, D(arg), c.n_cols)
    k_big = last_kernel()
    got = gx[D(cols)].cpu().numpy()
    del gx
    inv = np.searchsorted(cols, np.maximum(arg, 0))
    arg_t = np.where(arg >= 0, inv, -1).astype(np.int32)
    gx_t = scatter_max_bwd_raw(grad, D(arg_t), cols.size)
    check_kernel(c, k_big, last_kernel())
    same_bits(got, gx_t.cpu().numpy(), c.id)
    gh = grad.cpu().numpy().astype(np.float64)
    want, mag, cnt = (np.zeros((cols.size, c.F)) for _ in range(3))
    ok = arg_t >= 0
    fcol = np.broadcast_to(np.arange(c.F), arg.shape)[ok]
    np.add.at(want, (arg_t[ok], fcol), gh[ok])
    np.add.at(mag, (arg_t[ok], fcol), np.abs(gh[ok]))
    np.add.at(cnt, (arg_t[ok], fcol), 1)
    assert_within(got, want, cnt * U32 * mag + TINY, c.id)


# ------------------------------------------------------------------------------------------ edge-aligned tensors
def edge_graph(g):
    deg = np.array(LT.edge_degrees(), np.int64)
    rp = np.concatenate([[0], np.cumsum(deg)])
    n = deg.size
    ci = torch.randint(0, n, (int(rp[-1]),), generator=g, device=DEV, dtype=torch.int32)
    tail = int(rp[LT.EDGE_FULL])
    ci[tail:] = torch.randint(0, TAIL_COLS, (int(rp[-1]) - tail,), generator=g, device=DEV, dtype=torch.int32)
    return deg, rp, ci, n


TAIL_COLS = 8   # the tail rows' edges point at columns below this: the first rows of the transpose hold them all


def edge_twin(c, deg, rp, ci):
    """Rows owning a sampled edge, their edges (positions in the large graph) and the twin's (rowptr, colind, cols)."""
    e = np.array([s for s in c.samples if s < rp[-1]])
    rows = np.unique(np.searchsorted(rp, e, side="right") - 1)
    rp_t, edges = twin_rows(deg, rp, rows)
    cols = ci[D(edges)].cpu().numpy().astype(np.int64)
    ci_t, uniq = compact(rp_t, cols)
    return rows, edges, rp_t, ci_t, uniq


def run_edge(c):
    from cogdl_b200.operators import _raw
    from tests.gat_dropout_ref import draw, drop_below

    g = gen(53)
    if c.entry == "cogdl_b200_gather_rows_f32":
        return run_gather_rows(c, g)
    deg, rp, ci, n = edge_graph(g)
    H = c.H
    rows, edges, rp_t, ci_t, uniq = edge_twin(c, deg, rp, ci)
    Ed, Rd, Ud = D(edges), D(rows), D(uniq)
    st = structure(rp, ci, n, "default")
    st_t = structure(rp_t, ci_t, uniq.size, "default")
    name = c.entry
    if name == "cogdl_b200_edge_softmax_fwd_f32":
        x = normal((st.nnz, H), g, scale=2.0)
        out = _raw.edge_softmax_fwd_raw(st, x)
        k_big = last_kernel()
        got = out[Ed].cpu().numpy()
        x_t = x[Ed].contiguous()
        del out, x
        out_t = _raw.edge_softmax_fwd_raw(st_t, x_t)
        check_kernel(c, k_big, last_kernel())
        same_bits(got, out_t.cpu().numpy(), c.id)
        check_softmax(got, x_t.cpu().numpy(), rp_t, c.id)
        from tests.test_gpu_dispatch import RATIOS as DR
        RATIOS[c.id] = DR.pop(c.id)
    elif name == "cogdl_b200_edge_softmax_bwd_f32":
        y = torch.rand((st.nnz, H), generator=g, device=DEV)
        out = _raw.edge_softmax_bwd_raw(st, y, y)
        k_big = last_kernel()
        got = out[Ed].cpu().numpy()
        y_t = y[Ed].contiguous()
        del out, y
        out_t = _raw.edge_softmax_bwd_raw(st_t, y_t, y_t)
        check_kernel(c, k_big, last_kernel())
        same_bits(got, out_t.cpu().numpy(), c.id)
        yh = y_t.cpu().numpy()
        ref, bound, _, _ = softmax_bwd64(rp_t, yh, yh, 1.0)
        assert_within(got, ref, bound, c.id)
    elif name in ("cogdl_b200_gat_fwd_f32", "cogdl_b200_gat_fwd_dropout_f32"):
        hl = normal((n, H), g)
        hr = normal((n, H), g, scale=8.0)
        feat = normal((n, H, c.F), g)
        p = 0.4
        drop = (0x5EED, drop_below(p), 1.0 / (1.0 - p)) if "dropout" in name else None
        out, att = _raw.gat_fwd_raw(st, hl, hr, feat, float(SLOPE), True, drop=drop)
        k_big = last_kernel()
        got_att, got_out = att[Ed].cpu().numpy(), out[Rd].cpu().numpy()
        del out, att
        hl_t, hr_t, feat_t = hl[Rd].contiguous(), hr[Ud].contiguous(), feat[Ud].contiguous()
        out_t, att_t = _raw.gat_fwd_raw(st_t, hl_t, hr_t, feat_t, float(SLOPE), True, drop=drop)
        check_kernel(c, k_big, last_kernel())
        att_t = att_t.cpu().numpy()
        if drop is None:
            same_bits(got_att, att_t, f"{c.id} attention")
            same_bits(got_out, out_t.cpu().numpy(), f"{c.id} out")
        else:
            same_bits(np.abs(got_att), np.abs(att_t), f"{c.id} |attention|")
            keep = draw(drop[0], edges.astype(np.uint64)[:, None], np.arange(H, dtype=np.uint64)[None, :]) \
                >= np.uint64(drop[1])
            assert np.array_equal(np.signbit(got_att), ~keep), f"{c.id}: the sign bits are not the dropout mask"
        hlh, hrh = hl_t.cpu().numpy(), hr_t.cpu().numpy()
        check_softmax(np.abs(got_att), gat_logits32(rp_t, ci_t, hlh, hrh)[1], rp_t, c.id)
        from tests.test_gpu_dispatch import RATIOS as DR
        RATIOS[c.id] = DR.pop(c.id)
        eff = got_att if drop is None else np.where(np.signbit(got_att), 0, np.abs(got_att) * np.float32(drop[2]))
        fh = feat_t.cpu().numpy()
        for h in range(H):
            ref, mag, _ = spmm_bound(rp_t, ci_t, eff[:, h].astype(np.float32), fh[:, h, :])
            assert_within(got_out[:, h, :], ref, mag + TINY, f"{c.id} out")
    else:
        raise AssertionError(name)
    assert int(st.plan.counters.abs().sum()) == 0, f"{c.id}: arrival counters not back at zero"


def run_gather_rows(c, g):
    """out[q] = in[perm[q]] over [nnz, H] with the reversing permutation: checked against the operand itself."""
    from cogdl_b200.operators import _raw

    nnz = int(sum(LT.edge_degrees()))
    perm = torch.arange(nnz - 1, -1, -1, dtype=torch.int32, device=DEV)
    x = normal((nnz, c.H), g)
    out = _raw.gather_rows_raw(perm, x)
    q = D(np.array(c.samples))
    assert torch.equal(out[q], x[nnz - 1 - q]), f"{c.id}: out[q] != in[perm[q]]"
    assert c.kernel == LT.NO_KERNEL
    RATIOS[c.id] = 0.0


# ------------------------------------------------------------------------------------------ activation compression
def run_actnn(c):
    from cogdl_b200.actnn import kernels as K
    from tests import actnn_ref as R

    g = gen(59)
    N, Dm = c.n_rows, c.F
    S = np.array(c.samples)
    Sd = D(S)
    x = normal((N, Dm), g)
    name = c.entry
    if name in ("cogdl_b200_actnn_minmax_f32", "cogdl_b200_actnn_pack_f32", "cogdl_b200_actnn_unpack_f32"):
        gs = 256
        if name == "cogdl_b200_actnn_minmax_f32":
            mn, mx = K.group_minmax(x, gs)
            k_big = last_kernel()
            got = np.stack([mn[Sd].cpu().numpy(), mx[Sd].cpu().numpy()], 1)
            del mn, mx
            x_t = x[Sd].contiguous()
            mn_t, mx_t = K.group_minmax(x_t, gs)
            check_kernel(c, k_big, last_kernel())
            same_bits(got, np.stack([mn_t.cpu().numpy(), mx_t.cpu().numpy()], 1), c.id)
            xh = x_t.cpu().numpy()
            assert np.array_equal(got[:, 0, 0], xh[:, :gs].min(1)) and np.array_equal(got[:, 1, 0], xh[:, :gs].max(1)), c.id
        else:
            packed, scale, mn = K.pack(x, 8, gs, False)
            k_pack = last_kernel()
            x_t = x[Sd].contiguous()
            del x
            if name == "cogdl_b200_actnn_pack_f32":
                got = packed.view(N, -1)[Sd].cpu().numpy()
                k_big = k_pack
            else:
                out = K.unpack(packed, 8, scale, mn, N, Dm, gs)
                k_big = last_kernel()
                got = out[Sd].cpu().numpy()
                del out
            p_t = packed.view(N, -1)[Sd].contiguous().view(-1)
            s_t, m_t = scale[Sd].contiguous(), mn[Sd].contiguous()
            if name == "cogdl_b200_actnn_pack_f32":
                pt, st_, mt = K.pack(x_t, 8, gs, False)
                check_kernel(c, k_big, last_kernel())
                same_bits(got, pt.view(S.size, -1).cpu().numpy(), c.id)
                codes, rscale, rmn = R.quantize(x_t.cpu().numpy(), 8, gs)
                assert np.array_equal(got, R.pack(codes, 8).reshape(S.size, -1)), f"{c.id}: codes"
            else:
                out_t = K.unpack(p_t, 8, s_t, m_t, S.size, Dm, gs)
                check_kernel(c, k_big, last_kernel())
                same_bits(got, out_t.cpu().numpy(), c.id)
                codes = p_t.cpu().numpy().reshape(S.size, -1)
                want = R.dequantize(codes, s_t.float().cpu().numpy(), m_t.float().cpu().numpy(), Dm, gs)
                assert np.array_equal(got, want), f"{c.id}: not the dequantized codes"
        RATIOS[c.id] = 0.0
        return
    flat = x.view(-1)
    idx = (Sd[:, None] * Dm + torch.arange(Dm, device=DEV)[None, :]).view(-1)   # every element of the sampled rows
    ih = idx.cpu().numpy()
    xs = flat[idx].cpu().numpy()
    p = 0.3
    if name in ("cogdl_b200_actnn_relu_fwd_f32", "cogdl_b200_actnn_dropout_fwd_f32"):
        y, mask = K.relu_fwd(flat) if "relu" in name else K.dropout_fwd(flat, p, 61)
        k_big = last_kernel()
        ys = y[idx].cpu().numpy()
        bits = ((mask[idx >> 5].cpu().numpy().astype(np.uint32) >> (ih & 31).astype(np.uint32)) & 1).astype(bool)
        if "relu" in name:
            keep = xs > 0
            want = np.where(keep, xs, np.float32(0))
        else:
            keep = R.draw(61, ih.astype(np.uint64), 0) >= np.uint64(K.dropout_threshold(p))
            want = np.where(keep, (xs.astype(np.float64) / (1.0 - float(np.float32(p)))).astype(np.float32),
                            np.float32(0))
        del y, mask
        K.relu_fwd(flat[:64]) if "relu" in name else K.dropout_fwd(flat[:64], p, 61)
    else:
        mask = torch.randint(-2 ** 31, 2 ** 31 - 1, ((flat.numel() + 31) // 32,), generator=g, device=DEV,
                             dtype=torch.int32)
        gx = K.relu_bwd(flat, mask) if "relu" in name else K.dropout_bwd(flat, mask, p)
        k_big = last_kernel()
        ys = gx[idx].cpu().numpy()
        keep = ((mask[idx >> 5].cpu().numpy().astype(np.uint32) >> (ih & 31).astype(np.uint32)) & 1).astype(bool)
        bits = keep
        want = np.where(keep, xs if "relu" in name else
                        (xs.astype(np.float64) / (1.0 - float(np.float32(p)))).astype(np.float32), np.float32(0))
        del gx
        K.relu_bwd(flat[:64], mask[:2]) if "relu" in name else K.dropout_bwd(flat[:64], mask[:2], p)
    check_kernel(c, k_big, last_kernel())
    assert np.array_equal(bits, keep), f"{c.id}: mask bits"
    same_bits(ys[:, None], want[:, None], c.id)
    RATIOS[c.id] = 0.0


# ------------------------------------------------------------------------------------------ message operators, fused
# layers and the other SpMM forms: one twin pattern per role
def _np(t):
    return t.cpu().numpy()


def twin_gather(c, seed, make_big, make_small, call, col_out=(), encode=None):
    """make_big(n_cols, g) -> column-indexed operands (the large ones); make_small(rp, ci, g) -> the rest;
    call(st, big, small) -> outputs.  Outputs listed in col_out are column-indexed (a pass over the transpose) and are
    compared at the columns the graph uses; the others whole.  Returns (outputs, rp, compact colind, big of the twin,
    small)."""
    rng = np.random.default_rng(seed)
    g = gen(seed)
    big = make_big(c.n_cols, g)
    rp, ci = gather_graph(c, rng)
    small = make_small(rp, ci, g)
    enc = encode or (lambda x: x)
    ci_t, uniq = compact(rp, ci)
    U = D(uniq)
    outs = call(structure(rp, enc(ci), c.n_cols, c.plan), big, small)
    k_big = last_kernel()
    got = [_np(o[U] if k in col_out else o) for k, o in enumerate(outs)]
    big_t = tuple(b[U].contiguous() for b in big)
    del big, outs
    outs_t = call(structure(rp, enc(ci_t), uniq.size, c.plan), big_t, small)
    check_kernel(c, k_big, last_kernel())
    for k, o in enumerate(outs_t):
        same_bits(got[k], _np(o), f"{c.id} output {k}")
    return got, rp, ci_t, big_t, small


def twin_store(c, seed, make_rows, make_small, call):
    """make_rows(n_rows, g) -> row-indexed large inputs; make_small(nnz, g) -> column operands and per-edge arrays;
    call(st, rows, small, E) -> row-indexed outputs, E slicing a per-edge array to the twin's edges (identity for the
    large call).  Compared at the sampled rows (the band, the straddling row, untouched low rows)."""
    rng = np.random.default_rng(seed)
    g = gen(seed)
    deg, rp, ci, S = store_graph(c, rng)
    Sd = D(S)
    small = make_small(int(rp[-1]), g)
    rows = make_rows(c.n_rows, g)
    rows_t = tuple(r[Sd].contiguous() for r in rows)
    outs = call(structure(rp, ci, c.n_cols, c.plan), rows, small, lambda t: t)
    k_big = last_kernel()
    got = [_np(o[Sd]) for o in outs]
    del rows, outs
    rp_t, edges = twin_rows(deg, rp, S)
    Ed = D(edges)
    outs_t = call(structure(rp_t, ci[edges], c.n_cols, c.plan), rows_t, small, lambda t: t[Ed].contiguous())
    check_kernel(c, k_big, last_kernel())
    for k, o in enumerate(outs_t):
        same_bits(got[k], _np(o), f"{c.id} output {k}")
    return got, S, deg


def twin_edge(c, seed, make_edge, make_small, call):
    """make_edge(nnz, g) -> [nnz, *] operands (the large ones); make_small(n, g) -> {name: (tensor, 'row' | 'col' |
    'etype' | 'none')}; call(st, e, small) -> [(output, 'edge' | 'row')].  The twin holds every row with an edge past
    the boundary, row 0 and the straddling row."""
    g = gen(seed)
    deg, rp, ci, n = edge_graph(g)
    rows, edges, rp_t, ci_t, uniq = edge_twin(c, deg, rp, ci)
    Ed, Rd, Ud = D(edges), D(rows), D(uniq)
    st = structure(rp, ci, n, "default")
    e = make_edge(st.nnz, g)
    small = make_small(n, g)
    sl = {"row": Rd, "col": Ud, "etype": Ed}
    small_t = {k: (v if kind == "none" else v[sl[kind]].contiguous(), kind) for k, (v, kind) in small.items()}
    e_t = tuple(x[Ed].contiguous() for x in e)
    outs = call(st, e, small)
    k_big = last_kernel()
    got = [_np(o[Ed] if kind == "edge" else o[Rd]) for o, kind in outs]
    assert int(st.plan.counters.abs().sum()) == 0, f"{c.id}: arrival counters not back at zero"
    del outs, e, st
    st_t = structure(rp_t, ci_t, uniq.size, "default")
    outs_t = call(st_t, e_t, small_t)
    check_kernel(c, k_big, last_kernel())
    for k, (o, _) in enumerate(outs_t):
        same_bits(got[k], _np(o), f"{c.id} output {k}")


def twin_transpose(c, seed, make_edge, make_rows, call):
    """A pass over the transpose of the edge graph with an [nnz, *] operand read through perm.  The tail's edges all
    point at columns 0..TAIL_COLS-1, so those rows of the transpose hold every edge past the boundary; the twin is
    those rows, the operand gathered through perm and an identity perm.  make_rows(n, g) -> operands indexed by the
    transpose's colind (rows of the graph); call(st_T, perm, e, rows) -> output [n_T, ...]."""
    g = gen(seed)
    deg, rp, ci, n = edge_graph(g)
    st = structure(rp, ci, n, "default")
    st_T, perm = st.csc()
    e = make_edge(st.nnz, g)
    rows = make_rows(n, g)
    outs = call(st_T, perm, e, rows)
    k_big = last_kernel()
    R = torch.arange(TAIL_COLS, device=DEV)
    got = [_np(o[R]) for o in outs]
    assert int(st_T.plan.counters.abs().sum()) == 0
    cp = _np(st_T.rowptr[:TAIL_COLS + 1]).astype(np.int64)
    q = torch.arange(int(cp[0]), int(cp[-1]), device=DEV)
    e_t = tuple(x[perm[q].long()].contiguous() for x in e)
    ci_t, uniq = compact(cp - cp[0], _np(st_T.colind[q]).astype(np.int64))
    rows_t = tuple(r[D(uniq)].contiguous() for r in rows)
    del outs, e, st, st_T, perm
    st_t = structure(cp - cp[0], ci_t, uniq.size, "default")
    outs_t = call(st_t, torch.arange(q.numel(), dtype=torch.int32, device=DEV), e_t, rows_t)
    check_kernel(c, k_big, last_kernel())
    for k, o in enumerate(outs_t):
        same_bits(got[k], _np(o), f"{c.id} output {k}")


def _launch_plain(st, val, x, y):
    from cogdl_b200.operators._raw import _launch, _scratch
    from cogdl_b200.structure import _ptr

    _launch("cogdl_b200_spmm_csr_f32", st, _scratch("spmm", st, x.shape[1]), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(val), _ptr(x), _ptr(y), st.n_rows, x.shape[1])
    return y


def _launch_sage(st, val, x, w_neigh, S):
    """cogdl_b200_sage_fused_f32 (sum aggregation) with the self half S given: x may have fewer rows than the graph."""
    from cogdl_b200.operators._raw import _launch, _scratch
    from cogdl_b200.structure import _ptr

    n, K, Fout = st.n_rows, x.shape[1], w_neigh.shape[0]
    out = torch.empty((n, Fout), device=DEV)
    hub = torch.empty((n, K), device=DEV) if st.plan.n_chunks > 0 else None
    _launch("cogdl_b200_sage_fused_f32", st, _scratch("sage_fused", st, K, 0), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(val), None, _ptr(x), _ptr(w_neigh), _ptr(S), _ptr(out), _ptr(hub), n, K, Fout, 0, 0)
    return out


PEER_SHIFT = 28


def _launch_peers(st, val, shard, y, n_local=1):
    """cogdl_b200_spmm_csr_f32_peers with one peer (owner 0): column n_local + r reads row r of `shard`."""
    import ctypes

    from cogdl_b200.operators._raw import _launch, _scratch
    from cogdl_b200.structure import _ptr

    local = torch.zeros((n_local, shard.shape[1]), device=DEV)
    ptrs = (ctypes.c_void_p * 1)(shard.data_ptr())
    _launch("cogdl_b200_spmm_csr_f32_peers", st, _scratch("spmm", st, shard.shape[1]), _ptr(st.rowptr),
            _ptr(st.colind), _ptr(val), _ptr(local), n_local, ctypes.cast(ptrs, ctypes.c_void_p), 1, PEER_SHIFT,
            _ptr(y), st.n_rows, shard.shape[1])
    return y


def run_spmm_forms(c):
    """The plain entry, the two-source form (the large operand is X1, behind 256 rows of X0) and the peer form (the
    large operand is a peer's shard)."""
    from cogdl_b200.operators._raw import spmm_2src_raw

    F = c.F
    n0 = 256
    e = c.entry

    def call(st, X1, X0, val):
        y = torch.empty((st.n_rows, F), device=DEV)
        if e == "cogdl_b200_spmm_csr_f32":
            return _launch_plain(st, val, X1, y)
        if e == "cogdl_b200_spmm_csr_f32_2src":
            return spmm_2src_raw(st, val, X0, X1)
        return _launch_peers(st, val, X1, y)

    if c.role == "gather":
        X0 = normal((n0, F), gen(1))
        shift = {"cogdl_b200_spmm_csr_f32": 0, "cogdl_b200_spmm_csr_f32_2src": n0}.get(e, 1)
        got, rp, ci_t, (X1_t,), (val,) = twin_gather(
            c, 71, lambda n, g: (normal((n, F), g),), lambda rp, ci, g: (torch.rand(int(rp[-1]), generator=g,
                                                                                     device=DEV),),
            lambda st, big, small: [call(st, big[0], X0, small[0])],
            encode=lambda ci: ci + shift)
        ref, mag, _ = spmm_bound(rp, ci_t, _np(val), _np(X1_t))
        assert_within(got[0], ref, mag + TINY, c.id)
        return
    X0 = normal((c.n_cols, F), gen(2))

    def scall(st, rows, small, E):
        val = E(small[0])
        if e == "cogdl_b200_spmm_csr_f32":
            return [_launch_plain(st, val, X0, torch.empty((st.n_rows, F), device=DEV))]
        if e == "cogdl_b200_spmm_csr_f32_2src":
            return [spmm_2src_raw(st, val, X0, X0[:0])]
        return [_launch_peers(st, val, X0, torch.empty((st.n_rows, F), device=DEV), n_local=c.n_cols)]

    got, S, deg = twin_store(c, 73, lambda n, g: (), lambda nnz, g: (torch.rand(nnz, generator=g, device=DEV),), scall)
    assert not got[0][deg[S] == 0].any(), f"{c.id}: an empty row is not zero"


def run_message(c):
    """Multi-head SpMM / SDDMM, GENConv, CompGCN, R-GCN and the fused GCN / SAGE layers on the gather, transpose-store
    and store graphs."""
    from cogdl_b200.operators import _raw
    from cogdl_b200.operators.fused_gcn import fused_gcn_raw

    e, F, H = c.entry, c.F, c.H
    beta = torch.tensor([0.7], device=DEV)
    R = c.n_rows

    def small_default(rp, ci, g):
        nnz = int(rp[-1])
        return {"w": torch.rand(nnz, generator=g, device=DEV),
                "att": torch.rand((nnz, H), generator=g, device=DEV),
                "rows": normal((R, H, F), g),
                "etype": torch.randint(0, 3, (nnz,), generator=g, device=DEV, dtype=torch.int32),
                "coef": normal((3, 2), g),
                "B": normal((64, F), g),
                "idx2": torch.randint(0, 64, (nnz,), generator=g, device=DEV, dtype=torch.int32),
                "attr": normal((nnz, 4), g),
                "W": normal((F, 4), g, scale=0.3),
                "G": normal((R, F), g),
                "Wl": normal((16, 128), g, scale=0.1),
                "S": normal((R, 16), g)}

    width = F * H
    if c.role in ("gather", "tstore"):
        def big(n, g):
            return (normal((n, width), g),)

        def call(st, b, s):
            X = b[0]
            if e == "cogdl_b200_mhspmm_f32":
                return [_raw.mhspmm_raw(st, s["att"], X.view(-1, H, F))]
            if e == "cogdl_b200_mhsddmm_f32":
                return [_raw.mhsddmm_raw(st, s["rows"], X.view(-1, H, F))]
            if e == "cogdl_b200_softmax_aggr_fwd_f32":
                return list(_raw.softmax_aggr_fwd_raw(st, X, beta, 1e-7, want_lse=True, want_q=True))
            if e == "cogdl_b200_softmax_aggr_bwd_f32":
                out, lse2, _ = _raw.softmax_aggr_fwd_raw(st, X, beta, 1e-7, want_lse=True)
                return [_raw.softmax_aggr_bwd_raw(st, X, beta, 1e-7, s["G"], out, lse2)[0]]
            if e == "cogdl_b200_genconv_edge_fwd_f32":
                return list(_raw.genconv_edge_fwd_raw(st, X, s["attr"], s["W"], beta, 1e-7, True, True))
            if e == "cogdl_b200_genconv_edge_bwd_f32":
                out, lse2, _ = _raw.genconv_edge_fwd_raw(st, X, s["attr"], s["W"], beta, 1e-7, want_lse=True)
                return [_raw.genconv_edge_bwd_raw(st, X, s["attr"], s["W"], beta, 1e-7, s["G"], out, lse2,
                                                  want_dw=False)[0]]
            if e == "cogdl_b200_comp_aggr_f32":
                return [_raw.comp_aggr_raw(st, s["idx2"], s["w"], X, s["B"], "mult")]
            if e == "cogdl_b200_rgcn_aggr_f32":
                if H > 1:
                    return [_raw.rgcn_aggr_raw(st, s["etype"], s["w"], s["coef"], X.view(-1, H, F), per_basis=True)]
                return [_raw.rgcn_aggr_raw(st, s["etype"], s["w"], s["coef"], X)]
            if e == "cogdl_b200_rgcn_edge_dot_f32":
                return [_raw.rgcn_edge_dot_raw(st, s["w"], s["rows"].view(R, 1, F).expand(R, 2, F).contiguous(), X)]
            if e == "cogdl_b200_gcn_fused_f32":
                return [fused_gcn_raw(st, s["w"], X, s["Wl"])]
            if e == "cogdl_b200_sage_fused_f32":
                return [_launch_sage(st, s["w"], X, s["Wl"], s["S"])]
            raise AssertionError(e)

        def small(rp, ci, g):
            return small_default(rp, ci, g)

        twin_gather(c, 83, big, small, call, col_out=(0,) if c.role == "tstore" else ())
        RATIOS[c.id] = 0.0
        return
    # store side: the row-indexed output is the large operand
    Xs = normal((c.n_cols, width), gen(3))

    def make_small(nnz, g):
        return {"w": torch.rand(nnz, generator=g, device=DEV), "att": torch.rand((nnz, H), generator=g, device=DEV),
                "etype": torch.randint(0, 3, (nnz,), generator=g, device=DEV, dtype=torch.int32),
                "coef": normal((3, H), g), "idx2": torch.randint(0, 64, (nnz,), generator=g, device=DEV,
                                                                 dtype=torch.int32),
                "B": normal((64, F), g), "Wl": normal((128, 128), g, scale=0.1)}

    def scall(st, rows, s, E):
        if e == "cogdl_b200_mhspmm_f32":
            return [_raw.mhspmm_raw(st, E(s["att"]), Xs.view(-1, H, F))]
        if e == "cogdl_b200_comp_aggr_f32":
            return [_raw.comp_aggr_raw(st, E(s["idx2"]), E(s["w"]), Xs, s["B"], "mult")]
        if e == "cogdl_b200_rgcn_aggr_f32":
            return [_raw.rgcn_aggr_raw(st, E(s["etype"]), E(s["w"]), s["coef"], Xs[:, :F].contiguous())]
        if e == "cogdl_b200_gcn_fused_f32":
            return [fused_gcn_raw(st, E(s["w"]), Xs, s["Wl"])]
        if e == "cogdl_b200_sage_fused_f32":
            return [_launch_sage(st, E(s["w"]), Xs, s["Wl"][:16].contiguous(), rows[0])]
        if e == "cogdl_b200_disen_route_fwd_f32":
            raise AssertionError("square: run_disen")
        raise AssertionError(e)

    rows = (lambda n, g: (normal((n, 16), g),)) if e == "cogdl_b200_sage_fused_f32" else (lambda n, g: ())
    twin_store(c, 89, rows, make_small, scall)
    RATIOS[c.id] = 0.0


def run_disen(c):
    """DisenGCN routing on a square structure of n just past 2^31 / F nodes: the band rows route over neighbours among
    the sampled rows, q and c are one [n, F] tensor (aliased inputs) and out is the other.  The twin's nodes are the
    sampled rows; only the band rows hold edges in both."""
    from cogdl_b200.operators._raw import disen_route_fwd_raw

    K = 3
    rng = np.random.default_rng(97)
    g = gen(97)
    S = np.array(c.samples)
    band = [r for r in S if r >= c.n_rows - LT.BAND or r == c.straddle]
    deg = np.zeros(c.n_rows, np.int64)
    for k, r in enumerate(band):
        deg[r] = LT.DEGREES[k % len(LT.DEGREES)]
    rp = np.concatenate([[0], np.cumsum(deg)])
    ci = rng.choice(S, rp[-1])
    qc = normal((c.n_rows, c.F), g)
    Sd = D(S)
    qc_t = qc[Sd].contiguous()
    out = disen_route_fwd_raw(structure(rp, ci, c.n_rows, c.plan), qc, qc, K, 0.8)[0]
    k_big = last_kernel()
    got = _np(out[Sd])
    del out, qc
    pos = {int(r): i for i, r in enumerate(S)}
    rp_t = np.concatenate([[0], np.cumsum(deg[S])])
    ci_t = np.concatenate([[pos[int(j)] for j in ci[rp[r]:rp[r + 1]]] for r in S] + [np.zeros(0)]).astype(np.int64)
    out_t = disen_route_fwd_raw(structure(rp_t, ci_t, S.size, c.plan), qc_t, qc_t, K, 0.8)[0]
    check_kernel(c, k_big, last_kernel())
    same_bits(got, _np(out_t), c.id)
    RATIOS[c.id] = 0.0


def run_edge_ops(c):
    """The entries whose large operand is edge-aligned, beyond the softmax and the GAT forward."""
    from cogdl_b200.operators import _raw

    e, H = c.entry, c.H
    if c.transpose:
        drop = e == "cogdl_b200_mhspmm_dropout_f32"

        def make_edge(nnz, g):
            a = torch.rand((nnz, H), generator=g, device=DEV)
            if drop:
                a[::3] = -a[::3]                           # the sign bit marks a dropped attention
            return (a,)

        def call(stT, perm, ev, rows):
            if e == "cogdl_b200_edge_colsum_f32":
                return [_raw.edge_colsum_raw(stT, perm, ev[0])]
            return [_raw.mhspmm_raw(stT, ev[0], rows[0], perm=perm, drop_scale=1.25 if drop else None)]

        twin_transpose(c, 101, make_edge, lambda n, g: (normal((n, H, c.F), g),), call)
        RATIOS[c.id] = 0.0
        return
    W = H

    def make_edge(nnz, g):
        if e in ("cogdl_b200_gat_attn_bwd_f32", "cogdl_b200_gat_attn_bwd_dropout_f32", "cogdl_b200_hgn_attn_bwd_f32"):
            a = torch.rand((nnz, W), generator=g, device=DEV)
            if "dropout" in e or "hgn" in e:
                a[1::3] = -a[1::3]
            return (a,)
        if e in ("cogdl_b200_softmax_aggr_fwd_f32", "cogdl_b200_genconv_edge_fwd_f32"):
            return (normal((nnz, W), g),)
        return ()

    def make_small(n, g):
        return {"hl": (normal((n, H), g), "row"), "hr": (normal((n, H), g, scale=4.0), "col"),
                "he": (normal((4, H), g), "none"), "feat": (normal((n, H, c.F), g), "col"),
                "grad": (normal((n, H, c.F), g), "row"), "X": (normal((n, 4), g), "col"),
                "Gr": (normal((n, W, 4), g), "row"), "w": (torch.rand(int(sum(LT.edge_degrees())), generator=g,
                                                                       device=DEV), "etype"),
                "etype": (torch.randint(0, 4, (int(sum(LT.edge_degrees())),), generator=g, device=DEV,
                                        dtype=torch.int32), "etype"),
                "W": (normal((4, W), g, scale=0.3), "none")}

    beta = torch.tensor([0.7], device=DEV)

    def call(st, ev, s):
        v = {k: t for k, (t, _) in s.items()}
        if e == "cogdl_b200_mhsddmm_f32":
            return [(_raw.mhsddmm_raw(st, v["grad"], v["feat"]), "edge")]
        if e in ("cogdl_b200_gat_attn_bwd_f32", "cogdl_b200_gat_attn_bwd_dropout_f32"):
            d_edge, g_row = _raw.gat_attn_bwd_raw(st, ev[0], ev[0], v["hl"], v["hr"], float(SLOPE),
                                                  drop_scale=1.25 if "dropout" in e else None)
            return [(d_edge, "edge"), (g_row, "row")]
        if e == "cogdl_b200_hgn_attn_f32":
            mix, att = _raw.hgn_attn_raw(st, v["etype"], v["hl"], v["hr"], v["he"], float(SLOPE), True)
            return [(mix, "edge"), (att, "edge")]
        if e == "cogdl_b200_hgn_attn_bwd_f32":
            d_edge, g_row = _raw.hgn_attn_bwd_raw(st, v["etype"], ev[0], ev[0], v["hl"], v["hr"], v["he"],
                                                  float(SLOPE), 0.75)
            return [(d_edge, "edge"), (g_row, "row")]
        if e == "cogdl_b200_softmax_aggr_fwd_f32":
            out = _raw.softmax_aggr_fwd_raw(st, v["X"][:, :1].repeat(1, W).contiguous() if False else
                                            v["X"].repeat(1, 2).contiguous(), beta, 1e-7, edge_term=ev[0],
                                            want_lse=True)
            return [(out[0], "row"), (out[1], "row")]
        if e == "cogdl_b200_genconv_edge_fwd_f32":
            out = _raw.genconv_edge_fwd_raw(st, v["X"], ev[0], v["W"], beta, 1e-7, want_lse=True)
            return [(out[0], "row"), (out[1], "row")]
        if e == "cogdl_b200_rgcn_edge_dot_f32":
            return [(_raw.rgcn_edge_dot_raw(st, v["w"], v["Gr"], v["X"]), "edge")]
        raise AssertionError(e)

    twin_edge(c, 103, make_edge, make_small, call)
    RATIOS[c.id] = 0.0


def run_actnn_packed(c):
    """The 8-bit unpack of a packed input of more than 2^32 bytes into a small output: D = 1 is padded to a 256-byte
    row, so row n starts at byte 256 n, computed in the kernel from n."""
    from cogdl_b200.actnn import kernels as K

    g = gen(107)
    N = c.n_rows
    x = normal((N, 1), g)
    packed, scale, mn = K.pack(x, 8, 256, False)
    out = K.unpack(packed, 8, scale, mn, N, 1, 256)
    k_big = last_kernel()
    S = D(np.array(c.samples))
    got = _np(out[S])
    p_t = packed.view(N, -1)[S].contiguous().view(-1)
    s_t, m_t = scale[S].contiguous(), mn[S].contiguous()
    del packed, out
    out_t = K.unpack(p_t, 8, s_t, m_t, S.numel(), 1, 256)
    check_kernel(c, k_big, last_kernel())
    same_bits(got, _np(out_t), c.id)
    from tests import actnn_ref as R

    codes = _np(p_t).reshape(S.numel(), -1)
    assert np.array_equal(got, R.dequantize(codes, _np(s_t.float()), _np(m_t.float()), 1, 256)), c.id
    RATIOS[c.id] = 0.0


OLD_EDGE = ("cogdl_b200_edge_softmax_fwd_f32", "cogdl_b200_edge_softmax_bwd_f32", "cogdl_b200_gat_fwd_f32",
            "cogdl_b200_gat_fwd_dropout_f32", "cogdl_b200_gather_rows_f32")
SPMM_FORMS = ("cogdl_b200_spmm_csr_f32", "cogdl_b200_spmm_csr_f32_2src", "cogdl_b200_spmm_csr_f32_peers")


def run(c):
    if c.role == "packed":
        return run_actnn_packed(c)
    if c.role == "elements":
        return run_actnn(c)
    if c.role == "edge":
        return run_edge(c) if c.entry in OLD_EDGE else run_edge_ops(c)
    if c.role == "partials":
        return run_spmm_partials(c)
    if c.entry in SPMM_FORMS:
        return run_spmm_forms(c)
    if c.entry == "cogdl_b200_disen_route_fwd_f32":
        return run_disen(c)
    if not c.entry.startswith("cogdl_b200_spmm") and c.entry not in (
            "cogdl_b200_sddmm_csr_f32", "cogdl_b200_scatter_max_fwd_f32", "cogdl_b200_scatter_max_bwd_f32",
            "cogdl_b200_label_prop_f32"):
        return run_message(c)
    if c.entry == "cogdl_b200_sddmm_csr_f32":
        return run_sddmm(c)
    if c.entry == "cogdl_b200_scatter_max_fwd_f32":
        return run_scatter_max(c)
    if c.entry == "cogdl_b200_scatter_max_bwd_f32":
        return run_scatter_max_bwd(c)
    return run_spmm_gather(c) if c.role == "gather" else run_spmm_store(c)


@pytest.fixture(scope="module")
def report():
    free, total = torch.cuda.mem_get_info()
    print(f"\n{torch.cuda.get_device_name(0)}: {free / LT.GIB:.1f} of {total / LT.GIB:.1f} GiB free; largest row "
          f"{LT.LARGEST.id}, {LT.LARGEST.bytes_needed / 1e9:.1f} GB")
    yield
    for k, v in sorted(RATIOS.items()):
        print(f"  worst error / bound  {k:40s} {v:.3g}")


@pytest.mark.parametrize("c", LT.TABLE, ids=lambda c: c.id)
def test_large_offset_row(report, c):
    import cogdl_b200

    assert cogdl_b200._cabi.load().cogdl_b200_check_device() == 0
    need(c)
    assert c.crossing_elems > c.limit
    try:
        run(c)
    except BaseException as exc:
        # a failing row's frames would keep its multi-GB tensors alive through the traceback
        traceback.clear_frames(exc.__traceback__)
        raise

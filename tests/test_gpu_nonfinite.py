"""Every row of tests/nonfinite_table.py under every plan form of PLAN_FORMS (and the fp32 SpMM under forced panel
counts), against the fp64 composition of the same formula on the same fp32 inputs.

The rule, unless a family's reference says otherwise: NaN exactly where the fp64 reference is NaN, +-Inf exactly where
it is +-Inf with the same sign, every finite element within the family's bound, and the hub plan's arrival counters
back at zero after the call.  The documented exceptions (DESIGN.md, "Non-finite operands"):
  scatter_max   the running max starts at -inf and takes a value only when `max < value`, so a NaN is never selected
  fused layers  an aggregated +-Inf goes through the bf16x3 split whole, and its products with W's split terms may
                cancel (Inf - Inf): the output is non-finite exactly where fp64 is, NaN wherever fp64 is NaN
Finite elements are held to the bounds the finite suites derive (u = 2^-24): the sum of d fp32 terms within
(d + 2) u sum|term|; the softmax forms within the bounds of tests/test_gpu_dispatch.py and
tests/test_gpu_dispatch_message.py, loosened to 2^-12 relative for the GENConv edge encoder, whose edge term is formed
in a different order.  The fused layers' finite elements within 2^-15 of the magnitude of their terms: their precision
is held to the tighter split-product bound by tests/test_gpu_dispatch_message.py.

A GradScaler test runs GCN (fused and unfused), GAT, GraphSAGE-max and a GENConv aggregation end to end with a NaN in one
row of the incoming gradient: the library's backward must carry it to the input gradient of that row's neighbours, and
the scaler must find it, skip the step and leave every parameter bit-identical.
"""
import numpy as np
import pytest
import torch

import oracle
from tests.gpu_util import T, check_counters, dev, plan_structure
from tests.graphs import boundary_csr, case
from tests.nonfinite_table import PANEL_F, PLAN_FORMS, SPMM_PANELS, TABLE
from tests.test_gpu_dispatch import softmax64
from tests.test_gpu_dispatch_message import EPS, LN2, LOG2E, seg_reduce

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
TINY = float(np.finfo(np.float32).tiny)
BF16_OVERFLOW = float.fromhex("0x1.fefp127")     # the smallest fp32 that rounds to a bf16 infinity


def graph_of(c, chunk):
    return boundary_csr(chunk or 16) if c.graph == "bounds" else case(c.graph)


def structure(rp, ci, n_cols, dev, form):
    _, chunk, seg_cost = form
    return plan_structure(rp, ci, n_cols, dev, chunk=chunk, seg_cost=seg_cost)


def check_hub_plan(st, what):
    """A planned structure has hub chunks, and the call left their arrival counters at zero."""
    if st.chunk_edges > 0:
        assert st.plan.n_chunks > 0, f"{what}: the graph should have hub rows at chunk {st.chunk_edges}"
    check_counters(st, what)


def rows_of(rp):
    return np.repeat(np.arange(rp.size - 1), np.diff(rp))


def check(got, ref, bound, what, nan_superset=False):
    """NaN and +-Inf exactly where the reference has them (with nan_superset: non-finite exactly where the reference
    is, NaN at least where it is), finite elements within the bound.  The reference must hold both a NaN and an
    infinity or a NaN, so the case is not vacuous."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert (~np.isfinite(ref)).any(), f"{what}: the reference has no non-finite element"
    fin = np.isfinite(ref)
    if nan_superset:
        bad = np.isfinite(got) != fin
        assert not bad.any(), f"{what}: finite mask differs at {np.argwhere(bad)[:4].tolist()}"
        bad = np.isnan(ref) & ~np.isnan(got)
        assert not bad.any(), f"{what}: NaN lost at {np.argwhere(bad)[:4].tolist()}, got {got[bad][:4]}"
    else:
        bad = np.isnan(got) != np.isnan(ref)
        assert not bad.any(), (f"{what}: NaN mask differs at {np.argwhere(bad)[:4].tolist()}: got {got[bad][:4]}, "
                               f"ref {ref[bad][:4]} ({int(np.isnan(got).sum())} NaN, reference {int(np.isnan(ref).sum())})")
        bad = (np.isposinf(got) != np.isposinf(ref)) | (np.isneginf(got) != np.isneginf(ref))
        assert not bad.any(), (f"{what}: Inf mask differs at {np.argwhere(bad)[:4].tolist()}: got {got[bad][:4]}, "
                               f"ref {ref[bad][:4]}")
    err = np.abs(got[fin] - ref[fin])
    b = np.broadcast_to(bound, ref.shape)[fin]
    out = ~(err <= b)
    assert not out.any(), (f"{what}: {int(out.sum())} finite elements outside the bound, first got {got[fin][out][0]!r},"
                           f" ref {ref[fin][out][0]!r}, bound {b[out][0]!r}")


def sites(rp):
    """Edges where the values go: the first, a middle and the last edge (so the first, a middle and the last chunk)
    of the largest hub, the edge of a one-edge row, and an edge of a short row (which the default plan streams)."""
    deg = np.diff(rp)
    hub = int(np.argmax(deg))
    one = int(np.nonzero(deg == 1)[0][0])
    short = int(np.nonzero((deg > 3) & (deg < 16))[0][0])
    return {"first": int(rp[hub]), "middle": int(rp[hub] + deg[hub] // 2), "last": int(rp[hub + 1] - 1),
            "one": int(rp[one]), "short": int(rp[short] + 1), "zero": int(rp[short])}


def plant_features(X, ci, s):
    """NaN, +Inf and -Inf in feature columns 0 (first), F - 1 (the F % 4 tail) and a middle one of the source rows the
    chosen edges read; +Inf in column 1 of the source row of the edge "zero" (the callers give it weight 0)."""
    F = X.shape[-1]
    X[ci[s["first"]], ..., 0] = np.nan
    X[ci[s["middle"]], ..., F - 1] = np.inf
    X[ci[s["last"]], ..., F // 2] = -np.inf
    X[ci[s["one"]], ..., F - 1] = np.nan
    X[ci[s["short"]], ..., 0] = -np.inf
    X[ci[s["zero"]], ..., 1] = np.inf


def spmm64(rp, ci, w, X):
    rows = rows_of(rp)
    with np.errstate(invalid="ignore", over="ignore"):
        prod = w.astype(np.float64)[:, None] * X.astype(np.float64)[ci]
        ref = np.zeros((rp.size - 1, X.shape[1]))
        mag = np.zeros_like(ref)
        np.add.at(ref, rows, prod)
        np.add.at(mag, rows, np.abs(prod))
    deg = np.diff(rp)[:, None]
    return ref, (deg + 2) * U32 * np.where(np.isfinite(mag), mag, 0) + TINY


# ------------------------------------------------------------------------------------------ runners
def run_spmm(dev, c, form):
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(1)
    s = sites(rp)
    panel_sets = [(c.F, 0)] + ([(PANEL_F, p) for p in SPMM_PANELS] if form[0].startswith("default") and
                               c.operand == "features" else [])
    split = np.diff(rp) > form[1] if form[1] > 0 else np.zeros(rp.size - 1, bool)
    by_panels = {}
    for F, panels in panel_sets:
        rng = np.random.default_rng(1)
        X = rng.standard_normal((n, F)).astype(np.float32)
        w = rng.uniform(0.25, 2.0, ci.size).astype(np.float32)
        if c.operand == "features":
            plant_features(X, ci, s)
            w[s["zero"]] = 0.0
        else:
            w[s["first"]], w[s["middle"]], w[s["last"]], w[s["one"]] = np.nan, np.inf, -np.inf, np.nan
        st = structure(rp, ci, n, dev, form)
        got = spmm_raw(st, T(w, dev), T(X, dev), panels=panels).cpu().numpy()
        ref, bound = spmm64(rp, ci, w, X)
        check(got, ref, bound, f"{c.id} {form[0]} F={F} panels={panels}")
        check_hub_plan(st, c.id)
        # rows the plan does not split: equal to the oracle's CSR-order fp32 sum (NaN where it is NaN)
        want = oracle.spmm_csr(rp, ci, w, X)
        assert np.array_equal(got[~split], want[~split], equal_nan=True), \
            f"{c.id} {form[0]} F={F} panels={panels}: unsplit rows differ from the oracle"
        if F == PANEL_F:
            by_panels[panels] = got
    for panels, got in by_panels.items():              # whatever the panel count: bitwise the single-pass result
        assert np.array_equal(got.view(np.uint32), by_panels[1].view(np.uint32)), \
            f"{c.id} {form[0]}: panels={panels} differs bitwise from panels=1"


def run_spmm_f16(dev, c, form):
    """Row sums past 65504 become +-Inf in the fp16 output; a NaN feature stays NaN."""
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(2)
    s = sites(rp)
    X = rng.uniform(-1, 1, (n, c.F)).astype(np.float16)
    X[:, 2] = 60000.0                             # every row with two or more unit-weight edges overflows column 2
    X[:, 3] = -40000.0
    X[ci[s["first"]], 0] = np.nan
    w = np.ones(ci.size, np.float16)
    st = structure(rp, ci, n, dev, form)
    got = spmm_raw(st, T(w, dev), T(X, dev)).cpu().numpy().astype(np.float64)
    ref, _ = spmm64(rp, ci, w.astype(np.float32), X.astype(np.float32))
    mag = np.zeros_like(ref)
    np.add.at(mag, rows_of(rp), np.abs(X.astype(np.float64)[ci]))
    with np.errstate(over="ignore"):
        ref16 = ref.astype(np.float16).astype(np.float64)
    deg = np.diff(rp)[:, None]
    check(got, ref16, 2.0 ** -11 * np.abs(ref) + deg * U32 * mag + 2.0 ** -24, f"{c.id} {form[0]}")
    assert np.isinf(got[:, 2]).any() and np.isinf(got[:, 3]).any()
    check_hub_plan(st, c.id)


def run_residual(dev, c, form):
    """y = a (A x) + b z with NaN / +-Inf in z: each stays in its own element, with b's sign."""
    from cogdl_b200.operators._raw import spmm_residual_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(3)
    X = rng.standard_normal((n, c.F)).astype(np.float32)
    w = rng.uniform(0.25, 2.0, ci.size).astype(np.float32)
    Z = rng.standard_normal((n, c.F)).astype(np.float32)
    Z[0, 0], Z[n // 2, c.F - 1], Z[n - 1, c.F // 2], Z[int(np.argmax(np.diff(rp))), 1] = np.nan, np.inf, -np.inf, np.nan
    st = structure(rp, ci, n, dev, form)
    for a, b in ((0.75, 0.5), (1.0, -2.0)):
        got = spmm_residual_raw(st, T(w, dev), T(X, dev), T(Z, dev), a, b).cpu().numpy()
        agg, bound = spmm64(rp, ci, w, X)
        with np.errstate(invalid="ignore"):
            ref = a * agg + b * Z.astype(np.float64)
        check(got, ref, a * bound + 2 * U32 * (np.abs(a * agg) + np.abs(b * np.nan_to_num(Z, posinf=0, neginf=0))),
              f"{c.id} {form[0]} a={a} b={b}")
    check_hub_plan(st, c.id)


def run_sddmm(dev, c, form):
    from cogdl_b200.operators._raw import sddmm_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(4)
    s = sites(rp)
    d1 = rng.standard_normal((n, c.F)).astype(np.float32)
    d2 = rng.standard_normal((n, c.F)).astype(np.float32)
    plant_features(d2, ci, s)
    d1[rows_of(rp)[s["zero"]], 1] = 0.0
    st = structure(rp, ci, n, dev, form)
    got = sddmm_raw(st, T(d1, dev), T(d2, dev)).cpu().numpy()
    with np.errstate(invalid="ignore"):
        p = d1.astype(np.float64)[rows_of(rp)] * d2.astype(np.float64)[ci]
    ref = p.sum(1)
    check(got, ref, (c.F + 2) * U32 * np.abs(np.where(np.isfinite(p), p, 0)).sum(1) + TINY, f"{c.id} {form[0]}")


def run_mhspmm(dev, c, form):
    from cogdl_b200.operators._raw import mhspmm_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(5)
    s = sites(rp)
    att = rng.uniform(0, 1, (ci.size, c.H)).astype(np.float32)
    feat = rng.standard_normal((n, c.H, c.F)).astype(np.float32)
    att[s["first"], 0], att[s["middle"], 1], att[s["last"], c.H - 1], att[s["one"], 2] = np.nan, np.inf, -np.inf, np.nan
    att[s["zero"], 3] = 0.0
    feat[ci[s["zero"]], 3, c.F - 1] = np.inf
    st = structure(rp, ci, n, dev, form)
    got = mhspmm_raw(st, T(att, dev), T(feat, dev)).cpu().numpy()
    for h in range(c.H):
        ref, bound = spmm64(rp, ci, att[:, h], feat[:, h, :])
        check(got[:, h], ref, bound, f"{c.id} {form[0]} head {h}")
    check_hub_plan(st, c.id)


def run_scatter_max(dev, c, form):
    """A NaN is never the max (strict `<` from -inf): the result and argmax equal the oracle's, +-Inf included."""
    from cogdl_b200.operators._raw import scatter_max_fwd_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(6)
    X = np.round(rng.standard_normal((n, c.F)) * 4).astype(np.float32) / 4
    plant_features(X, ci, sites(rp))
    hub = int(np.argmax(np.diff(rp)))
    X[ci[rp[hub]:rp[hub + 1]], 2] = np.nan        # a whole hub row of NaN in one column: its max stays -inf
    st = structure(rp, ci, n, dev, form)
    out, arg = scatter_max_fwd_raw(st, T(X, dev))
    ref, ref_id = oracle.scatter_max_fwd(rp, ci, X)
    assert not np.isnan(ref).any() and np.isinf(ref).any()
    assert np.array_equal(out.cpu().numpy(), ref), f"{c.id} {form[0]}: max differs"
    assert np.array_equal(arg.cpu().numpy(), ref_id), f"{c.id} {form[0]}: argmax differs"
    check_hub_plan(st, c.id)


def run_edge_softmax(dev, c, form):
    """A whole (row, head) of NaN, a NaN and a +Inf logit in chunks of the largest hub, a +Inf logit in a one-edge row
    and in a short row: fp64 gives NaN over each of those (row, head)s, as torch.softmax does."""
    from cogdl_b200.operators._raw import edge_softmax_fwd_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(7)
    s = sites(rp)
    x = (rng.standard_normal((ci.size, c.H)) * 2).astype(np.float32)
    deg = np.diff(rp)
    r7 = int(np.nonzero(deg == 7)[0][0])
    x[rp[r7]:rp[r7 + 1], c.H - 1] = np.nan
    x[s["first"], 0] = np.nan
    x[s["last"], c.H - 1] = np.inf
    x[s["one"], 0] = np.inf
    x[s["short"], 0] = np.inf
    x[s["middle"], c.H // 2] = -np.inf
    st = structure(rp, ci, n, dev, form)
    got = edge_softmax_fwd_raw(st, T(x, dev)).cpu().numpy().astype(np.float64)
    with np.errstate(invalid="ignore"):
        y, t, Tm, d = softmax64(rp, x)
    check(got, y, y * ((d + 3) * 2.0 ** -22 + d * U32 + (2 * t + 2 * Tm) * 2.0 ** -23) + 2.0 ** -126,
          f"{c.id} {form[0]}")
    check_hub_plan(st, c.id)


def sa64(rp, ci, x, A, beta):
    """fp64 GENConv softmax aggregation of m = relu(x[col] + A) + eps with torch's ReLU (a NaN passes), and the
    forward bound of tests/test_gpu_dispatch_message.py for the finite elements."""
    with np.errstate(invalid="ignore", over="ignore"):
        pre = x[ci] if A is None else (x[ci] + A).astype(np.float32)
        m = (np.where(pre < 0, np.float32(0), pre) + np.float32(EPS)).astype(np.float32)
        rows = rows_of(rp)
        t = beta * m.astype(np.float64)
        mx = seg_reduce(np.maximum, t, rp, fill=0.0)
        mn = seg_reduce(np.minimum, t, rp, fill=0.0)
        ex = np.exp(t - mx[rows])
        S = seg_reduce(np.add, ex, rp)
        out = seg_reduce(np.add, ex / S[rows] * m, rp)
        deg = np.diff(rp).astype(np.float64)[:, None]
        Z = seg_reduce(np.maximum, np.abs(t), rp) * LOG2E
        E = (deg + 3) * 2.0 ** -22 + deg * U32 + LN2 * U32 * (6 * Z + 2 * (mx - mn) * LOG2E)
        bound = np.abs(out) * (2 * E + (2 * deg + 1) * U32) + TINY
    return out, np.where(np.isfinite(bound), bound, 0)


def sa_inputs(c, rp, ci, n, rng, edge_term):
    s = sites(rp)
    x = rng.uniform(-1, 3, (n, c.F)).astype(np.float32)
    A = (rng.standard_normal((ci.size, c.F))).astype(np.float32) if edge_term else None
    if edge_term:
        A[s["first"], 0], A[s["middle"], c.F - 1], A[s["last"], c.F // 2], A[s["one"], 1] = np.nan, np.inf, -np.inf, np.nan
    else:
        plant_features(x, ci, s)
    return x, A


def run_softmax_aggr(dev, c, form):
    from cogdl_b200.operators._raw import softmax_aggr_fwd_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(8)
    x, A = sa_inputs(c, rp, ci, n, rng, c.operand == "edge term")
    st = structure(rp, ci, n, dev, form)
    for beta in (1.0, 0.0):
        beta_d = torch.tensor([beta], dtype=torch.float32, device=dev)
        out, _, _ = softmax_aggr_fwd_raw(st, T(x, dev), beta_d, EPS, None if A is None else T(A, dev))
        ref, bound = sa64(rp, ci, x, A, beta)
        check(out.cpu().numpy(), ref, bound, f"{c.id} {form[0]} beta={beta}")
    check_hub_plan(st, c.id)


def run_genconv_edge(dev, c, form):
    from cogdl_b200.operators._raw import genconv_edge_fwd_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(9)
    x, _ = sa_inputs(c, rp, ci, n, rng, False)
    attr = rng.standard_normal((ci.size, 5)).astype(np.float32)
    W = (rng.standard_normal((c.F, 5)) / 3).astype(np.float32)
    st = structure(rp, ci, n, dev, form)
    beta_d = torch.tensor([1.0], dtype=torch.float32, device=dev)
    out, _, _ = genconv_edge_fwd_raw(st, T(x, dev), T(attr, dev), T(W, dev), beta_d, EPS)
    A = (attr.astype(np.float64) @ W.astype(np.float64).T).astype(np.float32)
    ref, bound = sa64(rp, ci, x, A, 1.0)
    check(out.cpu().numpy(), ref, bound + 2.0 ** -12 * np.abs(np.nan_to_num(ref)), f"{c.id} {form[0]}")
    check_hub_plan(st, c.id)


def run_fused(dev, c, form):
    if c.operand == "overflow":
        fused_case(dev, c, form, True)
    elif c.name.startswith("sage_fused-max"):
        # a (row, column) whose neighbours are all NaN keeps the max's -inf: an aggregated Inf, so no ReLU case
        fused_case(dev, c, form, False)
    else:
        fused_case(dev, c, form, True)       # NaN only: every output of a row with a NaN aggregated value is NaN
        fused_case(dev, c, form, False)      # +-Inf too, without the ReLU (relu(-Inf) = 0 hides the Inf - Inf)


def fused_case(dev, c, form, relu):
    """The aggregated rows A32 come from spmm_raw (the fused kernel's aggregation is bit-identical to it); the reference
    is fp64(A32) fp64(W)^T plus the epilogue, with torch's ReLU.  The overflow row puts a finite 0x1.fffp127 in one
    feature column (above the bf16 overflow threshold) with W's entries below 1/2 in magnitude, so fp64 gives finite
    outputs near it; the features row plants NaN (with the ReLU) or NaN and +-Inf (without) as the other families
    do."""
    from cogdl_b200.operators._raw import scatter_max_fwd_raw, spmm_raw
    from cogdl_b200.operators.fused_gcn import fused_gcn_raw
    from cogdl_b200.operators.fused_sage import fused_sage_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(10)
    K, Fout = 128, 40
    X = rng.standard_normal((n, K)).astype(np.float32)
    sage = c.entry == "cogdl_b200_sage_fused_f32"
    W = (rng.uniform(-0.45, 0.45, (Fout, 2 * K if sage else K))).astype(np.float32)
    b = rng.standard_normal(Fout).astype(np.float32)
    s = sites(rp)
    if c.operand == "overflow":
        # one source row, read by one-edge rows only (so each aggregated value is the feature times its weight)
        one = np.nonzero(np.diff(rp) == 1)[0]
        src = int(ci[rp[one[0]]])
        ci = ci.copy()
        ci[ci == src] = (src + 1) % n
        ci[rp[one[:5]]] = src
        X[src, 5] = float.fromhex("0x1.fffp127")
        w = np.ones(ci.size, np.float32)
    else:
        plant_features(X, ci, s)
        w = rng.uniform(0.25, 2.0, ci.size).astype(np.float32)
        w[s["zero"]] = 0.0
        if relu:
            X[~np.isnan(X)] = np.nan_to_num(X[~np.isnan(X)], posinf=1.0, neginf=-1.0)
    st = structure(rp, ci, n, dev, form)
    Xd, Wd, bd = T(X, dev), T(W, dev), T(b, dev)
    if sage:
        aggr = c.name.split("-")[1]
        rs = None
        if aggr == "max":
            A32 = scatter_max_fwd_raw(st, Xd)[0]
        else:
            A32 = spmm_raw(st, None, Xd)
            if aggr == "mean":
                rs = (1.0 / torch.diff(st.rowptr).clamp_min(1).float()).contiguous()
                A32 = rs[:, None] * A32              # the kernel's one rounding of row_scale * (A.x)
        A32 = A32.cpu().numpy().astype(np.float64)
        got = fused_sage_raw(st, None, rs, Xd, Wd, bd, "max" if aggr == "max" else "sum", relu).cpu().numpy()
        Wn, Ws = W[:, K:].astype(np.float64), W[:, :K].astype(np.float64)
        with np.errstate(invalid="ignore", over="ignore"):
            selfp = X[:n].astype(np.float64) @ Ws.T + b
            ref = selfp + A32 @ Wn.T
            mag = np.abs(X[:n].astype(np.float64)) @ np.abs(Ws).T + np.abs(b) + np.abs(A32) @ np.abs(Wn).T
    else:
        A32 = spmm_raw(st, T(w, dev), Xd).cpu().numpy().astype(np.float64)
        got = fused_gcn_raw(st, T(w, dev), Xd, Wd, bd, relu).cpu().numpy()
        rsum = seg_reduce(np.add, w.astype(np.float64), rp)
        with np.errstate(invalid="ignore", over="ignore"):
            ref = A32 @ W.astype(np.float64).T + rsum[:, None] * b
            mag = np.abs(A32) @ np.abs(W.astype(np.float64)).T + np.abs(rsum[:, None] * b)
    with np.errstate(invalid="ignore"):
        if relu:
            ref = np.where(ref < 0, 0.0, ref)              # torch.relu: a NaN passes
        ref = np.where(np.abs(ref) > np.finfo(np.float32).max, np.sign(ref) * np.inf, ref)
    if relu:
        assert not np.isinf(A32).any(), f"{c.id}: the ReLU case must not aggregate an Inf"
    if c.operand == "overflow":
        assert np.abs(A32).max() > BF16_OVERFLOW and np.isfinite(A32).all()
        assert np.isfinite(ref).all()
        g = np.asarray(got, np.float64)
        assert np.isfinite(g).all(), f"{c.id} {form[0]}: non-finite at {np.argwhere(~np.isfinite(g))[:4].tolist()}"
        bad = ~(np.abs(g - ref) <= 2.0 ** -15 * mag + TINY)
        assert not bad.any(), f"{c.id} {form[0]}: {int(bad.sum())} elements outside the bound"
    else:
        check(got, ref, 2.0 ** -15 * np.where(np.isfinite(mag), mag, 0) + TINY, f"{c.id} {form[0]} relu={relu}",
              nan_superset=not relu)
    check_hub_plan(st, c.id)


RUN = {
    "cogdl_b200_spmm_csr_f32_ex": run_spmm,
    "cogdl_b200_spmm_csr_f16": run_spmm_f16,
    "cogdl_b200_spmm_residual_f32": run_residual,
    "cogdl_b200_sddmm_csr_f32": run_sddmm,
    "cogdl_b200_mhspmm_f32": run_mhspmm,
    "cogdl_b200_scatter_max_fwd_f32": run_scatter_max,
    "cogdl_b200_edge_softmax_fwd_f32": run_edge_softmax,
    "cogdl_b200_softmax_aggr_fwd_f32": run_softmax_aggr,
    "cogdl_b200_genconv_edge_fwd_f32": run_genconv_edge,
    "cogdl_b200_gcn_fused_f32": run_fused,
    "cogdl_b200_sage_fused_f32": run_fused,
}


FUSED = ("cogdl_b200_gcn_fused_f32", "cogdl_b200_sage_fused_f32")     # run on the default plan only (row-stream form)


def cases():
    for c in TABLE:
        for form in PLAN_FORMS:
            if c.entry in FUSED and not form[0].startswith("default"):
                continue
            yield pytest.param(c, form, id=f"{c.id}-{form[0]}")


@pytest.mark.parametrize("c,form", list(cases()))
def test_nonfinite_row(dev, c, form):
    RUN[c.entry](dev, c, form)


# ------------------------------------------------------------------------------------------ GradScaler end to end
SCALER_LAYERS = ["gcn", "gcn-fused", "gat", "sage-max", "genconv"]


class GENConvAggr(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(128, 64)
        self.beta = torch.nn.Parameter(torch.tensor(1.0))

    def forward(self, graph, x):
        from cogdl_b200.operators.softmax_aggr import genconv_aggregate

        return genconv_aggregate(graph, self.lin(x), "softmax_sg", beta=self.beta)


@pytest.mark.parametrize("kind", SCALER_LAYERS)
def test_grad_scaler_skips_a_non_finite_step(dev, kind):
    """A NaN in one row i of the incoming gradient (the 700-edge hub of two_hubs), every other element finite and the
    scale small enough (2^8) that nothing overflows.  The library's backward kernels must carry the NaN to the input
    gradient of i's neighbours (for max aggregation: of the neighbours the max selected), and the scaler must find it,
    skip the step, back the scale off and leave every parameter bit-identical."""
    from cogdl_b200.operators.scatter_max import scatter_max_with_argmax
    from tests.test_gpu_autograd import graph_np, layer_graphs, make_layer

    graphs, n = layer_graphs("two_hubs", dev)
    g = graphs[1]
    rp, ci, _ = graph_np("two_hubs")
    hub = int(np.argmax(np.diff(rp)))
    if kind.startswith("gcn"):
        g.sym_norm()
    layer = (GENConvAggr() if kind == "genconv" else make_layer(kind)).to(dev)
    before = [p.detach().clone() for p in layer.parameters()]
    opt = torch.optim.SGD(layer.parameters(), lr=0.1)
    scale = 2.0 ** 8
    scaler = torch.amp.GradScaler("cuda", init_scale=scale)
    x = torch.randn(n, 128, generator=torch.Generator().manual_seed(9)).to(dev).requires_grad_(True)
    out = layer(g, x)
    G = torch.randn(out.shape, generator=torch.Generator().manual_seed(10)).to(dev)
    G[hub] = float("nan")
    scaler.scale((out * G).sum()).backward()
    if kind == "sage-max":
        _, arg = scatter_max_with_argmax(graphs[1].structure(), None, x.detach())
        reach = set(arg[hub].cpu().numpy().tolist()) - {-1}
    elif kind.startswith("gcn") and g.is_symmetric():
        # a graph flagged symmetric runs its backward over A itself: the rows that have the hub as a neighbour
        reach = set(rows_of(rp)[ci == hub].tolist())
    else:
        reach = set(ci[rp[hub]:rp[hub + 1]].tolist())
    reach = sorted(reach - {hub})
    assert reach
    ok = torch.isfinite(x.grad[reach]).all(dim=1).cpu().numpy()
    assert not ok.any(), f"{kind}: input-gradient rows {np.array(reach)[ok][:4].tolist()} lost the NaN"
    near = set(ci[rp[hub]:rp[hub + 1]].tolist()) | set(rows_of(rp)[ci == hub].tolist())
    far = sorted(set(range(n)) - near - {hub})
    assert torch.isfinite(x.grad[far]).any(), f"{kind}: the NaN spread to every row"
    scaler.step(opt)
    scaler.update()
    assert scaler.get_scale() < scale, f"{kind}: the scaler did not find the NaN"
    for i, (p, q) in enumerate(zip(before, layer.parameters())):
        assert torch.equal(p.reshape(-1).view(torch.int8), q.detach().reshape(-1).view(torch.int8)), \
            f"{kind}: parameter {i} changed"

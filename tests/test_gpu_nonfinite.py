"""Every row of tests/nonfinite_table.py under every plan form of PLAN_FORMS (and the fp32 SpMM under forced panel
counts), against the fp64 composition of the same formula on the same fp32 inputs.

The rule, unless a family's reference says otherwise: NaN exactly where the fp64 reference is NaN, +-Inf exactly where
it is +-Inf with the same sign, every finite element within the family's bound, and the hub plan's arrival counters
back at zero after the call.  The documented exceptions (DESIGN.md, "Non-finite operands"):
  scatter_max   the running max starts at -inf and takes a value only when `max < value`, so a NaN is never selected
  fused layers  an aggregated +-Inf goes through the bf16x3 split whole, and its products with W's split terms may
                cancel (Inf - Inf): the output is non-finite exactly where fp64 is, NaN wherever fp64 is NaN
The overflow rows of GENConv and DisenGCN compare with the fp64 softmax of the kernel's fp32 logits, which are +-Inf
where the fp32 product overflows (an fp64 logit would not).  Backward rows over the transpose run under the
transpose's plan at the same form.
Finite elements are held to the bounds the finite suites derive (u = 2^-24): the sum of d fp32 terms within
(d + 2) u sum|term|; the softmax forms within the bounds of tests/test_gpu_dispatch.py and
tests/test_gpu_dispatch_message.py, loosened to 2^-12 relative for the GENConv edge encoder, whose edge term is formed
in a different order.  The fused layers' finite elements within 2^-15 of the magnitude of their terms: their precision
is held to the tighter split-product bound by tests/test_gpu_dispatch_message.py.

A GradScaler test runs GCN (fused and unfused), GAT (also with attention dropout), GraphSAGE-max, GENConv, DisenGCN,
CompGCN, R-GCN, Simple-HGN, GIN with a learnable eps and a GTN-style spspmm layer end to end with a NaN in one row of
the incoming gradient: the library's backward must carry it to the input gradient of that row's neighbours, and
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
from tests.test_gpu_dispatch_message import EPS, LN2, LOG2E, col_sum, seg_reduce

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


def sa64(rp, ci, x, A, beta, fp32_logits=False):
    """fp64 GENConv softmax aggregation of m = relu(x[col] + A) + eps with torch's ReLU (a NaN passes), and the
    forward bound of tests/test_gpu_dispatch_message.py for the finite elements.  fp32_logits: the softmax runs over
    the kernel's fp32 base-2 logits fl(m fl(beta log2 e)), which are -Inf where beta m passes the fp32 range (an fp64
    logit would not overflow); the bound then takes the logit range and magnitude over the finite logits only."""
    with np.errstate(invalid="ignore", over="ignore"):
        pre = x[ci] if A is None else (x[ci] + A).astype(np.float32)
        m = (np.where(pre < 0, np.float32(0), pre) + np.float32(EPS)).astype(np.float32)
        rows = rows_of(rp)
        if fp32_logits:
            t = (m * (np.float32(beta) * np.float32(LOG2E))).astype(np.float64) * LN2
        else:
            t = beta * m.astype(np.float64)
        tf = np.where(np.isfinite(t), t, np.nan)
        mx = seg_reduce(np.maximum, t, rp, fill=0.0)
        ex = np.exp(t - mx[rows])
        S = seg_reduce(np.add, ex, rp)
        out = seg_reduce(np.add, ex / S[rows] * m, rp)
        deg = np.diff(rp).astype(np.float64)[:, None]
        Z = np.nan_to_num(seg_reduce(np.fmax, np.abs(tf), rp)) * LOG2E
        R = np.nan_to_num(seg_reduce(np.fmax, tf, rp) - seg_reduce(np.fmin, tf, rp)) * LOG2E
        E = (deg + 3) * 2.0 ** -22 + deg * U32 + LN2 * U32 * (6 * Z + 2 * R)
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


def sa_overflow_inputs(c, rp, ci, n, rng, chunk):
    """x in [-1, 3] and, in one column each, 1.5e38 (so the logit beta m log2 e is -Inf for beta = -2, while beta m
    stays finite) at the source of the first
    edge of the largest hub's first and second chunks, of a streamed short row and of a one-edge row, and at every
    source of a degree-7 row (whose logits are then all -Inf: NaN, as in the softmax)."""
    s = sites(rp)
    x = rng.uniform(-1, 3, (n, c.F)).astype(np.float32)
    deg = np.diff(rp)
    hub = int(np.argmax(deg))
    r7 = int(np.nonzero(deg == 7)[0][0])
    big = np.float32(1.5e38)
    for e, col in ((s["first"], 0), (rp[hub] + chunk, c.F - 1), (s["zero"], c.F // 2), (s["one"], 1)):
        x[ci[e], col] = big
    x[ci[rp[r7]:rp[r7 + 1]], 2] = big
    return x


def run_softmax_aggr(dev, c, form):
    """beta = 1 and 0; the overflow row at beta = -2, against the fp64 softmax of the kernel's fp32 logits: a -Inf
    logit has weight 0 wherever it falls in its row or chunk, and a row of nothing but -Inf logits is NaN."""
    from cogdl_b200.operators._raw import softmax_aggr_fwd_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(8)
    st = structure(rp, ci, n, dev, form)
    if c.operand == "overflow":
        x = sa_overflow_inputs(c, rp, ci, n, rng, form[1] or 16)
        beta_d = torch.tensor([-2.0], dtype=torch.float32, device=dev)
        out, _, _ = softmax_aggr_fwd_raw(st, T(x, dev), beta_d, EPS)
        ref, bound = sa64(rp, ci, x, None, -2.0, fp32_logits=True)
        assert np.isfinite(ref[int(np.argmax(np.diff(rp)))]).all(), "the hub row's reference should stay finite"
        check(out.cpu().numpy(), ref, bound, f"{c.id} {form[0]} beta=-2")
        check_hub_plan(st, c.id)
        return
    x, A = sa_inputs(c, rp, ci, n, rng, c.operand == "edge term")
    for beta in (1.0, 0.0):
        beta_d = torch.tensor([beta], dtype=torch.float32, device=dev)
        out, _, _ = softmax_aggr_fwd_raw(st, T(x, dev), beta_d, EPS, None if A is None else T(A, dev))
        ref, bound = sa64(rp, ci, x, A, beta)
        check(out.cpu().numpy(), ref, bound, f"{c.id} {form[0]} beta={beta}")
    check_hub_plan(st, c.id)


def run_softmax_aggr_bwd(dev, c, form):
    """dx of the GENConv softmax aggregation over the transpose, from the kernel's own out and lse2: the fp64 formula
    sum over the column's edges of [pre > 0] w g (1 + beta (m - out)) with w = 2^(beta m log2 e - lse2), and the bound
    of tests/test_gpu_dispatch_message.py.  grad_out: NaN and +-Inf in g on the hub, a one-edge and a short row
    (beta = 1).  overflow: the forward's -Inf logits at beta = -2 (weight 0 against a message of 1.5e38, where
    beta (m - out) stays finite) and its all -Inf rows, whose lse2 is -Inf and whose out is NaN."""
    from cogdl_b200.operators._raw import softmax_aggr_bwd_raw, softmax_aggr_fwd_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(18)
    st = structure(rp, ci, n, dev, form)
    deg = np.diff(rp)
    if c.operand == "overflow":
        beta = -2.0
        x = sa_overflow_inputs(c, rp, ci, n, rng, form[1] or 16)
    else:
        beta = 1.0
        x = rng.uniform(-1, 3, (n, c.F)).astype(np.float32)
    g = rng.standard_normal((n, c.F)).astype(np.float32)
    if c.operand == "grad_out":
        hub, one = int(np.argmax(deg)), int(np.nonzero(deg == 1)[0][0])
        short = int(np.nonzero((deg > 3) & (deg < 16))[0][0])
        g[hub, 0], g[hub, c.F - 1], g[one, c.F // 2], g[short, 1] = np.nan, np.inf, -np.inf, np.nan
    beta_d = torch.tensor([beta], dtype=torch.float32, device=dev)
    out, lse2, _ = softmax_aggr_fwd_raw(st, T(x, dev), beta_d, EPS, want_lse=True)
    dx, _ = softmax_aggr_bwd_raw(st, T(x, dev), beta_d, EPS, T(g, dev), out, lse2)
    rows = rows_of(rp)
    pre = x[ci]
    m = (np.where(pre < 0, np.float32(0), pre) + np.float32(EPS)).astype(np.float32).astype(np.float64)
    o32, l32 = out.cpu().numpy().astype(np.float64), lse2.cpu().numpy().astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore"):
        z = beta * LOG2E * m
        arg = z - l32[rows]
        w = np.exp2(arg)
        dm = w * g[rows] * (1 + beta * (m - o32[rows]))
        dpre = np.where(pre <= 0, 0.0, dm)
        mag = np.where(pre <= 0, 0.0, w * np.abs(g[rows]) * (1 + abs(beta) * np.abs(m - o32[rows])))
        eb = mag * (2.0 ** -22 + LN2 * U32 * (3 * np.abs(z) + np.abs(np.where(np.isfinite(arg), arg, 0))) + 4 * U32)
        coldeg = np.bincount(ci, minlength=n).astype(np.float64)[:, None]
        bound = col_sum(np.nan_to_num(eb, nan=0, posinf=0), ci, n) + \
            coldeg * U32 * col_sum(np.nan_to_num(mag, nan=0, posinf=0), ci, n) + TINY
        ref = col_sum(dpre, ci, n)
    check(dx.cpu().numpy(), ref, bound, f"{c.id} {form[0]} dX")
    check_hub_plan(st, c.id)
    check_hub_plan(st.csc()[0], c.id)


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


def run_residual_dcoef(dev, c, form):
    """y = a (A x) + b z with b read on the device (GIN's learnable epsilon): a NaN or +-Inf b reaches every element of
    b z (Inf * 0 = NaN where z is 0), features planted as for the SpMM rows; without z, b is not read."""
    from cogdl_b200.operators._raw import spmm_residual_dcoef_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(14)
    X = rng.standard_normal((n, c.F)).astype(np.float32)
    w = rng.uniform(0.25, 2.0, ci.size).astype(np.float32)
    s = sites(rp)
    plant_features(X, ci, s)
    w[s["zero"]] = 0.0
    Z = rng.standard_normal((n, c.F)).astype(np.float32)
    Z[3, 5] = Z[n - 1, c.F - 1] = 0.0
    st = structure(rp, ci, n, dev, form)
    agg, abound = spmm64(rp, ci, w, X)
    a = 0.75
    for b in (np.nan, np.inf, -np.inf, -2.0):
        b_d = torch.tensor([b], dtype=torch.float32, device=dev)
        got = spmm_residual_dcoef_raw(st, T(w, dev), T(X, dev), T(Z, dev), a, b_d).cpu().numpy()
        with np.errstate(invalid="ignore"):
            bz = b * Z.astype(np.float64)
            ref = a * agg + bz
        check(got, ref, a * abound + 2 * U32 * (np.abs(a * agg) + np.abs(np.nan_to_num(bz, posinf=0, neginf=0))),
              f"{c.id} {form[0]} b={b}")
    b_d = torch.tensor([np.nan], dtype=torch.float32, device=dev)
    got = spmm_residual_dcoef_raw(st, T(w, dev), T(X, dev), None, a, b_d).cpu().numpy()
    check(got, a * agg, a * abound + 2 * U32 * np.abs(a * agg), f"{c.id} {form[0]} without z")
    check_hub_plan(st, c.id)


def signed_att(y, keep):
    """The saved attention of the dropout kernels: y with the sign bit set on the dropped entries (NaN included)."""
    return (y.view(np.uint32) | np.where(keep, 0, 0x80000000).astype(np.uint32)).view(np.float32)


def kept_times(v, keep, scale):
    """fl(v * scale) on the kept entries and v * 0 on the dropped ones, as torch's v * mask * scale (NaN * 0 = NaN)."""
    with np.errstate(invalid="ignore"):
        return (v.astype(np.float64) * np.where(keep, np.float64(np.float32(scale)), 0.0)).astype(np.float32)


def run_mhspmm_dropout(dev, c, form):
    """The dropout GAT's aggregation and its d feat (the transpose with perm): a dropped entry reads as |att| * 0, so a
    dropped NaN or Inf attention gives NaN, and a dropped entry against an Inf feature gives NaN (0 * Inf).  At the
    row's F (scalar lanes) and at F = 16 (float4 lanes)."""
    for F in (c.F, 16):                                 # scalar lanes and float4 lanes
        mhspmm_dropout_case(dev, c, form, F)


def mhspmm_dropout_case(dev, c, form, F):
    from cogdl_b200.operators._raw import mhspmm_raw
    from tests.gat_dropout_ref import keep_mask

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(15)
    s = sites(rp)
    H = c.H
    att = rng.uniform(0, 1, (ci.size, H)).astype(np.float32)
    feat = rng.standard_normal((n, H, F)).astype(np.float32)
    att[s["first"], 0], att[s["middle"], 1], att[s["last"], H - 1], att[s["one"], 2] = np.nan, np.inf, np.nan, np.inf
    att[s["short"], :] = np.nan
    feat[ci[s["zero"]], :, F - 1] = np.inf
    keep = keep_mask(0xA77 + H, ci.size, H, 0.4)
    keep[s["zero"], 3] = False                          # a dropped entry against an Inf feature
    keep[s["first"], 0], keep[s["middle"], 1], keep[s["one"], 2] = False, True, False   # dropped NaN, kept / dropped Inf
    assert (~keep & ~np.isfinite(att)).any() and (keep & ~np.isfinite(att)).any()
    scale = 1.0 / (1.0 - 0.4)
    eff = kept_times(np.abs(att), keep, scale)
    st = structure(rp, ci, n, dev, form)
    att_d = T(signed_att(att, keep), dev)
    got = mhspmm_raw(st, att_d, T(feat, dev), drop_scale=scale).cpu().numpy()
    for h in range(H):
        ref, bound = spmm64(rp, ci, eff[:, h], feat[:, h, :])
        check(got[:, h], ref, bound, f"{c.id} {form[0]} F={F} head {h}")
    check_hub_plan(st, c.id)
    st_t, perm = st.csc()
    g = rng.standard_normal((n, H, F)).astype(np.float32)
    got = mhspmm_raw(st_t, att_d, T(g, dev), perm=perm, drop_scale=scale).cpu().numpy()
    cp, ri, pm = (t.cpu().numpy() for t in (st_t.rowptr, st_t.colind, perm))
    for h in range(H):
        ref, bound = spmm64(cp, ri, eff[pm, h], g[:, h, :])
        check(got[:, h], ref, bound, f"{c.id} {form[0]} F={F} d feat head {h}")
    check_hub_plan(st_t, c.id)


def run_scatter_max_bwd(dev, c, form):
    """d x of scatter_max: each gradient element goes to the source its argmax names, NaN and +-Inf included; one of a
    row without edges (argmax -1) goes nowhere."""
    from cogdl_b200.operators._raw import scatter_max_bwd_raw, scatter_max_fwd_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(16)
    X = rng.standard_normal((n, c.F)).astype(np.float32)
    st = structure(rp, ci, n, dev, form)
    _, arg = scatter_max_fwd_raw(st, T(X, dev))
    arg_n = arg.cpu().numpy()
    deg = np.diff(rp)
    hub, one, empty = int(np.argmax(deg)), int(np.nonzero(deg == 1)[0][0]), int(np.nonzero(deg == 0)[0][0])
    short = int(np.nonzero((deg > 3) & (deg < 16))[0][0])
    G = rng.standard_normal((n, c.F)).astype(np.float32)
    G[hub, 0], G[hub, c.F - 1], G[one, c.F // 2], G[short, 1], G[empty, 2] = np.nan, np.inf, -np.inf, np.nan, np.nan
    got = scatter_max_bwd_raw(T(G, dev), arg, n).cpu().numpy()
    ok = arg_n >= 0
    col = np.broadcast_to(np.arange(c.F), G.shape)
    ref, mag, cnt = np.zeros((n, c.F)), np.zeros((n, c.F)), np.zeros((n, c.F))
    with np.errstate(invalid="ignore"):
        np.add.at(ref, (arg_n[ok], col[ok]), G[ok].astype(np.float64))
        np.add.at(mag, (arg_n[ok], col[ok]), np.abs(G[ok].astype(np.float64)))
    np.add.at(cnt, (arg_n[ok], col[ok]), 1.0)
    check(got, ref, (cnt + 2) * U32 * np.where(np.isfinite(mag), mag, 0) + TINY, f"{c.id} {form[0]}")


SLOPE = np.float32(0.2)
P_DROP = 0.4
HGN_ALPHA = 0.3


def sm_bwd_inputs(c, rp, ci, rng, keep):
    """(y, g) [nnz, H] of a softmax backward: y a softmax of random logits, g random, with NaN / +-Inf planted in g
    (grad_out) or in y (saved) at the sites of sites(), a zero attention against an Inf gradient, and non-finite
    gradients on both a kept and a dropped entry of the largest hub."""
    s = sites(rp)
    H = c.H
    y = softmax64(rp, (rng.standard_normal((ci.size, H)) * 2).astype(np.float32))[0].astype(np.float32)
    g = rng.standard_normal((ci.size, H)).astype(np.float32)
    deg = np.diff(rp)
    hub = int(np.argmax(deg))
    if c.operand == "grad_out":
        g[s["first"], 0], g[s["middle"], 1], g[s["last"], H - 1], g[s["one"], 2] = np.nan, np.inf, -np.inf, np.nan
        g[s["short"], 3] = np.inf
        y[s["zero"], 1], g[s["zero"], 1] = 0.0, np.inf
        e = np.arange(rp[hub] + 1, rp[hub + 1])
        g[e[~keep[e, 2]][0], 2] = np.nan          # a dropped entry of the hub's head 2
        g[e[keep[e, 3]][-1], 3] = -np.inf        # a kept one of head 3
    else:
        r7 = int(np.nonzero(deg == 7)[0][0])
        y[rp[r7]:rp[r7 + 1], H - 1] = np.nan      # a whole (row, head) of NaN, as a NaN logit leaves it
        y[s["first"], 0], y[s["middle"], 1], y[s["one"], 2], y[s["last"], H - 1] = np.nan, np.nan, np.nan, np.inf
        y[s["short"], :] = np.nan
    return y, g


def run_softmax_bwd(dev, c, form):
    """The softmax backward y (g - sum_row y g) (times LeakyReLU' for GAT and Simple-HGN, and its row sums), against
    the fp64 formula of tests/test_gpu_dispatch.py on the same fp32 operands.  With dropout the kernel's gradient is
    g * (kept ? scale : 0), so a NaN or Inf gradient on a dropped entry makes its (row, head) NaN, as torch's
    dropout backward g * mask * scale does."""
    from cogdl_b200.operators._raw import edge_softmax_bwd_raw, gat_attn_bwd_raw, hgn_attn_bwd_raw
    from tests.gat_dropout_ref import keep_mask
    from tests.test_gpu_dispatch import softmax_bwd64

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(11)
    H = c.H
    keep = keep_mask(0xD0 + H, ci.size, H, P_DROP)
    y, g = sm_bwd_inputs(c, rp, ci, rng, keep)
    st = structure(rp, ci, n, dev, form)
    rows = rows_of(rp)
    hl = rng.standard_normal((n, H)).astype(np.float32)
    hr = rng.standard_normal((n, H)).astype(np.float32)
    scale = 1.0 / (1.0 - P_DROP)
    if c.entry == "cogdl_b200_edge_softmax_bwd_f32":
        d_edge, g_row = edge_softmax_bwd_raw(st, T(y, dev), T(g, dev)), None
        geff, dact = g, 1.0
    elif c.entry == "cogdl_b200_hgn_attn_bwd_f32":
        n_types = 3
        etype = rng.integers(0, n_types, ci.size).astype(np.int32)
        he = rng.standard_normal((n_types, H)).astype(np.float32)
        gs = np.float32((1.0 - HGN_ALPHA) * scale)
        d_edge, g_row = hgn_attn_bwd_raw(st, T(etype, dev), T(signed_att(y, keep), dev), T(g, dev), T(hl, dev),
                                         T(hr, dev), T(he, dev), float(SLOPE), float(gs))
        geff = kept_times(g, keep, gs)
        z = (hl[rows] + hr[ci]) + he[etype]
        dact = np.where(z > 0, 1.0, np.float64(SLOPE))
    else:
        drop = c.entry == "cogdl_b200_gat_attn_bwd_dropout_f32"
        att = signed_att(y, keep) if drop else y
        d_edge, g_row = gat_attn_bwd_raw(st, T(att, dev), T(g, dev), T(hl, dev), T(hr, dev), float(SLOPE),
                                         drop_scale=scale if drop else None)
        geff = kept_times(g, keep, scale) if drop else g
        z = hl[rows] + hr[ci]
        dact = np.where(z > 0, 1.0, np.float64(SLOPE))
    with np.errstate(invalid="ignore", over="ignore"):
        ref, bound, grow, gbound = softmax_bwd64(rp, y, geff, dact)
    check(d_edge.cpu().numpy(), ref, np.where(np.isfinite(bound), bound, 0), f"{c.id} {form[0]} d edge")
    if g_row is not None:
        check(g_row.cpu().numpy(), grow, np.where(np.isfinite(gbound), gbound, 0), f"{c.id} {form[0]} g_row")
    check_hub_plan(st, c.id)


def run_hgn_attn(dev, c, form):
    """Simple-HGN's attention stage with dropout and the residual blend: one head each of a NaN logit (a NaN h_r), a
    +Inf logit, rows of nothing but -Inf (a -Inf h_l) and single -Inf logits (a -Inf h_r).  The attention is the fp64
    softmax of the fp32 logits; mix = (1 - alpha) |att| (kept ? scale : 0) + alpha res, so a dropped NaN stays NaN."""
    from cogdl_b200.operators._raw import attn_dropout_args, hgn_attn_raw
    from tests.gat_dropout_ref import keep_mask

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(13)
    s = sites(rp)
    H, n_types = c.H, 3
    rows = rows_of(rp)
    etype = rng.integers(0, n_types, ci.size).astype(np.int32)
    hl = rng.standard_normal((n, H)).astype(np.float32)
    hr = rng.standard_normal((n, H)).astype(np.float32)
    he = rng.standard_normal((n_types, H)).astype(np.float32)
    res = rng.uniform(0, 1, (ci.size, H)).astype(np.float32)
    hr[ci[s["first"]], 0] = np.nan
    hr[ci[s["one"]], 1] = np.inf
    hl[rows[s["short"]], 2] = -np.inf
    hr[ci[s["middle"]], 3] = -np.inf
    st = structure(rp, ci, n, dev, form)
    seed = 0x4E6 + H
    drop_below, scale = attn_dropout_args(P_DROP)
    mix, att = hgn_attn_raw(st, T(etype, dev), T(hl, dev), T(hr, dev), T(he, dev), float(SLOPE), True,
                            (seed, drop_below, scale), T(res, dev), HGN_ALPHA)
    mix, att = mix.cpu().numpy(), att.cpu().numpy()
    keep = keep_mask(seed, ci.size, H, P_DROP)
    assert np.array_equal(np.signbit(att), ~keep), f"{c.id} {form[0]}: the sign bits are not the dropout mask"
    with np.errstate(invalid="ignore", over="ignore"):
        z = (hl[rows] + hr[ci]) + he[etype]
        logit = np.where(z > 0, z, z * SLOPE).astype(np.float32)
        y, t, Tm, d = softmax64(rp, logit)
    sb = y * ((d + 3) * 2.0 ** -22 + d * U32 + (2 * t + 2 * Tm) * 2.0 ** -23) + 2.0 ** -126
    check(np.abs(att), y, np.where(np.isfinite(sb), sb, 0), f"{c.id} {form[0]} attention")
    assert (~keep & np.isnan(y)).any()
    keep32, ks, al = np.float32(1 - np.float32(HGN_ALPHA)), np.float64(np.float32(scale)), np.float32(HGN_ALPHA)
    with np.errstate(invalid="ignore"):
        kept = y * np.where(keep, ks, 0.0) * keep32
        ref = kept + res.astype(np.float64) * al
        bound = np.where(keep, ks, 0.0) * keep32 * sb + 3 * U32 * (np.abs(kept) + res * al) + TINY
    check(mix, ref, np.where(np.isfinite(bound), bound, 0), f"{c.id} {form[0]} mix")
    check_hub_plan(st, c.id)


def disen_overflow_inputs(rp, ci, n, K, d, chunk, rng):
    """q, c [n, K, d] fp32 whose every logit is one fp32 product, fl(fl(q0 c0) zs): q is zero past component 0 of each
    channel (|q0| <= 2) and c is unit with |c0| <= 1/2.  In channel 0, q0 = 3e38 on the largest hub, a streamed short
    row and a one-edge row, and c = -e0 on the sources of their first edges and of the first edge of the hub's second
    chunk: those logits are -Inf, the row's other logits finite (|q0 c0 zs| <= 2.2e38), and the one-edge row is all
    -Inf (NaN).  In channel 1 (and 2), q0 = 3e38 on the hub and a degree-7 row and c = +e0 on the sources of an edge in
    the middle of the hub and of the degree-7 row: +Inf logits, so those channels are NaN."""
    s = sites(rp)
    deg = np.diff(rp)
    hub, one = int(np.argmax(deg)), int(np.nonzero(deg == 1)[0][0])
    short = int(np.nonzero((deg > 3) & (deg < 16))[0][0])
    r7 = int(np.nonzero(deg == 7)[0][0])
    C = rng.standard_normal((n, K, d))
    c0 = rng.uniform(-0.5, 0.5, (n, K))
    C[..., 1:] *= (np.sqrt(1 - c0 ** 2) / np.linalg.norm(C[..., 1:], axis=-1))[..., None]
    C[..., 0] = c0
    Q = np.zeros((n, K, d))
    Q[..., 0] = rng.uniform(-2, 2, (n, K))
    big = 3e38
    for r, e in ((hub, s["first"]), (hub, rp[hub] + chunk), (short, s["zero"]), (one, s["one"])):
        Q[r, 0, 0] = big
        C[ci[e], 0] = 0.0
        C[ci[e], 0, 0] = -1.0
    for k in range(1, K):
        for r, e in ((hub, s["middle"]), (r7, rp[r7] + 3)):
            Q[r, k, 0] = big
            C[ci[e], k] = 0.0
            C[ci[e], k, 0] = 1.0
    return Q.astype(np.float32), C.astype(np.float32)


def disen_z64(rp, ci, z2, C):
    """fp64 routing step over given base-2 logits z2 [nnz, K] (the kernel's fp32 ones), with the forward bound of
    tests/test_gpu_dispatch_message.py.  The logits are exact, so only the base-2 exponent's argument d = z - M is
    rounded: by at most U32 |d|, and only for |d| < 150, since past that both the exact and the computed weight are
    below 2^-149 of the row's largest; the logit range R in the bound is capped there."""
    n, K, d = C.shape
    rows = rows_of(rp)
    C64 = C.astype(np.float64)
    with np.errstate(invalid="ignore", over="ignore", divide="ignore"):
        mx = seg_reduce(np.maximum, z2, rp)
        ex = np.exp2(z2 - mx[rows])
        S = seg_reduce(np.add, ex, rp)
        w = ex / S[rows]
        a = seg_reduce(np.add, (w[..., None] * C64[ci]).reshape(-1, K * d), rp).reshape(n, K, d)
        amag = seg_reduce(np.add, (w[..., None] * np.abs(C64[ci])).reshape(-1, K * d), rp).reshape(n, K, d)
        u = C64 + a
        r = np.linalg.norm(u, axis=2)
        out = u / r[..., None]
        zf = np.where(np.isfinite(z2), z2, np.nan)
        R = np.minimum(np.nan_to_num(seg_reduce(np.fmax, zf, rp) - seg_reduce(np.fmin, zf, rp)), 150.0)
        deg = np.diff(rp).astype(np.float64)[:, None]
        E = (deg + 3) * 2.0 ** -22 + deg * U32 + LN2 * 2 * U32 * R
        du = amag * (2 * E + (2 * deg + 1) * U32)[..., None] + U32 * np.abs(u)
        dun = np.linalg.norm(du, axis=2, keepdims=True)
        o3 = np.abs(out)
        bound = (du + o3 * dun) / r[..., None] + o3 * (d + 3) * U32 + TINY
    return out.reshape(n, K * d), np.where(np.isfinite(bound), bound, 0).reshape(n, K * d)


def run_disen(dev, c, form):
    """DisenGCN routing with +-Inf logits from a large q against unit c, at d = F / K (scalar lanes) and at K = 2,
    d = 8 (float4 lanes), against the fp64 softmax of the kernel's fp32 logits: a -Inf logit has weight 0 wherever it
    falls, a channel with a +Inf logit or with nothing but -Inf logits is NaN."""
    from cogdl_b200.operators._raw import disen_route_fwd_raw

    rp, ci, n = graph_of(c, form[1])
    rng = np.random.default_rng(17)
    st = structure(rp, ci, n, dev, form)
    hub = int(np.argmax(np.diff(rp)))
    tau = 1.0
    zs = np.float32(np.float32(LOG2E) / np.float32(tau))
    for K, d in ((c.K, c.F // c.K), (2, 8)):
        Q, C = disen_overflow_inputs(rp, ci, n, K, d, form[1] or 16, rng)
        with np.errstate(over="ignore"):
            z2 = ((Q[rows_of(rp), :, 0] * C[ci, :, 0]).astype(np.float32) * zs).astype(np.float64)
        assert np.isneginf(z2[:, 0]).any() and np.isposinf(z2[:, 1]).any()
        out, _, _ = disen_route_fwd_raw(st, T(Q.reshape(n, K * d), dev), T(C.reshape(n, K * d), dev), K, tau)
        ref, bound = disen_z64(rp, ci, z2, C)
        assert np.isfinite(ref[hub, :d]).all(), "channel 0 of the hub should stay finite"
        check(out.cpu().numpy(), ref, bound, f"{c.id} {form[0]} K={K} d={d}")
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
    "cogdl_b200_spmm_residual_dcoef_f32": run_residual_dcoef,
    "cogdl_b200_mhspmm_dropout_f32": run_mhspmm_dropout,
    "cogdl_b200_scatter_max_bwd_f32": run_scatter_max_bwd,
    "cogdl_b200_edge_softmax_bwd_f32": run_softmax_bwd,
    "cogdl_b200_gat_attn_bwd_f32": run_softmax_bwd,
    "cogdl_b200_gat_attn_bwd_dropout_f32": run_softmax_bwd,
    "cogdl_b200_hgn_attn_bwd_f32": run_softmax_bwd,
    "cogdl_b200_hgn_attn_f32": run_hgn_attn,
    "cogdl_b200_disen_route_fwd_f32": run_disen,
    "cogdl_b200_softmax_aggr_bwd_f32": run_softmax_aggr_bwd,
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
SCALER_LAYERS = ["gcn", "gcn-fused", "gat", "sage-max", "genconv", "gat-dropout", "disengcn", "compgcn", "rgcn",
                 "simple-hgn", "gin-eps", "gtn-spspmm"]
N_TYPES = 3


def edge_types(graph, dev):
    """Fixed pseudo-random relation types, one per edge of the graph."""
    E = graph.edge_index[0].numel()
    return torch.from_numpy(np.random.default_rng(21).integers(0, N_TYPES, E)).to(dev)


class GENConvAggr(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(128, 64)
        self.beta = torch.nn.Parameter(torch.tensor(1.0))

    def forward(self, graph, x):
        from cogdl_b200.operators.softmax_aggr import genconv_aggregate

        return genconv_aggregate(graph, self.lin(x), "softmax_sg", beta=self.beta)


class DisenRouting(torch.nn.Module):
    """DisenGCN's layer: h = x W + b, then one routing step over K = 4 channels of 16."""

    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(128, 64)

    def forward(self, graph, x):
        from cogdl_b200.operators.disen_routing import disen_routing

        return disen_routing(graph, self.lin(x), 4, 1)


class CompAggr(torch.nn.Module):
    """CompGCN's two half aggregations with the "mult" composition and a relation table, summed."""

    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(128, 64)
        self.rel = torch.nn.Parameter(torch.randn(N_TYPES, 64, generator=torch.Generator().manual_seed(4)))

    def forward(self, graph, x):
        from cogdl_b200.operators.comp_aggr import compgcn_aggregate

        a_in, a_out = compgcn_aggregate(graph.edge_index, edge_types(graph, x.device), self.lin(x), self.rel, "mult")
        return a_in + a_out


class RgcnConv(torch.nn.Module):
    """R-GCN with two bases over N_TYPES relations (the types in graph.edge_attr)."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(5)
        self.coef = torch.nn.Parameter(torch.randn(N_TYPES, 2, generator=g))
        self.weight = torch.nn.Parameter(torch.randn(2, 128, 64, generator=g) / 11.3)

    def forward(self, graph, x):
        from cogdl_b200.operators.rgcn import rgcn_conv

        graph.edge_attr = edge_types(graph, x.device)
        return rgcn_conv(graph, x, self.coef, self.weight)


class HgnAttn(torch.nn.Module):
    """Simple-HGN's attention layer: 4 heads of 16, a type table, attention dropout 0.3 and the residual blend."""

    def __init__(self):
        super().__init__()
        g = torch.Generator().manual_seed(6)
        self.lin = torch.nn.Linear(128, 64)
        self.a_l = torch.nn.Parameter(torch.randn(4, 16, generator=g) / 4)
        self.a_r = torch.nn.Parameter(torch.randn(4, 16, generator=g) / 4)
        self.h_e = torch.nn.Parameter(torch.randn(N_TYPES, 4, generator=g))

    def forward(self, graph, x):
        from cogdl_b200.operators.simple_hgn import hgn_attention

        h = self.lin(x).view(-1, 4, 16)
        etype = edge_types(graph, x.device)
        res = torch.full((etype.numel(), 4), 0.25, device=x.device)
        out, _ = hgn_attention(graph, h, (h * self.a_l).sum(-1), (h * self.a_r).sum(-1), self.h_e, etype, 0.2,
                               attn_drop=0.3, res_attn=res, alpha=0.3, seed=1234)
        return out.reshape(out.shape[0], -1)


class GinEps(torch.nn.Module):
    """GIN's aggregation (1 + eps) x + A x with a learnable eps."""

    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(128, 64)
        self.eps = torch.nn.Parameter(torch.tensor([0.1]))

    def forward(self, graph, x):
        from cogdl_b200.operators.gin import gin_aggregate

        return gin_aggregate(graph, self.lin(x), self.eps)


class GTNLayer(torch.nn.Module):
    """A GTN-style layer: A1 = the graph with its edges weighted by softmax(w1) of their relation, A2 = the identity
    channel weighted by softmax(w2)[0], the product A1 A2 by spspmm and its SpMM with x W."""

    def __init__(self):
        super().__init__()
        self.lin = torch.nn.Linear(128, 64)
        self.w1 = torch.nn.Parameter(torch.tensor([0.3, -0.2, 0.5]))
        self.w2 = torch.nn.Parameter(torch.tensor([0.1, 0.4]))

    def forward(self, graph, x):
        from cogdl_b200.operators.spspmm import coo_spmm, spspmm

        n = x.shape[0]
        row, col = graph.edge_index
        ia = torch.stack([row, col]).long()
        va = torch.softmax(self.w1, 0)[edge_types(graph, x.device)] * graph.edge_weight.float()
        eye = torch.arange(n, device=x.device)
        vb = torch.softmax(self.w2, 0)[0].expand(n).contiguous()
        ic, vc = spspmm(ia, va, torch.stack([eye, eye]), vb, n, n, n)
        return coo_spmm(ic, vc, n, n, self.lin(x))


MODULES = {"genconv": GENConvAggr, "disengcn": DisenRouting, "compgcn": CompAggr, "rgcn": RgcnConv,
           "simple-hgn": HgnAttn, "gin-eps": GinEps, "gtn-spspmm": GTNLayer}


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
    torch.manual_seed(3)
    if kind in MODULES:
        layer = MODULES[kind]()
    elif kind == "gat-dropout":
        from cogdl_b200.layers import GATLayer

        layer = GATLayer(128, 16, nhead=4, attn_drop=0.3, fused=True)
    else:
        layer = make_layer(kind)
    layer = layer.to(dev)
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
    elif (kind.startswith("gcn") or kind == "gin-eps") and g.is_symmetric():
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

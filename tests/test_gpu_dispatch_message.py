"""Every dispatch branch of GENConv's softmax aggregation, DisenGCN's routing, CompGCN's composition aggregation and the
fused GCN / SAGE layers, one row of tests/dispatch_table.py MESSAGE_TABLE each: the call must record exactly the
kernels the row names, every output element must lie within a bound derived below from the fp32 operations the kernels
perform, and every row with hub chunks must leave the arrival counters of its plan (and of the transpose's) at zero.
u = 2^-24 is the unit roundoff of fp32, d a row's (or column's) degree.  Every bound is per element and scales with
the sum of the absolute values of the terms that make that element, never with a row maximum.

GENConv forward (out, lse2, Q), against fp64 on the fp32 m_e = relu(x[c_e] + A_e) + eps (formed as the kernel does:
an IEEE add, a max, an add).  In base 2 the logits are z_e = beta log2(e) m_e; Z is a row's largest |z|, R its range.
The kernel forms z_e = fl(m_e fl(beta fl(log2 e))), three roundings (3u|z_e|), and keeps an online (M, S, T[, Q]) with
one MUFU.EX2 per edge: the exponential is off by 2 ulp (2^-22) plus the rounding of its argument z - M (u|z - M|
absolute, at most u R), and the running sums are rescaled at most d times by exponentials whose arguments add up to at
most R.  So each weight 2^(z_e - M) / S carries relative error at most
    E = (d + 3) 2^-22 + d u + ln2 u (6 Z + 2 R),
T and S each a further d u from their fp32 sums (fma rescales, the chunk merge in chunk order), and
    |out - out64| <= out64 (2E + (2d + 1) u),   |Q - Q64| <= Q64 (2E + (2d + 3) u)
(every term is positive: m >= eps > 0), |lse2 - lse2_64| <= (E + d u) log2(e) + 2^-21 + 2u |lse2_64|.  Degree-0 rows
give exactly 0.  Betas 0, 0.5, 4 and 20 with beta m spread over at least 60 in every row, pre-activations of
exactly 0 on every 7th column (and, with an edge term, every 5th edge cancels x exactly).
GENConv backward (dX, dA), evaluated in fp64 on the kernel's inputs (the fp32 out and lse2 of the forward): per edge
w_e = 2^(z_e - lse2_i), dpre_e = [pre_e > 0] w_e g_i (1 + beta (m_e - out_i)).  The kernel's weight is one EX2 of
fma(m, b2, -lse2): relative error 2^-22 + ln2 u (3|z_e| + |z_e - lse2_i|); the factor (1 + beta(m - out)) two more
roundings relative to 1 + |beta| |m - out|, the products two.  With mag_e = w_e |g_i| (1 + |beta| |m_e - out_i|):
    |dA_e - dpre_e| <= mag_e (2^-22 + ln2 u (3|z_e| + |z_e - lse2_i|) + 4u),
    |dX_j - sum_e dpre_e| <= sum_e (that bound) + d_j u sum_e mag_e      (the column's fp32 sum, hub chunks included)
and dA is exactly 0 where pre <= 0 (ReLU'(0) = 0).
DisenGCN forward: per channel, s_e = q_i . c_j / tau.  The dot of d floats is off by d u P_e (P_e = sum |q c|), the
logit in base 2 by log2(e)/tau d u P_e + 3u|z_e| (the scale log2(e)/tau is two roundings); with E as above (Z replaced
by the largest of those logit errors, counted twice) a_k = sum_e w_e c_j,k is within sum_e w_e |c_j,k| (2E + (2d+1)u),
and u = a + c_i one rounding more: du_k.  Then out = u / |u|:
    |out_k - out64_k| <= (du_k + |out64_k| |du|) / |u64| + |out64_k| (d + 3) u,
which grows as 1/|u64| by itself: no channel is left out.  r = |u| within |du| + (d + 2) u r64.  A NaN channel of c
(what normalising a zero-norm channel gives) must give NaN exactly where fp64 does.
DisenGCN backward, in fp64 on the kernel's inputs (the forward's out, lse2, r): g_u = (g - out (out . g)) / r with
magnitude GU = (|g| + |out| sum|out g|) / r, t_e = g_u,i . c_j with magnitude Tm_e = sum GU_i |c_j|, D_i = sum w t.
Every term of dq_i = (sum w t c_j - D_i sum w c_j) / tau and of dc_j = g_u,j + sum [w g_u,i + w (t - D_i) q_i / tau]
carries relative error at most rho = (the largest weight error of the row) + (2 d_ch + d + 8) u (the dot products,
g_u, the sequential sums, the chunk merges; d_ch = channel width), so each output is within rho times the sum of its
terms' magnitudes (|t| counted as |t| + Tm, |D| as |D| + sum w (|t| + Tm)).
CompGCN: the step is axpy_rn(acc, w, a o b) with separate roundings and no contraction, in CSR order: rows the plan does
not split are bit-identical to a numpy fp32 emulation; every row is within (d + 2) u sum |w (a o b)| of fp64.
Fused layers: the aggregated fp32 tile A32 is bit-identical to spmm_raw (to scatter_max's values for max; times the row
scale with one rounding), so the reference is fp64(A32) fp64(W)^T plus the epilogue.  The tensor-core part: A32 and W
are each split into three bf16 terms (exactly, 3 x 8 = 24 bits); the three dropped products a2 w3, a3 w2, a3 w3 are at
most 2 u M together, M = |A32| |W|^T.  Without assuming round-to-nearest inside wgmma, each of the 8 K-steps x 6
products sums 16 exact products and adds them to the accumulator, each truncated at worst: 2 ulp of a partial sum
<= M per step, 96 x 2^-23 M in all.  The epilogue: + rowsum b (the kernel's fp32 row sum is within d u sum|v| of fp64,
the product one rounding), or + S, then one rounding of the sum; ReLU is 1-Lipschitz.
That worst-case bound cannot see a dropped a3 w1 product (at most 2^-16 |a| |w| per term, below 96 x 2^-23).  So every
fused row also runs with a one-hot W (W[j, p(j)] a power of two, no bias, no self term): then each output is a sum of
three retained split products of one column, and an exact numpy emulation of the six retained products (exact in fp64)
must match within 2 x 2^-23 per contributing K-step (3 here) of the split-product magnitudes -- about 2^-20 |a w|,
which a missing a3 w1 exceeds on most elements.  The test prints the worst ratio of error to bound of every row.
"""
import numpy as np
import pytest
import torch

from tests.dispatch_table import MESSAGE_TABLE
from tests.gpu_util import T, check_counters, dev, misaligned, plan_structure
from tests.graphs import boundary_csc, boundary_csr, case

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24
TINY = float(np.finfo(np.float32).tiny)
LOG2E = float(np.log2(np.e))
LN2 = float(np.log(2.0))
EPS = 1e-7


def graph_of(c):
    if c.graph == "bounds":
        return boundary_csr(c.chunk)
    if c.graph == "bounds_t":
        return boundary_csc(c.chunk)
    return case(c.graph)


def check_kernel(c):
    from cogdl_b200 import _cabi

    assert _cabi.last_kernel() == c.kernel, f"{c.id}: launched {_cabi.last_kernel()!r}"


def has_chunks(c, st):
    assert st.plan.n_chunks > 0, f"{c.id}: the structure should have hub rows at chunk {c.chunk}"


RATIOS = {}


def assert_within(got, ref, bound, what):
    """|got - ref| <= bound element-wise (NaN anywhere fails); records the worst err / bound."""
    got = np.asarray(got, np.float64)
    err = np.abs(got - ref)
    bad = np.argwhere(~(err <= bound))
    assert bad.size == 0, (f"{what}: {len(bad)} elements outside the bound, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]!r}, ref {ref[tuple(bad[0])]!r}, bound {bound[tuple(bad[0])]!r}")
    if err.size:
        RATIOS[what] = float(np.max(err / np.maximum(bound, 1e-300)))


def assert_nan_within(got, ref, bound, what):
    """NaN exactly where the fp64 reference has it (a channel whose |u| is exactly 0, or a NaN input), the rest within
    the bound."""
    got = np.asarray(got, np.float64)
    nan = np.isnan(ref)
    assert np.array_equal(np.isnan(got), nan), f"{what}: NaN at {np.argwhere(np.isnan(got) != nan)[:4].tolist()}"
    assert_within(np.where(nan, 0, got), np.where(nan, 0, ref), np.where(nan, 1, bound), what)


def seg_reduce(ufunc, a, rp, fill=0.0):
    """ufunc over each CSR row's slice of a (edges on axis 0); rows without edges get fill."""
    deg = np.diff(rp)
    out = np.full((deg.size,) + a.shape[1:], fill, dtype=np.float64)
    nz = deg > 0
    if nz.any():
        out[nz] = ufunc.reduceat(np.asarray(a, np.float64), rp[:-1][nz], axis=0)
    return out


def col_sum(a, ci, n):
    """Sum of a's edge rows per column (the transpose's rows)."""
    order = np.argsort(ci, kind="stable")
    cp = np.zeros(n + 1, np.int64)
    cp[1:] = np.cumsum(np.bincount(ci, minlength=n))
    return seg_reduce(np.add, a[order], cp)


def edge_rows(rp):
    return np.repeat(np.arange(rp.size - 1), np.diff(rp))


# ------------------------------------------------------------------------------------------ GENConv
def sa_inputs(c, rp, ci, n, rng):
    """x [n, F] with beta m spread over >= 60 (70) in a row, every 7th column 0; edge term or None, every 5th edge
    -x[col] exactly (pre = 0)."""
    F = c.F
    top = 3.0 if c.beta == 0 else max(3.0, 70.0 / c.beta)
    x = rng.uniform(-top / 3, top, (n, F)).astype(np.float32)
    x[::7] = 0
    A = None
    if c.edge_term:
        A = (rng.standard_normal((ci.size, F)) * top / 4).astype(np.float32)
        A[::5] = -x[ci[::5]]
    return x, A


def sa_m(x, A, ci):
    pre = x[ci] if A is None else (x[ci] + A).astype(np.float32)
    m = (np.maximum(pre, np.float32(0)) + np.float32(EPS)).astype(np.float32)
    return pre, m


def sa_fwd64(rp, m, beta):
    """(out, lse2, Q, bound factor E, degree) per row and channel, fp64, of the fp32 m."""
    rows = edge_rows(rp)
    t = beta * m.astype(np.float64)
    mx = seg_reduce(np.maximum, t, rp, fill=0.0)
    mn = seg_reduce(np.minimum, t, rp, fill=0.0)
    ex = np.exp(t - mx[rows])
    S = seg_reduce(np.add, ex, rp)
    deg = np.diff(rp).astype(np.float64)[:, None]
    with np.errstate(divide="ignore", invalid="ignore"):
        w = ex / S[rows]
        out = seg_reduce(np.add, w * m, rp)
        Q = seg_reduce(np.add, w * m.astype(np.float64) ** 2, rp)
        lse2 = np.where(deg > 0, (mx + np.log(np.where(S > 0, S, 1.0))) * LOG2E, 0.0)
    Z = seg_reduce(np.maximum, np.abs(t), rp) * LOG2E
    R = (mx - mn) * LOG2E
    E = (deg + 3) * 2.0 ** -22 + deg * U32 + LN2 * U32 * (6 * Z + 2 * R)
    return out, lse2, Q, E, deg


def sa_fwd_call(dev, c, st, x, A, beta_d, want_q):
    """The forward through softmax_aggr_fwd_raw, or with c.partials_offset straight through the C entry point with the
    plan's partial scratch shifted off 16-byte alignment."""
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import _sa_scratch, softmax_aggr_fwd_raw
    from cogdl_b200.structure import _ptr, _stream

    xd = T(x, dev) if c.aligned else misaligned(T(x, dev))
    Ad = None if A is None else T(A, dev)
    if not c.partials_offset:
        return softmax_aggr_fwd_raw(st, xd, beta_d, EPS, Ad, want_lse=True, want_q=want_q)
    has_chunks(c, st)
    out = torch.empty((st.n_rows, c.F), device=dev)
    lse2, q = torch.empty_like(out), (torch.empty_like(out) if want_q else None)
    plan, keep = st.plan_struct(_sa_scratch(st, c.F) + 16)
    keep[0].partials += c.partials_offset
    keep[0].partials_bytes -= c.partials_offset
    _cabi.call("cogdl_b200_softmax_aggr_fwd_f32", _ptr(st.rowptr), _ptr(st.colind), _ptr(xd), _ptr(Ad), _ptr(beta_d),
               float(EPS), _ptr(out), _ptr(lse2), _ptr(q), st.n_rows, c.F, plan, _stream(dev))
    torch.cuda.synchronize(dev)
    del keep
    return out, lse2, q


def run_sa_fwd(dev, c):
    rp, ci, n = graph_of(c)
    rng = np.random.default_rng(1000 + c.F)
    x, A = sa_inputs(c, rp, ci, n, rng)
    st = plan_structure(rp, ci, n, dev, c.plan, c.chunk)
    beta_d = torch.tensor([c.beta], dtype=torch.float32, device=dev)
    out, lse2, q = sa_fwd_call(dev, c, st, x, A, beta_d, c.want_q)
    check_kernel(c)
    _, m = sa_m(x, A, ci)
    out64, lse64, Q64, E, deg = sa_fwd64(rp, m, c.beta)
    assert_within(out.cpu().numpy(), out64, out64 * (2 * E + (2 * deg + 1) * U32) + TINY, f"{c.id} out")
    assert_within(lse2.cpu().numpy(), lse64, (E + deg * U32) * LOG2E + 2.0 ** -21 + 2 * U32 * np.abs(lse64),
                  f"{c.id} lse2")
    if c.want_q:
        assert_within(q.cpu().numpy(), Q64, Q64 * (2 * E + (2 * deg + 3) * U32) + TINY, f"{c.id} Q")
    empty = np.diff(rp) == 0
    assert np.all(out.cpu().numpy()[empty] == 0) and np.all(lse2.cpu().numpy()[empty] == 0)
    if c.plan != "none":
        has_chunks(c, st)
    check_counters(st, c.id)


def run_sa_bwd(dev, c):
    from cogdl_b200.operators._raw import softmax_aggr_bwd_raw, softmax_aggr_fwd_raw

    rp, ci, n = graph_of(c)
    rng = np.random.default_rng(2000 + c.F)
    x, A = sa_inputs(c, rp, ci, n, rng)
    st = plan_structure(rp, ci, n, dev, c.plan, c.chunk)
    beta_d = torch.tensor([c.beta], dtype=torch.float32, device=dev)
    Ad = None if A is None else T(A, dev)
    out, lse2, _ = softmax_aggr_fwd_raw(st, T(x, dev), beta_d, EPS, Ad, want_lse=True)
    g = rng.standard_normal((n, c.F)).astype(np.float32)
    dx, da = softmax_aggr_bwd_raw(st, T(x, dev), beta_d, EPS, T(g, dev), out, lse2, Ad,
                                  want_edge_grad=c.want_edge_grad)
    check_kernel(c)
    st_t, _ = st.csc()
    has_chunks(c, st_t)
    rows = edge_rows(rp)
    pre, m = sa_m(x, A, ci)
    o32, l32 = out.cpu().numpy().astype(np.float64), lse2.cpu().numpy().astype(np.float64)
    z = c.beta * LOG2E * m.astype(np.float64)
    arg = z - l32[rows]
    w = np.exp2(arg)
    dev_m = np.abs(m - o32[rows])
    dm = w * g[rows] * (1 + c.beta * (m - o32[rows]))
    live = pre > 0
    dpre = np.where(live, dm, 0.0)
    mag = np.where(live, w * np.abs(g[rows]) * (1 + abs(c.beta) * dev_m), 0.0)
    eb = mag * (2.0 ** -22 + LN2 * U32 * (3 * np.abs(z) + np.abs(arg)) + 4 * U32)
    coldeg = np.bincount(ci, minlength=n).astype(np.float64)[:, None]
    assert_within(dx.cpu().numpy(), col_sum(dpre, ci, n),
                  col_sum(eb, ci, n) + coldeg * U32 * col_sum(mag, ci, n) + TINY, f"{c.id} dX")
    if c.edge_term and c.want_edge_grad:
        got = da.cpu().numpy()
        assert np.all(got[~live] == 0), f"{c.id}: dA is not 0 where the pre-activation is <= 0"
        assert_within(got, dpre, eb + TINY, f"{c.id} dA")
    else:
        assert da is None
    check_counters(st, c.id)
    check_counters(st_t, c.id)


# ------------------------------------------------------------------------------------------ DisenGCN
def unit(a, K):
    n, F = a.shape
    v = a.reshape(n, K, F // K).astype(np.float64)
    return (v / np.linalg.norm(v, axis=2, keepdims=True)).reshape(n, F).astype(np.float32)


def disen_inputs(c, rp, ci, n, rng):
    q = unit(rng.standard_normal((n, c.F)), c.K)
    cc = unit(rng.standard_normal((n, c.F)), c.K)
    if c.zero_norm:
        j = int(ci[rp[3]])                        # a column of the degree-C row
        cc[j, : c.F // c.K] = np.nan              # channel 0 of node j: 0 / 0
    return q, cc


def disen_fwd64(rp, ci, q, cc, K, tau):
    """fp64 routing step on the fp32 q, c with the forward bound's pieces: (out, lse2, r, u, du)."""
    n, F = q.shape
    d = F // K
    rows = edge_rows(rp)
    Q = q.reshape(n, K, d).astype(np.float64)
    C = cc.reshape(n, K, d).astype(np.float64)
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        s = (Q[rows] * C[ci]).sum(-1) / tau                              # [nnz, K]
        P = np.abs(Q[rows] * C[ci]).sum(-1)
        mx = seg_reduce(np.maximum, s, rp)
        mn = seg_reduce(np.minimum, s, rp)
        ex = np.exp(s - mx[rows])
        S = seg_reduce(np.add, ex, rp)
        w = ex / S[rows]
        a = seg_reduce(np.add, (w[..., None] * C[ci]).reshape(-1, F), rp).reshape(n, K, d)
        amag = seg_reduce(np.add, (w[..., None] * np.abs(C[ci])).reshape(-1, F), rp).reshape(n, K, d)
        deg = np.diff(rp).astype(np.float64)[:, None]
        u = C + a
        r = np.linalg.norm(u, axis=2)
        out = u / r[..., None]
        lse2 = np.where(deg > 0, (mx + np.log(np.where(S > 0, S, 1.0))) * LOG2E, 0.0)
        dz = LOG2E / tau * d * U32 * P + 3 * U32 * np.abs(s) * LOG2E             # logit error, base 2
        Zerr = seg_reduce(np.maximum, dz, rp)
        R = (mx - mn) * LOG2E
        E = (deg + 3) * 2.0 ** -22 + deg * U32 + LN2 * (2 * Zerr + 2 * U32 * R)
        du = amag * (2 * E + (2 * deg + 1) * U32)[..., None] + U32 * np.abs(u)
    return out.reshape(n, F), lse2, r, u, du, E


def run_disen_fwd(dev, c):
    from cogdl_b200.operators._raw import disen_route_fwd_raw

    rp, ci, n = graph_of(c)
    rng = np.random.default_rng(3000 + c.F * 10 + c.K)
    q, cc = disen_inputs(c, rp, ci, n, rng)
    st = plan_structure(rp, ci, n, dev, c.plan, c.chunk)
    qd, cd = T(q, dev), T(cc, dev)
    if not c.aligned:
        qd, cd = misaligned(qd), misaligned(cd)
    out, lse2, r = disen_route_fwd_raw(st, qd, cd, c.K, c.tau, want_saved=c.want_saved)
    check_kernel(c)
    has_chunks(c, st)
    out64, lse64, r64, u64, du, E = disen_fwd64(rp, ci, q, cc, c.K, c.tau)
    d = c.F // c.K
    got = out.cpu().numpy()
    nan = np.isnan(out64)
    assert np.array_equal(np.isnan(got), nan), f"{c.id}: NaN at {np.argwhere(np.isnan(got) != nan)[:4].tolist()}"
    if c.zero_norm:
        assert nan.any()
    n_ = rp.size - 1
    with np.errstate(invalid="ignore", divide="ignore"):
        dun = np.linalg.norm(du, axis=2, keepdims=True)
        o3 = np.abs(out64.reshape(n_, c.K, d))
        bound = (du + o3 * dun) / r64[..., None] + o3 * (d + 3) * U32 + TINY
    bound = bound.reshape(n_, c.F)
    assert_within(np.where(nan, 0, got), np.where(nan, 0, out64), np.where(nan, 1, bound), f"{c.id} out")
    if c.want_saved:
        okk = ~np.isnan(r64)
        rb = np.where(okk, dun[..., 0] + (d + 2) * U32 * r64, 1) + TINY
        assert_within(np.where(okk, r.cpu().numpy(), 0), np.where(okk, r64, 0), rb, f"{c.id} r")
        lb = np.where(okk, (E + np.diff(rp)[:, None] * U32) * LOG2E + 2.0 ** -21 + 2 * U32 * np.abs(lse64), 1)
        assert_within(np.where(okk, lse2.cpu().numpy(), 0), np.where(okk, lse64, 0), lb, f"{c.id} lse2")
    else:
        assert lse2 is None and r is None
    check_counters(st, c.id)


def run_disen_bwd(dev, c):
    from cogdl_b200.operators._raw import disen_route_bwd_raw, disen_route_fwd_raw

    rp, ci, n = graph_of(c)
    rng = np.random.default_rng(4000 + c.F * 10 + c.K)
    q, cc = disen_inputs(c, rp, ci, n, rng)
    st = plan_structure(rp, ci, n, dev, c.plan, c.chunk)
    qd, cd = T(q, dev), T(cc, dev)
    gd = T(rng.standard_normal((n, c.F)).astype(np.float32), dev)
    if not c.aligned:
        qd, cd, gd = misaligned(qd), misaligned(cd), misaligned(gd)
    out, lse2, r = disen_route_fwd_raw(st, qd, cd, c.K, c.tau, want_saved=True)
    dq, dc = disen_route_bwd_raw(st, qd, cd, c.K, c.tau, gd, out, lse2, r)
    check_kernel(c)
    st_t, _ = st.csc()
    has_chunks(c, st)
    has_chunks(c, st_t)
    K, d, tau = c.K, c.F // c.K, c.tau
    rows = edge_rows(rp)
    f = lambda t: t.cpu().numpy().astype(np.float64)  # noqa: E731
    Qv, Cv = q.reshape(n, K, d).astype(np.float64), cc.reshape(n, K, d).astype(np.float64)
    G, O = f(gd).reshape(n, K, d), f(out).reshape(n, K, d)
    L, Rr = f(lse2), f(r)
    og = (O * G).sum(-1, keepdims=True)
    with np.errstate(invalid="ignore", divide="ignore"):   # d = 1: u = a + c can cancel exactly, r = 0
        gu = (G - O * og) / Rr[..., None]
        GU = (np.abs(G) + np.abs(O) * np.abs(O * G).sum(-1, keepdims=True)) / Rr[..., None]
    s = (Qv[rows] * Cv[ci]).sum(-1)
    P = np.abs(Qv[rows] * Cv[ci]).sum(-1)
    z = s * LOG2E / tau
    arg = z - L[rows]
    w = np.exp2(arg)                                                     # [nnz, K]
    t = (gu[rows] * Cv[ci]).sum(-1)
    Tm = (GU[rows] * np.abs(Cv[ci])).sum(-1)
    ew = 2.0 ** -22 + LN2 * (LOG2E / tau * d * U32 * P + 3 * U32 * np.abs(z) + U32 * np.abs(arg))
    deg = np.diff(rp).astype(np.float64)
    rho = seg_reduce(np.maximum, ew, rp) + (2 * d + deg[:, None] + 8) * U32      # [n, K]
    D = seg_reduce(np.add, w * t, rp)
    Dm = seg_reduce(np.add, w * (np.abs(t) + Tm), rp)
    flat = lambda a: a.reshape(a.shape[0], -1)  # noqa: E731
    A1 = seg_reduce(np.add, flat(w[..., None] * t[..., None] * Cv[ci]), rp).reshape(n, K, d)
    A2 = seg_reduce(np.add, flat(w[..., None] * Cv[ci]), rp).reshape(n, K, d)
    A1m = seg_reduce(np.add, flat(w[..., None] * (np.abs(t) + Tm)[..., None] * np.abs(Cv[ci])), rp).reshape(n, K, d)
    A2m = seg_reduce(np.add, flat(w[..., None] * np.abs(Cv[ci])), rp).reshape(n, K, d)
    dq64 = (A1 - D[..., None] * A2) / tau
    dqm = (A1m + (np.abs(D) + Dm)[..., None] * A2m) / tau
    with np.errstate(invalid="ignore"):
        dqb = (rho[..., None] * dqm).reshape(n, -1) + TINY
    assert_nan_within(f(dq), dq64.reshape(n, -1), dqb, f"{c.id} dq")
    # dc over the transpose: each edge (i, j) adds w g_u,i + w (t - D_i) q_i / tau to column j
    term = w[..., None] * gu[rows] + (w * (t - D[rows]))[..., None] * Qv[rows] / tau
    tmag = w[..., None] * GU[rows] + (w * (np.abs(t) + Tm + np.abs(D[rows]) + Dm[rows]))[..., None] * np.abs(Qv[rows]) / tau
    coldeg = np.bincount(ci, minlength=n).astype(np.float64)
    rho_e = rho[rows] + (coldeg[ci][:, None] + 4) * U32
    dc64 = gu.reshape(n, -1) + col_sum(flat(term), ci, n)
    dcb = col_sum(flat(rho_e[..., None] * tmag), ci, n) + (d + 4) * U32 * GU.reshape(n, -1) + U32 * np.abs(dc64) + TINY
    assert_nan_within(f(dc), dc64, dcb, f"{c.id} dc")
    check_counters(st, c.id)
    check_counters(st_t, c.id)


# ------------------------------------------------------------------------------------------ CompGCN
def run_comp(dev, c):
    from cogdl_b200.operators._raw import comp_aggr_raw

    rp, ci, n = graph_of(c)
    rng = np.random.default_rng(5000 + c.F * 10 + c.T)
    nnz = ci.size
    idx2 = rng.integers(0, c.T, nnz).astype(np.int32)
    w = rng.standard_normal(nnz).astype(np.float32)
    a = rng.standard_normal((n, c.F)).astype(np.float32)
    b = rng.standard_normal((c.T, c.F)).astype(np.float32)
    st = plan_structure(rp, ci, n, dev, c.plan, c.chunk)
    y = comp_aggr_raw(st, T(idx2, dev), T(w, dev), T(a, dev), T(b, dev), c.comp).cpu().numpy()
    check_kernel(c)
    has_chunks(c, st)
    phi = {"mult": lambda: a[ci] * b[idx2], "sub": lambda: a[ci] - b[idx2], "copy": lambda: a[ci]}[c.comp]()
    phi = phi.astype(np.float32)
    term32 = (w[:, None] * phi).astype(np.float32)
    # rows the plan does not split: fp32 in CSR order, bit for bit
    deg = np.diff(rp)
    whole = deg <= c.chunk
    acc = np.zeros((n, c.F), np.float32)
    for k in range(int(deg[whole].max())):
        r = np.nonzero(whole & (deg > k))[0]
        acc[r] = (acc[r] + term32[rp[r] + k]).astype(np.float32)
    assert np.array_equal(y[whole], acc[whole]), f"{c.id}: rows not split by the plan must be bit-identical"
    a64, b64 = a[ci].astype(np.float64), b[idx2].astype(np.float64)
    terms = w[:, None].astype(np.float64) * {"mult": a64 * b64, "sub": a64 - b64, "copy": a64}[c.comp]
    ref = seg_reduce(np.add, terms, rp)
    assert_within(y, ref, (deg[:, None] + 2) * U32 * seg_reduce(np.add, np.abs(terms), rp) + TINY, c.id)
    check_counters(st, c.id)


# ------------------------------------------------------------------------------------------ fused layers
def bf16_rn(a):
    """fp32 -> the nearest bf16 (ties to even), returned as fp32."""
    b = np.ascontiguousarray(a, np.float32).view(np.uint32).astype(np.uint64)
    b = (b + 0x7FFF + ((b >> 16) & 1)) & 0xFFFF0000
    return b.astype(np.uint32).view(np.float32)


def split3(a):
    a = np.asarray(a, np.float32)
    a1 = bf16_rn(a)
    r1 = (a - a1).astype(np.float32)
    a2 = bf16_rn(r1)
    a3 = bf16_rn((r1 - a2).astype(np.float32))
    return a1, a2, a3


PRODUCTS = ((2, 0), (1, 1), (0, 2), (1, 0), (0, 1), (0, 0))    # (A split, W split), the kernel's order


def emulate(A32, W):
    """The six retained split products, exact in fp64, their magnitude, and per output the number of (product, K-step)
    pairs that add anything (a 16-wide block of k where both split operands have a nonzero)."""
    As, Ws = split3(A32), split3(W)
    E = np.zeros((A32.shape[0], W.shape[0]))
    Mg = np.zeros_like(E)
    steps = np.zeros_like(E)
    for i, j in PRODUCTS:
        a, w = As[i].astype(np.float64), Ws[j].astype(np.float64)
        E += a @ w.T
        Mg += np.abs(a) @ np.abs(w).T
        for k0 in range(0, 128, 16):
            steps += ((a[:, k0:k0 + 16] != 0).astype(np.float64) @ (w[:, k0:k0 + 16] != 0).T.astype(np.float64)) > 0
    return E, Mg, steps


def fused_call(c, st, val, rs, x, W, bias, relu):
    from cogdl_b200.operators.fused_gcn import fused_gcn_raw
    from cogdl_b200.operators.fused_sage import fused_sage_raw

    if c.op == "fused_gcn":
        return fused_gcn_raw(st, val, x, W, bias, relu)
    aggr = "max" if c.op == "fused_sage_max" else "sum"
    return fused_sage_raw(st, val, rs, x, W, bias, aggr, relu)


def run_fused(dev, c):
    import torch.nn.functional as F_

    from cogdl_b200.operators._raw import scatter_max_fwd_raw, spmm_raw

    rp, ci, n = graph_of(c)
    rng = np.random.default_rng(6000 + c.F)
    st = plan_structure(rp, ci, n, dev, c.plan, c.chunk)
    x = T(rng.standard_normal((n, 128)).astype(np.float32), dev)
    val = T(rng.random(ci.size).astype(np.float32), dev) if c.weighted and c.op != "fused_sage_max" else None
    rs = T((rng.random(n) + 0.5).astype(np.float32), dev) if c.row_scale else None
    sage = c.op != "fused_gcn"
    W = T((rng.standard_normal((c.F, 256 if sage else 128)) / 11.3).astype(np.float32), dev)
    bias = T(rng.standard_normal(c.F).astype(np.float32), dev) if c.bias else None
    out = fused_call(c, st, val, rs, x, W, bias, c.relu)
    check_kernel(c)
    if " + " in c.kernel:
        has_chunks(c, st)
    else:
        assert st.plan.n_chunks == 0, f"{c.id}: the structure should have no hub rows"
    check_counters(st, c.id)
    # the aggregated tile, as the kernel forms it
    if c.op == "fused_sage_max":
        A32 = scatter_max_fwd_raw(st, x)[0].cpu().numpy()
    else:
        A32 = spmm_raw(st, val, x).cpu().numpy()
        if rs is not None:
            A32 = (rs.cpu().numpy()[:, None] * A32).astype(np.float32)
    Wn = (W[:, 128:] if sage else W).cpu().numpy()
    A64, W64 = A32.astype(np.float64), Wn.astype(np.float64)
    M = np.abs(A64) @ np.abs(W64).T
    ref = A64 @ W64.T
    bound = 98 * 2.0 ** -23 * M
    if sage:
        S = F_.linear(x[:n], W[:, :128], bias).cpu().numpy().astype(np.float64)
        ref = ref + S
    elif bias is not None:
        v = np.ones(ci.size) if val is None else val.cpu().numpy().astype(np.float64)
        rsum = seg_reduce(np.add, v, rp)[:, None]
        b64 = bias.cpu().numpy().astype(np.float64)[None, :]
        ref = ref + rsum * b64
        deg = np.diff(rp)[:, None]
        bound = bound + np.abs(b64) * (deg * U32 * seg_reduce(np.add, np.abs(v), rp)[:, None]) + U32 * np.abs(rsum * b64)
    bound = bound + U32 * np.abs(ref) + TINY
    if c.relu:
        ref = np.maximum(ref, 0)
    assert_within(out.cpu().numpy(), ref, bound, f"{c.id} fp64")
    # one-hot W, no bias, no self term: every output is three retained split products of one column
    perm = rng.permutation(128)[: c.F]
    Woh = np.zeros((c.F, 128), np.float32)
    Woh[np.arange(c.F), perm] = 2.0 ** (np.arange(c.F) % 5 - 2)
    Wfull = np.concatenate([np.zeros_like(Woh), Woh], 1) if sage else Woh
    got = fused_call(c, st, val, rs, x, T(Wfull, dev), None, False).cpu().numpy()
    E, Mg, steps = emulate(A32, Woh)
    assert np.all(steps <= 3)
    assert_within(got, E, 2.0 ** -22 * steps * Mg + TINY, f"{c.id} split emulation")
    check_counters(st, c.id)


RUN = {"sa_fwd": run_sa_fwd, "sa_bwd": run_sa_bwd, "disen_fwd": run_disen_fwd, "disen_bwd": run_disen_bwd,
       "comp": run_comp, "fused_gcn": run_fused, "fused_sage_sum": run_fused, "fused_sage_max": run_fused}


@pytest.mark.parametrize("c", MESSAGE_TABLE, ids=lambda c: c.id)
def test_message_row(dev, c):
    RATIOS.clear()
    RUN[c.op](dev, c)
    print(" ".join(f"[{k}: worst err/bound {v:.3g}]" for k, v in RATIOS.items()))

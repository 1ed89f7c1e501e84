"""Every dispatch branch of the SpMM (fp32 and fp16), SDDMM, multi-head SpMM, scatter_max, edge softmax and GAT
attention entry points, one row of tests/dispatch_table.py each: the call must record exactly the kernel the row
names, and its output must match a reference.

- fp32 SpMM: rows the hub plan does not split are bit-identical to the oracle (CSR order, separate fp32 multiply
  and add); every element is within the fp64 bound below.
- scatter_max: values and argmax equal the oracle's, ties included (quantised inputs).
- SDDMM, multi-head SDDMM and multi-head SpMM: per element, |got - ref| <= n * 2^-24 * sum|terms| + tiny against an
  fp64 evaluation, n the number of terms (row degree or dot length).  A bound relative to the largest output would
  let a row of small values be wrong by a large relative amount.
- fp16 SpMM: fp64 over the fp16-rounded inputs, bound 2^-11 |ref| + deg * 2^-24 * sum|v x| + 2^-24 (one fp16
  rounding of the output plus the fp32 accumulation), with outputs in the fp16 subnormal range and a row whose
  terms cancel exactly.
- Edge softmax forward and the GAT attention, per element against the fp64 softmax of the fp32 logits (for the
  attention, leakyrelu(h_l[row] + h_r[col]) formed in fp32 as the kernels do: an IEEE add, then the product with the
  slope).  With t = x - m, T the row's largest finite |t| and d the degree:

      |y - y64| <= y64 ((d + 3) 2^-22 + d 2^-24 + (2|t| + 2T) 2^-23) + 2^-126

  An exp evaluated as MUFU.EX2 of fl(fl(x - m) * log2 e) is off by 2 ulp plus about 1.17 |t| ulp from the argument's
  two roundings (2^-22 + 1.7 |t| 2^-23 relative): once in the numerator, and in every rescale of the running sum by
  exp(m_old - m_new), which are at most d per row and whose arguments add up to at most T.  The terms of the sum carry
  the same relative error (their exp(-|t|) |t| is at most 1/e), the fp32 sum of d terms d 2^-24, the reciprocal and
  the product two more roundings.  MUFU.EX2 flushes results below 2^-126 to zero, hence the absolute term.  NaN
  positions (a (row, head) of nothing but -inf logits) must equal the reference's; a -inf logit in any other row gives
  exactly 0.  With dropout, the sign bits of the attention must equal the keep rule's mask bit for bit.
- Edge softmax backward and the GAT attention backward: y (g - sum_row y g) dact, dact the LeakyReLU derivative at
  the fp32 pre-activation (the slope at exactly 0), per element within (d + 3) 2^-24 dact y (|g| + sum_row |y g|)
  (the fp32 dot product of d terms, then the subtraction and two products); the row sums g_row within the row sum of
  those bounds plus d 2^-24 sum_row |d_edge|.  With dropout, y = |att| and g = d_att * scale rounded to fp32 on the
  kept entries and 0 on the dropped ones, as the kernels read them.
- Every row with hub chunks leaves the plan's arrival counters at zero.
"""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import oracle
from tests.dispatch_table import TABLE
from tests.gpu_util import T, check_counters, dev, misaligned, plan_structure
from tests.graphs import boundary_csr, case

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24                      # unit roundoff of fp32
TINY = float(np.finfo(np.float32).tiny)


def csr64(rp, ci, vals, n_cols):
    # copies: abs() of a scipy CSR sorts its indices in place, which must not reorder the caller's colind
    return sp.csr_matrix((np.array(vals, np.float64), ci.copy(), rp.copy()), shape=(rp.shape[0] - 1, n_cols))


RATIOS = {}


def assert_within(got, ref, bound, what):
    """|got - ref| <= bound element-wise (NaN anywhere fails); records the worst err / bound under `what`."""
    err = np.abs(np.asarray(got, np.float64) - ref)
    bad = np.argwhere(~(err <= bound))
    assert bad.size == 0, (f"{what}: {len(bad)} elements outside the bound, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]!r}, ref {ref[tuple(bad[0])]!r}, bound {bound[tuple(bad[0])]!r}")
    if err.size:
        RATIOS[what] = float(np.max(err / np.maximum(bound, 1e-300)))


def split_rows(rp, st):
    """Rows the hub plan cuts into chunks (their partial sums are combined in chunk order)."""
    deg = np.diff(rp)
    return deg > st.chunk_edges if st.chunk_edges > 0 else np.zeros_like(deg, bool)


def check_kernel(c):
    from cogdl_b200 import _cabi

    assert _cabi.last_kernel() == c.kernel, f"{c.id}: launched {_cabi.last_kernel()!r}"


# ------------------------------------------------------------------------------------------ fp32 SpMM
def _peer_call(dev, c, rp, ci, n_cols, val_d, X):
    """cogdl_b200_spmm_csr_f32_peers with three shards on this GPU: [0,400) local, [400,700) owner 1, [700,n) owner 2."""
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import _scratch
    from cogdl_b200.structure import _ptr, _stream

    bounds, shift = [0, 400, 700, n_cols], 9
    enc = ci.copy()
    for o in (1, 2):
        m = (ci >= bounds[o]) & (ci < bounds[o + 1])
        enc[m] = bounds[1] + (o << shift) + (ci[m] - bounds[o])
    st = plan_structure(rp, enc, n_cols, dev, c.plan, c.chunk)
    shards = [T(X[bounds[o]:bounds[o + 1]], dev) for o in range(3)]
    ptrs = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in shards])
    y = torch.empty((rp.shape[0] - 1, c.F), device=dev)
    plan, keep = st.plan_struct(_scratch("spmm", st, c.F) + 16)
    if c.partials_offset:
        assert st.plan.n_chunks > 0, "the partials offset only matters with hub chunks"
        keep[0].partials += c.partials_offset
        keep[0].partials_bytes -= c.partials_offset
    _cabi.call("cogdl_b200_spmm_csr_f32_peers", _ptr(st.rowptr), _ptr(st.colind), _ptr(val_d), _ptr(shards[0]),
               bounds[1], ctypes.cast(ptrs, ctypes.c_void_p), 3, shift, _ptr(y), rp.shape[0] - 1, c.F, plan,
               _stream(dev))
    return st, y


def run_spmm(dev, c):
    from cogdl_b200.operators._raw import spmm_2src_raw, spmm_raw

    rp, ci, n_cols = case(c.graph)
    rng = np.random.default_rng(100 + c.F)
    X = rng.standard_normal((n_cols, c.F)).astype(np.float32)
    val = rng.random(ci.shape[0]).astype(np.float32) if c.weighted else None
    val_d = None if val is None else T(val, dev)
    Xd = T(X, dev) if c.aligned else misaligned(T(X, dev))
    if c.src == "one":
        st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
        y = spmm_raw(st, val_d, Xd, panels=c.panels)
    elif c.src == "two":
        st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
        n0 = 400
        y = spmm_2src_raw(st, val_d, Xd[:n0], Xd[n0:])
    else:
        st, y = _peer_call(dev, c, rp, ci, n_cols, val_d, X)
    check_kernel(c)
    got = y.cpu().numpy()
    ref = oracle.spmm_csr(rp, ci, val, X)
    whole = ~split_rows(rp, st)
    assert np.array_equal(got[whole], ref[whole]), f"{c.id}: rows not split by the plan must be bit-identical"
    A = csr64(rp, ci, val if c.weighted else np.ones(ci.shape[0]), n_cols)
    X64 = X.astype(np.float64)
    deg = np.diff(rp)[:, None]
    assert_within(got, A @ X64, deg * U32 * (abs(A) @ np.abs(X64)) + TINY, c.id)
    if c.plan != "none":
        assert st.plan.n_chunks > 0, f"{c.id}: the graph should have hub rows at chunk {c.chunk}"
        assert int(st.plan.counters.abs().sum()) == 0


# ------------------------------------------------------------------------------------------ fp16 SpMM
def fp16_bound(ref, mag, n):
    return 2.0 ** -11 * np.abs(ref) + n * U32 * mag + 2.0 ** -24


def plant_cancelling_row(rp, ci, val, X, chunk):
    """Make one unsplit row's terms cancel exactly: two edges of weight v to columns c0 != c1 with X[c1] = -X[c0],
    every other edge of the row weighted 0.  Returns the row."""
    deg = np.diff(rp)
    for r in np.nonzero((deg >= 2) & (deg <= chunk))[0]:
        cols = ci[rp[r]:rp[r + 1]]
        if np.any(cols != cols[0]):
            e0 = rp[r]
            e1 = rp[r] + int(np.nonzero(cols != cols[0])[0][0])
            val[rp[r]:rp[r + 1]] = 0
            val[e0] = val[e1] = np.float16(0.75)
            X[ci[e1]] = -X[ci[e0]]
            # every other row that reads column ci[e1] now sees -X[ci[e0]]: still a valid input
            return int(r)
    raise AssertionError("no row to plant the cancellation in")


def run_spmm_f16(dev, c):
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n_cols = case(c.graph)
    rng = np.random.default_rng(200 + c.F)
    X = rng.standard_normal((n_cols, c.F))
    X[:, 1::2] *= 2.0 ** -16          # odd columns: sums in the fp16 subnormal range (below 2^-14)
    X = X.astype(np.float16)
    val = rng.random(ci.shape[0]).astype(np.float16) if c.weighted else None
    zero_row = plant_cancelling_row(rp, ci, val, X, c.chunk if c.plan != "none" else 1 << 30) if c.weighted else None
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    Xd = T(X, dev) if c.aligned else misaligned(T(X, dev))
    y = spmm_raw(st, None if val is None else T(val, dev), Xd)
    check_kernel(c)
    assert y.dtype == torch.float16
    got = y.cpu().numpy().astype(np.float64)
    A = csr64(rp, ci, val.astype(np.float64) if c.weighted else np.ones(ci.shape[0]), n_cols)
    X64 = X.astype(np.float64)
    ref = A @ X64
    assert_within(got, ref, fp16_bound(ref, abs(A) @ np.abs(X64), np.diff(rp)[:, None]), c.id)
    sub = (np.abs(ref) < 2.0 ** -14) & (np.abs(ref) > 2.0 ** -22)
    assert sub.sum() > 100, "the case should produce fp16 subnormal outputs"
    if zero_row is not None:
        assert np.all(got[zero_row] == 0), f"{c.id}: exactly cancelling row {zero_row} is not 0"


# ------------------------------------------------------------------------------------------ SDDMM
def run_sddmm(dev, c):
    from cogdl_b200.operators._raw import mhsddmm_raw, sddmm_raw

    rp, ci, n_cols = case(c.graph)
    n = rp.shape[0] - 1
    rng = np.random.default_rng(300 + c.H * 1000 + c.F)
    D1 = rng.standard_normal((n, c.H, c.F)).astype(np.float32)
    D2 = rng.standard_normal((n_cols, c.H, c.F)).astype(np.float32)
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    d1 = T(D1, dev)
    d2 = T(D2, dev) if c.aligned else misaligned(T(D2, dev))
    if c.H == 1:
        out = sddmm_raw(st, d1.view(n, c.F), d2.view(n_cols, c.F))
    else:
        out = mhsddmm_raw(st, d1, d2)
    check_kernel(c)
    got = out.cpu().numpy().reshape(ci.shape[0], c.H)
    rows = np.repeat(np.arange(n), np.diff(rp))
    terms = D1[rows].astype(np.float64) * D2[ci].astype(np.float64)
    assert_within(got, terms.sum(-1), c.F * U32 * np.abs(terms).sum(-1) + TINY, c.id)


# ------------------------------------------------------------------------------------------ multi-head SpMM
def run_mhspmm(dev, c):
    from cogdl_b200.operators._raw import mhspmm_raw

    rp, ci, n_cols = case(c.graph)
    n = rp.shape[0] - 1
    rng = np.random.default_rng(400 + c.H * 1000 + c.F)
    nnz = ci.shape[0]
    att = rng.random((nnz, c.H)).astype(np.float32)
    eff = att
    scale = None
    if c.drop:
        # dropped entries carry the sign bit; kept ones are read as att * scale (one fp32 rounding)
        scale = np.float32(1.0 / 0.7)
        mask = rng.random((nnz, c.H)) < 0.3
        eff = np.where(mask, np.float32(0), att * scale).astype(np.float32)
        att = np.where(mask, -att, att).astype(np.float32)
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    if c.perm:
        # the transposed pass (grad_feat of the GAT aggregation): rows of A^T, attention read through the permutation
        st, p = st.csc()
        ptr, idx, perm = oracle.csr2csc(rp, ci, n_cols)
        eff = eff[perm]
        n_out, n_in = n_cols, n
    else:
        p, ptr, idx, n_out, n_in = None, rp, ci, n, n_cols
    feat = rng.standard_normal((n_in, c.H, c.F)).astype(np.float32)
    fd = T(feat, dev) if c.aligned else misaligned(T(feat, dev))
    out = mhspmm_raw(st, T(att, dev), fd, perm=p, drop_scale=None if scale is None else float(scale))
    check_kernel(c)
    got = out.cpu().numpy()
    deg = np.diff(ptr)[:, None]
    for h in range(c.H):
        A = csr64(ptr, idx, eff[:, h], n_in)
        f64 = feat[:, h, :].astype(np.float64)
        assert_within(got[:, h, :], A @ f64, deg * U32 * (abs(A) @ np.abs(f64)) + TINY, f"{c.id} head {h}")
    assert got.shape == (n_out, c.H, c.F)
    if st.chunk_edges > 0:
        assert int(st.plan.counters.abs().sum()) == 0


# ------------------------------------------------------------------------------------------ scatter_max
def run_scatter_max(dev, c):
    from cogdl_b200.operators._raw import scatter_max_bwd_raw, scatter_max_fwd_raw

    rp, ci, n_cols = case(c.graph)
    n = rp.shape[0] - 1
    rng = np.random.default_rng(500 + c.F)
    # mixed signs and deliberate ties (quantised values): "first max wins" decides the argmax
    X = np.round(rng.standard_normal((n_cols, c.F)) * 4).astype(np.float32) / 4
    ref, ref_id = oracle.scatter_max_fwd(rp, ci, X)
    if c.op == "scatter_max_bwd":
        g = rng.standard_normal((n, c.F)).astype(np.float32)
        gx = scatter_max_bwd_raw(T(g, dev), T(ref_id, dev), n_cols).cpu().numpy()
        check_kernel(c)
        ok = ref_id >= 0
        cols = np.broadcast_to(np.arange(c.F), ref_id.shape)[ok]
        want, mag, cnt = (np.zeros((n_cols, c.F)) for _ in range(3))
        np.add.at(want, (ref_id[ok], cols), g[ok].astype(np.float64))
        np.add.at(mag, (ref_id[ok], cols), np.abs(g[ok]).astype(np.float64))
        np.add.at(cnt, (ref_id[ok], cols), 1)
        assert_within(gx, want, cnt * U32 * mag + TINY, c.id)
        return
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    Xd = T(X, dev) if c.aligned else misaligned(T(X, dev))
    out, arg = scatter_max_fwd_raw(st, Xd)
    check_kernel(c)
    assert np.array_equal(out.cpu().numpy(), ref), f"{c.id}: max differs"
    assert np.array_equal(arg.cpu().numpy(), ref_id), f"{c.id}: argmax differs"
    if c.plan != "none":
        assert st.plan.n_chunks > 0 and int(st.plan.counters.abs().sum()) == 0


# ------------------------------------------------------------------------------------------ edge softmax, GAT attention
SLOPE = np.float32(0.2)
P_DROP = 0.4


def es_graph(c):
    return boundary_csr(c.chunk) if c.graph == "bounds" else case(c.graph)


def es_logits(rp, H, rng, masked=False, chunk=0):
    """[nnz, H] fp32 logits: even rows uniform over [-90, 0] (exp of the smallest is below 2^-126, where MUFU.EX2
    flushes to zero), odd rows N(0, 4).  masked: per row a leading, middle or trailing -inf in one head, the whole first
    chunk of the largest hub in head 0, and every logit of a 3-edge row and (H > 1) of the 2 * chunk hub in head H - 1."""
    n, deg = rp.shape[0] - 1, np.diff(rp)
    rows = np.repeat(np.arange(n), deg)
    x = np.where((rows % 2 == 0)[:, None], rng.uniform(-90, 0, (rows.size, H)), rng.standard_normal((rows.size, H)) * 2)
    x = x.astype(np.float32)
    if masked:
        for r in np.nonzero(deg >= 2)[0]:
            x[rp[r] + (0, deg[r] // 2, deg[r] - 1)[r % 3], (r // 3) % H] = -np.inf
        big = int(np.argmax(deg))
        if chunk and deg[big] > chunk:
            x[rp[big]:rp[big] + chunk, 0] = -np.inf
        full = np.nonzero(deg == 3)[0][:1].tolist() + (np.nonzero(deg == 2 * chunk)[0][:1].tolist() if H > 1 else [])
        for r in full:
            x[rp[r]:rp[r + 1], H - 1] = -np.inf
    return x


def softmax64(rp, x):
    """fp64 softmax of fp32 logits over each row's edges, per head, with what its error bound needs: (y, |t|, T, d) per
    element, t = x - row max (0 where x is -inf), T the row's largest |t|, d the row's degree.  A (row, head) of
    nothing but -inf gives NaN."""
    n, deg = rp.shape[0] - 1, np.diff(rp)
    rows = np.repeat(np.arange(n), deg)
    x64 = x.astype(np.float64)
    m = np.full((n, x.shape[1]), -np.inf)
    np.maximum.at(m, rows, x64)
    with np.errstate(invalid="ignore", divide="ignore"):
        t = x64 - m[rows]
        ex = np.exp(t)
        s = np.zeros_like(m)
        np.add.at(s, rows, ex)
        y = ex / s[rows]
    t = np.where(np.isfinite(t), np.abs(t), 0.0)
    T = np.zeros_like(m)
    np.maximum.at(T, rows, t)
    return y, t, T[rows], deg[rows][:, None].astype(np.float64)


def check_softmax(got, x, rp, what):
    """got against the fp64 softmax of the fp32 logits x: NaN exactly where the reference is NaN, every other element
    within the forward bound of the module docstring."""
    y, t, T, d = softmax64(rp, x)
    nan = np.isnan(y)
    assert np.array_equal(np.isnan(got), nan), (f"{what}: NaN at {np.argwhere(np.isnan(got) != nan)[:4].tolist()}, "
                                                f"{int(np.isnan(got).sum())} NaN, reference {int(nan.sum())}")
    bound = y * ((d + 3) * 2.0 ** -22 + d * U32 + (2 * t + 2 * T) * 2.0 ** -23) + 2.0 ** -126
    assert_within(np.where(nan, 0, got), np.where(nan, 0, y), np.where(nan, 1, bound), what)


def softmax_bwd64(rp, y, g, dact):
    """fp64 y * (g - sum_row y * g) * dact from the fp32 y, g the kernel reads, with the per-element bound
    (d + 3) 2^-24 dact y (|g| + sum_row |y g|) and the row sums with theirs."""
    n, deg = rp.shape[0] - 1, np.diff(rp)
    rows = np.repeat(np.arange(n), deg)
    y64, g64 = y.astype(np.float64), g.astype(np.float64)
    s, mag = np.zeros((n, y.shape[1])), np.zeros((n, y.shape[1]))
    np.add.at(s, rows, y64 * g64)
    np.add.at(mag, rows, np.abs(y64 * g64))
    out = y64 * (g64 - s[rows]) * dact
    bound = (deg[rows][:, None] + 3) * U32 * dact * y64 * (np.abs(g64) + mag[rows]) + TINY
    grow, gmag, gbound = np.zeros_like(s), np.zeros_like(s), np.zeros_like(s)
    np.add.at(grow, rows, out)
    np.add.at(gmag, rows, np.abs(out))
    np.add.at(gbound, rows, bound)
    return out, bound, grow, gbound + deg[:, None] * U32 * gmag + TINY


def run_edge_softmax(dev, c):
    from cogdl_b200.operators._raw import edge_softmax_bwd_raw, edge_softmax_fwd_raw

    rp, ci, n_cols = es_graph(c)
    rng = np.random.default_rng(600 + c.H * 10 + c.chunk)
    x = es_logits(rp, c.H, rng, c.masked, c.chunk)
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    if c.op == "edge_softmax":
        got = edge_softmax_fwd_raw(st, T(x, dev) if c.aligned else misaligned(T(x, dev)))
        check_kernel(c)
        check_softmax(got.cpu().numpy(), x, rp, c.id)
    else:
        y = softmax64(rp, x)[0].astype(np.float32)
        g = rng.standard_normal(y.shape).astype(np.float32)
        got = edge_softmax_bwd_raw(st, T(y, dev), T(g, dev) if c.aligned else misaligned(T(g, dev)))
        check_kernel(c)
        ref, bound, _, _ = softmax_bwd64(rp, y, g, 1.0)
        assert_within(got.cpu().numpy(), ref, bound, c.id)
    check_counters(st, c.id)


def gat_logits32(rp, ci, hl, hr):
    """leakyrelu(h_l[row] + h_r[col]) as the kernels form it: an IEEE fp32 add, then the fp32 product with the slope."""
    rows = np.repeat(np.arange(rp.shape[0] - 1), np.diff(rp))
    z = hl[rows] + hr[ci]
    return z, np.where(z > 0, z, z * SLOPE).astype(np.float32)


def run_gat_fwd(dev, c):
    from cogdl_b200.operators._raw import gat_fwd_raw
    from tests.gat_dropout_ref import drop_below, keep_mask

    rp, ci, n = es_graph(c)
    rng = np.random.default_rng(700 + c.H * 10 + c.chunk)
    hl = rng.standard_normal((n, c.H)).astype(np.float32)
    hr = rng.uniform(-20, 90, (n, c.H)).astype(np.float32)          # logits spread over ~90 in a row
    feat = rng.standard_normal((n, c.H, c.F)).astype(np.float32)
    st = plan_structure(rp, ci, n, dev, c.plan, c.chunk)
    scale = np.float32(1.0 / (1.0 - P_DROP))
    seed = 0x5EED + c.H
    drop = (seed, drop_below(P_DROP), float(scale)) if c.drop else None
    out, att = gat_fwd_raw(st, T(hl, dev), T(hr, dev), T(feat, dev), float(SLOPE), True, drop=drop)
    check_kernel(c)
    att = att.cpu().numpy()
    check_softmax(np.abs(att), gat_logits32(rp, ci, hl, hr)[1], rp, f"{c.id} attention")
    eff = att
    if c.drop:
        keep = keep_mask(seed, ci.size, c.H, P_DROP)
        assert np.array_equal(np.signbit(att), ~keep), f"{c.id}: the sign bits are not the dropout mask"
        eff = np.where(keep, np.abs(att) * scale, np.float32(0)).astype(np.float32)
    else:
        assert not np.signbit(att).any()
    # the aggregation over the attention the kernel wrote (the multi-head SpMM bound)
    got, deg = out.cpu().numpy(), np.diff(rp)[:, None]
    for h in range(c.H):
        A = csr64(rp, ci, eff[:, h], n)
        f64 = feat[:, h, :].astype(np.float64)
        assert_within(got[:, h, :], A @ f64, deg * U32 * (abs(A) @ np.abs(f64)) + TINY, f"{c.id} head {h}")
    check_counters(st, c.id)


def run_gat_attn_bwd(dev, c):
    from cogdl_b200.operators._raw import gat_attn_bwd_raw
    from tests.gat_dropout_ref import keep_mask

    rp, ci, n = es_graph(c)
    rng = np.random.default_rng(800 + c.H * 10 + c.chunk)
    att = softmax64(rp, es_logits(rp, c.H, rng))[0].astype(np.float32)
    d_att = rng.standard_normal(att.shape).astype(np.float32)
    hl = rng.standard_normal((n, c.H)).astype(np.float32)
    hr = rng.standard_normal((n, c.H)).astype(np.float32)
    # the first edge of every row gets a pre-activation of exactly +0.0: LeakyReLU'(0) is the slope (z > 0 is the test)
    first = rp[:-1][np.diff(rp) > 0]
    hl[np.diff(rp) > 0] = -hr[ci[first]]
    z = gat_logits32(rp, ci, hl, hr)[0]
    assert np.all(z[first] == 0)
    dact = np.where(z > 0, 1.0, np.float64(SLOPE))
    st = plan_structure(rp, ci, n, dev, c.plan, c.chunk)
    y, g, ds = att, d_att, None
    if c.drop:
        scale = np.float32(1.0 / (1.0 - P_DROP))
        keep = keep_mask(0xD0 + c.H, ci.size, c.H, P_DROP)
        att = np.where(keep, att, -att).astype(np.float32)            # the dropped entries carry the sign bit
        g = np.where(keep, d_att * scale, np.float32(0)).astype(np.float32)
        ds = float(scale)
    gd = T(d_att, dev)
    d_edge, g_row = gat_attn_bwd_raw(st, T(att, dev), gd if c.aligned else misaligned(gd), T(hl, dev), T(hr, dev),
                                     float(SLOPE), drop_scale=ds)
    check_kernel(c)
    ref, bound, grow, gbound = softmax_bwd64(rp, y, g, dact)
    assert_within(d_edge.cpu().numpy(), ref, bound, f"{c.id} d_edge")
    assert_within(g_row.cpu().numpy(), grow, gbound, f"{c.id} g_row")
    check_counters(st, c.id)


RUN = {"spmm": run_spmm, "spmm_f16": run_spmm_f16, "sddmm": run_sddmm, "mhspmm": run_mhspmm,
       "scatter_max": run_scatter_max, "scatter_max_bwd": run_scatter_max, "edge_softmax": run_edge_softmax,
       "edge_softmax_bwd": run_edge_softmax, "gat_fwd": run_gat_fwd, "gat_attn_bwd": run_gat_attn_bwd}


@pytest.mark.parametrize("c", TABLE, ids=lambda c: c.id)
def test_dispatch_row(dev, c):
    RUN[c.op](dev, c)


# ------------------------------------------------------------------------------------------ last_kernel() follows
def test_last_kernel_names_sddmm_and_fp16_calls(dev):
    """After an SDDMM and after an fp16 SpMM, cogdl_b200_last_kernel() names that call's kernel, not the one of the
    fp32 SpMM before it."""
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import mhsddmm_raw, sddmm_raw, spmm_raw
    from cogdl_b200.structure import CSRStructure

    rp, ci, n_cols = case("hub")
    st = CSRStructure(T(rp, dev), T(ci, dev), n_cols=n_cols)
    x = torch.randn(n_cols, 128, device=dev)
    spmm_raw(st, None, x)
    assert _cabi.last_kernel().startswith("cogdl_b200::stream_kernel<")
    sddmm_raw(st, torch.randn(n_cols, 128, device=dev), x)
    assert _cabi.last_kernel() == "cogdl_b200::sddmm_stream_kernel<NV=1,U=4>", _cabi.last_kernel()
    spmm_raw(st, None, x)
    mhsddmm_raw(st, torch.randn(n_cols, 3, 8, device=dev), torch.randn(n_cols, 3, 8, device=dev))
    assert _cabi.last_kernel() == "cogdl_b200::sddmm_kernel<float4,GROUP=4,SUB=2,NV=1>", _cabi.last_kernel()
    spmm_raw(st, None, x)
    spmm_raw(st, torch.rand(ci.shape[0], device=dev).half(), x.half())
    assert _cabi.last_kernel() == "cogdl_b200::spmm_half_kernel<weighted,vec>", _cabi.last_kernel()


# ------------------------------------------------------------------------------------------ fp16 autograd
@pytest.mark.parametrize("sym", [False, True])
def test_fp16_csrspmm_autograd(dev, sym):
    """csrspmm on fp16 features with edge weights that require grad: out, grad_feat (A^T @ g, through the cached
    transpose or, with sym, the CSR itself) and grad_w (SDDMM in fp32, cast to fp16) against fp64 over the
    fp16-rounded inputs."""
    from cogdl_b200.operators.spmm import csrspmm
    from cogdl_b200.structure import CSRStructure

    rp, ci, n = case("two_hubs")
    rng = np.random.default_rng(31)
    w = rng.random(ci.shape[0])
    if sym:
        S = csr64(rp, ci, w, n)
        S = (S + S.T).tocsr()
        S.sort_indices()
        rp, ci, w = S.indptr.astype(np.int32), S.indices.astype(np.int32), S.data
    w16 = w.astype(np.float16)
    F = 64
    X16 = rng.standard_normal((n, F)).astype(np.float16)
    g16 = rng.standard_normal((n, F)).astype(np.float16)
    st = CSRStructure(T(rp, dev), T(ci, dev), n_cols=n)
    x = T(X16, dev).requires_grad_(True)
    wd = T(w16, dev).requires_grad_(True)
    y = csrspmm(st, None, x, wd, sym)
    y.backward(T(g16, dev))
    assert y.dtype == x.grad.dtype == wd.grad.dtype == torch.float16

    A = csr64(rp, ci, w16.astype(np.float64), n)
    X, g = X16.astype(np.float64), g16.astype(np.float64)
    ref = A @ X
    assert_within(y.detach().cpu().numpy(), ref, fp16_bound(ref, abs(A) @ np.abs(X), np.diff(rp)[:, None]), "out")
    gf = A.T @ g
    coldeg = np.bincount(ci, minlength=n)[:, None]
    assert_within(x.grad.cpu().numpy(), gf, fp16_bound(gf, abs(A).T @ np.abs(g), coldeg), "grad_feat")
    rows = np.repeat(np.arange(n), np.diff(rp))
    terms = g[rows] * X[ci]
    gw = terms.sum(1)
    assert_within(wd.grad.cpu().numpy(), gw, fp16_bound(gw, np.abs(terms).sum(1), F), "grad_w")

"""Every dispatch branch of the SpMM (fp32 and fp16), SDDMM, multi-head SpMM and scatter_max entry points, one
row of tests/dispatch_table.py each: the call must record exactly the kernel the row names, and its output must
match a reference.

- fp32 SpMM: rows the hub plan does not split are bit-identical to the oracle (CSR order, separate fp32 multiply
  and add); every element is within the fp64 bound below.
- scatter_max: values and argmax equal the oracle's, ties included (quantised inputs).
- SDDMM, multi-head SDDMM and multi-head SpMM: per element, |got - ref| <= n * 2^-24 * sum|terms| + tiny against an
  fp64 evaluation, n the number of terms (row degree or dot length).  A bound relative to the largest output would
  let a row of small values be wrong by a large relative amount.
- fp16 SpMM: fp64 over the fp16-rounded inputs, bound 2^-11 |ref| + deg * 2^-24 * sum|v x| + 2^-24 (one fp16
  rounding of the output plus the fp32 accumulation), with outputs in the fp16 subnormal range and a row whose
  terms cancel exactly.
"""
import ctypes

import numpy as np
import pytest
import scipy.sparse as sp
import torch

import oracle
from tests.dispatch_table import TABLE
from tests.graphs import case

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24                      # unit roundoff of fp32
TINY = float(np.finfo(np.float32).tiny)


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import cogdl_b200

    assert cogdl_b200._cabi.load().cogdl_b200_check_device() == 0, cogdl_b200._cabi.last_error()
    return torch.device("cuda:0")


def T(a, dev):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def misaligned(t):
    """A contiguous copy of t whose data starts one element past the allocation (not 16-byte aligned)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    out = buf[1:].view(t.shape)
    out.copy_(t)
    return out


def structure(rp, ci, n_cols, dev, c):
    from cogdl_b200.structure import CSRStructure

    chunk, seg_cost = {"none": (0, None), "chunks": (c.chunk, 0), "default": (c.chunk, None)}[c.plan]
    return CSRStructure(T(rp, dev), T(ci, dev), n_cols=n_cols, chunk_edges=chunk, seg_cost=seg_cost)


def csr64(rp, ci, vals, n_cols):
    # copies: abs() of a scipy CSR sorts its indices in place, which must not reorder the caller's colind
    return sp.csr_matrix((np.array(vals, np.float64), ci.copy(), rp.copy()), shape=(rp.shape[0] - 1, n_cols))


def assert_within(got, ref, bound, what):
    err = np.abs(np.asarray(got, np.float64) - ref)
    bad = np.argwhere(~(err <= bound))
    assert bad.size == 0, (f"{what}: {len(bad)} elements outside the bound, first at {tuple(bad[0])}: "
                           f"got {got[tuple(bad[0])]!r}, ref {ref[tuple(bad[0])]!r}, bound {bound[tuple(bad[0])]!r}")


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
    from cogdl_b200.structure import _ptr, _stream

    bounds, shift = [0, 400, 700, n_cols], 9
    enc = ci.copy()
    for o in (1, 2):
        m = (ci >= bounds[o]) & (ci < bounds[o + 1])
        enc[m] = bounds[1] + (o << shift) + (ci[m] - bounds[o])
    st = structure(rp, enc, n_cols, dev, c)
    shards = [T(X[bounds[o]:bounds[o + 1]], dev) for o in range(3)]
    ptrs = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in shards])
    y = torch.empty((rp.shape[0] - 1, c.F), device=dev)
    plan, keep = st.plan_struct(st.plan.n_chunks * c.F * 4 + 16)
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
        st = structure(rp, ci, n_cols, dev, c)
        y = spmm_raw(st, val_d, Xd, panels=c.panels)
    elif c.src == "two":
        st = structure(rp, ci, n_cols, dev, c)
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
    st = structure(rp, ci, n_cols, dev, c)
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
    st = structure(rp, ci, n_cols, dev, c)
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
    st = structure(rp, ci, n_cols, dev, c)
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
    st = structure(rp, ci, n_cols, dev, c)
    Xd = T(X, dev) if c.aligned else misaligned(T(X, dev))
    out, arg = scatter_max_fwd_raw(st, Xd)
    check_kernel(c)
    assert np.array_equal(out.cpu().numpy(), ref), f"{c.id}: max differs"
    assert np.array_equal(arg.cpu().numpy(), ref_id), f"{c.id}: argmax differs"
    if c.plan != "none":
        assert st.plan.n_chunks > 0 and int(st.plan.counters.abs().sum()) == 0


RUN = {"spmm": run_spmm, "spmm_f16": run_spmm_f16, "sddmm": run_sddmm, "mhspmm": run_mhspmm,
       "scatter_max": run_scatter_max, "scatter_max_bwd": run_scatter_max}


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

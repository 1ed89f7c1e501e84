"""GENConv edge-encoder kernels (cogdl_b200/csrc/genconv_edge.cu) and genconv_aggregate(edge_attr=, edge_weight=)
against the fp64 restatement of tests/genconv_ref.py with edge_term = attr @ W.T, against the edge-term kernels bit
for bit where the product is exact, and the reference DeeperGCN with an EdgeEncoder through install(genconv=True).

Every row of tests/genconv_edge_table.py is checked per element (test_table_row), with u = 2^-24:
- The kernel forms the edge term as one fmaf chain of D steps from 0, A32 = fl(attr @ W.T).  In the exact family
  (attr in {-2..2}, W a power of two times multiples of 1/8) every partial sum is exact, so A32 = attr @ W.T and the
  bounds of the edge-term kernel (tests/test_gpu_dispatch_message.py: sa_fwd64 for out, lse2 and Q, run_sa_bwd's
  terms for dX) apply unchanged to the fp32 m = relu(x[c] + A32) + eps.  For one edge per column (columns not a
  multiple of 7, whose x rows are 0) x[c] = -A_e, so that edge's pre-activation is exactly 0 and it adds nothing to dX
  or dW (ReLU'(0) = 0).  x spreads beta m over at least 60 in every row; beta in {0, 0.5, 4, 20, -2}.
- In the general family (attr ~ U[0, 1), W ~ N(0, 1/D)) the reference takes A = fl(attr @ W.T in fp64); the kernel's A
  is within dA = (D + 1) u sum_d |attr W| of it, its pre-activation within dpre = dA + 2u (|pre| + dA) (two adds
  rounded apart), its m within dm = dpre + 2u (m + dpre), and dm = 0 where pre <= -dpre (both sides give m = eps).
  With Dm the row's largest dm, each logit moves by at most |beta| log2(e) Dm in base 2, each normalised weight by
  k = 2 |beta| Dm relative (once its own, once the normaliser): out gains k (out64 + Dm) + Dm, Q gains
  k Q' + (Q' - Q64) with Q' = Q64 + 2 Dm out64 + Dm^2, lse2 gains |beta| log2(e) Dm.  Backward: the weight
  2^(z - lse2) and the factor 1 + beta (m - out) each move by |beta| dm, so dpre_e gains |beta| dm (mag_e + w_e |g_i|);
  an edge whose pre-activation is within dpre of 0 may change sides of the ReLU and counts its whole magnitude.
- dW[f, d] = sum_e dpre_e[f] attr[e, d]: each term carries the dpre bound times |attr|, and the fp32 sum has a depth of
  L + 8 + B + 2 (u times sum |dpre attr|), not nnz: B = min(ceil(items / 8), 264) blocks summed in block order, 8
  warps in warp order, and one lane's fmaf chain of at most L = ceil(items / (8 B)) x (edges of one item) products,
  items = the transpose's hub chunks + its columns.  The wide graph has more items than the grid has warps (every
  warp carries its dW partial into a second item); its dX and dW must also be bit-identical run to run.
The worst error / bound ratio of every check is printed."""
import json
import os
import subprocess
import sys
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from tests import graphs
from tests.genconv_edge_table import GE_BWD_BLOCKS, GE_WARPS, TABLE, wide_csr
from tests.genconv_ref import genconv_aggregate_fp64
from tests.gpu_util import check_counters, dev, misaligned, row_err
from tests.test_gpu_dispatch_message import (EPS, LN2, LOG2E, RATIOS, TINY, U32, assert_within, col_sum, edge_rows,
                                             sa_fwd64, sa_inputs, sa_m, seg_reduce)
from tests.test_gpu_genconv import structure

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOFTMAX_AGGRS = ("softmax_sg", "softmax", "mean", "sum")


def operands(st, F, D, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(st.n_cols, F, device=dev, generator=g)
    attr = torch.rand(st.nnz, D, device=dev, generator=g)
    w = torch.randn(F, D, device=dev, generator=g) / D ** 0.5
    return x, attr, w


def fp64(st, x, attr, w, aggr, beta=1.0):
    return genconv_aggregate_fp64(st.rowptr, st.colind, x, aggr, beta=beta, edge_term=attr.double() @ w.double().T)


@pytest.mark.parametrize("chunk", [None, 16])
@pytest.mark.parametrize("D", [1, 3, 8, 16])
@pytest.mark.parametrize("F", [7, 16, 64, 128, 256])
@pytest.mark.parametrize("name", list(graphs.CASES))
def test_forward_matches_fp64(dev, name, F, D, chunk):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev, chunk)
    x, attr, w = operands(st, F, D, dev, seed=F + D)
    for beta in (0.0, 0.5, 1.0, 4.0):
        got = genconv_aggregate(st, x, "softmax_sg", beta=beta, edge_attr=attr, edge_weight=w)
        assert got.shape == (st.n_rows, F)
        assert row_err(got, fp64(st, x, attr, w, "softmax_sg", beta)) <= 1e-5, f"beta={beta}"
    for aggr in ("softmax", "mean", "sum"):
        got = genconv_aggregate(st, x, aggr, edge_attr=attr, edge_weight=w)
        assert row_err(got, fp64(st, x, attr, w, aggr)) <= 1e-5, aggr


def q_fp64(st, x, attr, w, beta, eps=1e-7):
    """Q[i] = sum_e w_e m_e^2 in fp64 (the forward's d beta operand); 0 on degree-0 rows."""
    rp, ci = st.rowptr.long(), st.colind.long()
    n, F = st.n_rows, x.shape[1]
    row = torch.repeat_interleave(torch.arange(n, device=rp.device), rp[1:] - rp[:-1])
    m = torch.relu(x.double()[ci] + attr.double() @ w.double().T) + eps
    z = beta * m
    zmax = torch.full((n, F), -torch.inf, dtype=torch.float64, device=m.device).scatter_reduce(
        0, row[:, None].expand(-1, F), z, "amax")
    ex = torch.exp(z - zmax[row])
    zeros = torch.zeros(n, F, dtype=torch.float64, device=m.device)
    return zeros.index_add(0, row, ex * m * m) / zeros.index_add(0, row, ex).clamp_min(1e-300)


def _grads(fn, x, w, beta, r, dtype, need_x=True, need_w=True, need_b=True):
    xs = x.clone().to(dtype).requires_grad_(need_x)
    ws = w.clone().to(dtype).requires_grad_(need_w)
    bs = beta.clone().to(dtype).requires_grad_(need_b)
    out = fn(xs, ws, bs)
    (out * r.to(dtype)).sum().backward()
    return out.detach(), xs.grad, ws.grad, bs.grad


@pytest.mark.parametrize("aggr", SOFTMAX_AGGRS)
@pytest.mark.parametrize("name", ["ragged", "hub", "two_hubs", "rect"])
def test_gradients_match_fp64_autograd(dev, name, aggr):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev)
    F, D = 64, 8
    x, attr, w = operands(st, F, D, dev, seed=11)
    r = torch.randn(st.n_rows, F, device=dev, generator=torch.Generator(device=dev).manual_seed(12))
    beta = torch.full((1,), 1.5, device=dev)
    need_b = aggr == "softmax_sg"

    def mine(x_, w_, b_):
        return genconv_aggregate(st, x_, aggr, beta=b_, edge_attr=attr, edge_weight=w_)

    def exact(x_, w_, b_):
        return genconv_aggregate_fp64(st.rowptr, st.colind, x_, aggr, beta=b_, edge_term=attr.double() @ w_.T)

    want = _grads(exact, x, w, beta, r, torch.float64, need_b=need_b)
    got = _grads(mine, x, w, beta, r, torch.float32, need_b=need_b)
    assert row_err(got[1], want[1]) <= 1e-4
    assert row_err(got[2], want[2]) <= 1e-4
    if need_b:
        assert row_err(got[3], want[3]) <= 1e-4
    else:
        assert got[3] is None
    # only W needs grad: no dx; only x: no dW (and the frozen W costs no dW pass)
    only_w = _grads(mine, x, w, beta, r, torch.float32, need_x=False, need_b=False)
    assert only_w[1] is None and row_err(only_w[2], want[2]) <= 1e-4
    assert torch.equal(only_w[2], got[2])
    only_x = _grads(mine, x, w, beta, r, torch.float32, need_w=False, need_b=False)
    assert only_x[2] is None and torch.equal(only_x[1], got[1])


@pytest.mark.parametrize("aggr", SOFTMAX_AGGRS)
@pytest.mark.parametrize("F", [7, 128, 256])
@pytest.mark.parametrize("name", ["hub", "two_hubs", "rect"])
def test_bit_identical_to_edge_term_kernels(dev, name, F, aggr):
    """attr in {-2..2} and W in multiples of 1/8 make attr @ W.T exact in fp32 in any order: out and dx equal the
    edge-term kernels' bit for bit, dW is within 1e-5 of d_edge_term.T @ attr."""
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev, 16)
    D = 8
    g = torch.Generator(device=dev).manual_seed(F)
    x = torch.randn(st.n_cols, F, device=dev, generator=g)
    attr = torch.randint(-2, 3, (st.nnz, D), device=dev, generator=g).float()
    w = torch.randint(-8, 9, (F, D), device=dev, generator=g).float() / 8
    r = torch.randn(st.n_rows, F, device=dev, generator=g)
    beta = 0.7 if aggr == "softmax_sg" else None

    xa = x.clone().requires_grad_(True)
    wa = w.clone().requires_grad_(True)
    out_a = genconv_aggregate(st, xa, aggr, beta=beta, edge_attr=attr, edge_weight=wa)
    (out_a * r).sum().backward()
    xb = x.clone().requires_grad_(True)
    term = (attr @ w.T).requires_grad_(True)
    out_b = genconv_aggregate(st, xb, aggr, beta=beta, edge_term=term)
    (out_b * r).sum().backward()
    assert torch.equal(out_a, out_b)
    assert torch.equal(xa.grad, xb.grad)
    assert row_err(wa.grad, term.grad.T.double() @ attr.double()) <= 1e-5


@pytest.mark.parametrize("name", ["hub", "two_hubs"])
def test_forward_backward_bitwise_reproducible(dev, name):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev, 16)
    x0, attr, w0 = operands(st, 128, 8, dev, seed=5)
    r = torch.randn(st.n_rows, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(6))

    def once():
        x, w = x0.clone().requires_grad_(True), w0.clone().requires_grad_(True)
        b = torch.full((1,), 0.8, device=dev, requires_grad=True)
        out = genconv_aggregate(st, x, "softmax_sg", beta=b, edge_attr=attr, edge_weight=w)
        (out * r).sum().backward()
        return out.detach(), x.grad, w.grad, b.grad

    first, second = once(), once()
    assert all(torch.equal(u, v) for u, v in zip(first, second))


def _row_graph(c):
    if c.graph == "bounds":
        return graphs.boundary_csr(c.chunk)
    if c.graph == "bounds_t":
        return graphs.boundary_csc(c.chunk)
    if c.graph == "wide":
        return wide_csr()
    return graphs.case(c.graph)


def _row_inputs(c, rp, ci, n_cols):
    """x [n_cols, F], attr [nnz, D], W [F, D] (fp32 numpy) of the row's input family, the reference edge term A (fp32)
    and the bound dA of the kernel's A against it (0 in the exact family)."""
    rng = np.random.default_rng(c.F * 17 + c.D + (7919 if c.family == "exact" else 0))
    x, _ = sa_inputs(SimpleNamespace(F=c.F, beta=abs(c.beta), edge_term=False), rp, ci, n_cols, rng)
    nnz = ci.size
    if c.family == "exact":
        top = 3.0 if c.beta == 0 else max(3.0, 70.0 / abs(c.beta))
        s = 2.0 ** np.floor(np.log2(max(top / (2 * c.D ** 0.5), 1.0)))   # A spreads about as x does
        attr = rng.integers(-2, 3, (nnz, c.D)).astype(np.float32)
        w = (rng.integers(-8, 9, (c.F, c.D)) * (s / 8)).astype(np.float32)
        A = (attr.astype(np.float64) @ w.astype(np.float64).T).astype(np.float32)
        cols, first = np.unique(ci, return_index=True)
        pick = cols % 7 != 0
        x[cols[pick]] = -A[first[pick]]                   # that edge's pre-activation is exactly 0
        return x, attr, w, A, np.zeros_like(A, np.float64)
    attr = rng.random((nnz, c.D)).astype(np.float32)
    w = (rng.standard_normal((c.F, c.D)) / c.D ** 0.5).astype(np.float32)
    a64, w64 = attr.astype(np.float64), w.astype(np.float64)
    return x, attr, w, (a64 @ w64.T).astype(np.float32), (c.D + 1) * U32 * (np.abs(a64) @ np.abs(w64).T)


def _m_error(pre, m, dA):
    """Per-edge bound on |m_kernel - m| from the edge term's dA (module docstring), and the edges that may change
    sides of the ReLU."""
    dpre = dA + 2 * U32 * (np.abs(pre) + dA)
    dm = np.where((pre <= -dpre) | (dA == 0), 0.0, dpre + 2 * U32 * (m + dpre))
    return dm, (np.abs(pre) <= dpre) & (dA > 0)


def _fwd_call(c, st, xd, attr, w, beta_d, dev):
    """The forward through genconv_edge_fwd_raw, or with c.partials_offset straight through the C entry point with the
    plan's partial scratch shifted off 16-byte alignment (as test_gpu_dispatch_message.sa_fwd_call does)."""
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import _sa_scratch, genconv_edge_fwd_raw
    from cogdl_b200.structure import _ptr, _stream

    if not c.partials_offset:
        return genconv_edge_fwd_raw(st, xd, attr, w, beta_d, EPS, want_lse=True, want_q=c.want_q)
    assert st.plan.n_chunks > 0, f"{c.id}: the partials offset only matters with hub chunks"
    out = torch.empty((st.n_rows, c.F), device=dev)
    lse2, q = torch.empty_like(out), (torch.empty_like(out) if c.want_q else None)
    plan, keep = st.plan_struct(_sa_scratch(st, c.F) + 16)
    keep[0].partials += c.partials_offset
    keep[0].partials_bytes -= c.partials_offset
    _cabi.call("cogdl_b200_genconv_edge_fwd_f32", _ptr(st.rowptr), _ptr(st.colind), _ptr(xd), _ptr(attr), _ptr(w),
               c.D, _ptr(beta_d), float(EPS), _ptr(out), _ptr(lse2), _ptr(q), st.n_rows, c.F, plan, _stream(dev))
    torch.cuda.synchronize(dev)
    del keep
    return out, lse2, q


def _bwd_call(c, st, xd, attr, w, beta_d, g, out, lse2, dev):
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import _scratch, genconv_edge_bwd_raw
    from cogdl_b200.structure import _ptr, _stream

    if not c.partials_offset:
        return genconv_edge_bwd_raw(st, xd, attr, w, beta_d, EPS, g, out, lse2, want_dx="dx" in c.want,
                                    want_dw="dw" in c.want)
    assert c.want == "dx", "the plan's partial scratch is used by dX only"
    st_t, perm = st.csc()
    assert st_t.plan.n_chunks > 0, f"{c.id}: the partials offset only matters with hub chunks"
    dx = torch.empty_like(xd)
    plan, keep = st_t.plan_struct(_scratch("genconv_edge_bwd", st_t, c.F, 1) + 16)
    keep[0].partials += c.partials_offset
    keep[0].partials_bytes -= c.partials_offset
    _cabi.call("cogdl_b200_genconv_edge_bwd_f32", _ptr(st_t.rowptr), _ptr(st_t.colind), _ptr(perm), _ptr(xd),
               _ptr(attr), _ptr(w), c.D, _ptr(beta_d), float(EPS), _ptr(g), _ptr(out), _ptr(lse2), _ptr(dx), None,
               None, 0, st_t.n_rows, c.F, plan, _stream(dev))
    torch.cuda.synchronize(dev)
    del keep
    return dx, None


def _check_fwd(c, rp, out, lse2, q, m, dm):
    out64, lse64, Q64, E, deg = sa_fwd64(rp, m, c.beta)
    Dm = seg_reduce(np.maximum, dm, rp)
    k = 2.01 * abs(c.beta) * Dm
    assert_within(out.cpu().numpy(), out64, out64 * (2 * E + (2 * deg + 1) * U32) + k * (out64 + Dm) + Dm + TINY,
                  f"{c.id} out")
    assert_within(lse2.cpu().numpy(), lse64, (E + deg * U32) * LOG2E + 2.0 ** -21 + 2 * U32 * np.abs(lse64)
                  + abs(c.beta) * LOG2E * Dm, f"{c.id} lse2")
    if c.want_q:
        Qp = Q64 + 2 * Dm * out64 + Dm ** 2
        assert_within(q.cpu().numpy(), Q64, Q64 * (2 * E + (2 * deg + 3) * U32) + k * Qp + (Qp - Q64) + TINY,
                      f"{c.id} Q")
    else:
        assert q is None
    empty = np.diff(rp) == 0
    assert np.all(out.cpu().numpy()[empty] == 0) and np.all(lse2.cpu().numpy()[empty] == 0)


def _check_bwd(c, st, rp, ci, n, attr, g, out, lse2, dx, dw, pre, m, dm, flip):
    """dX and dW against fp64 on the kernel's out and lse2 (run_sa_bwd's terms, plus the edge term's and dW's)."""
    beta = c.beta
    rows = edge_rows(rp)
    o32, l32 = out.cpu().numpy().astype(np.float64), lse2.cpu().numpy().astype(np.float64)
    z = beta * LOG2E * m.astype(np.float64)
    arg = z - l32[rows]
    wgt = np.exp2(arg)
    dev_m = np.abs(m - o32[rows])
    live = pre > 0
    dpre = np.where(live, wgt * g[rows] * (1 + beta * (m - o32[rows])), 0.0)
    full = wgt * np.abs(g[rows]) * (1 + abs(beta) * dev_m)
    mag = np.where(live, full, 0.0)
    eb = mag * (2.0 ** -22 + LN2 * U32 * (3 * np.abs(z) + np.abs(arg)) + 4 * U32)
    eb = eb + np.where(live, 1.01 * abs(beta) * dm * (mag + wgt * np.abs(g[rows])), 0.0)
    eb = eb + np.where(flip, 1.01 * full * (1 + abs(beta) * dm) + dm, 0.0)
    coldeg = np.bincount(ci, minlength=n).astype(np.float64)[:, None]
    if "dx" in c.want:
        assert_within(dx.cpu().numpy(), col_sum(dpre, ci, n),
                      col_sum(eb, ci, n) + coldeg * U32 * col_sum(mag, ci, n) + TINY, f"{c.id} dX")
    else:
        assert dx is None
    if "dw" in c.want:
        st_t, _ = st.csc()
        n_chunks = st_t.plan.n_chunks if st_t.chunk_edges > 0 else 0
        items = n_chunks + n
        B = min(-(-items // GE_WARPS), GE_BWD_BLOCKS)
        per_item = st_t.chunk_edges if st_t.chunk_edges > 0 else int(coldeg.max(initial=0))
        L = -(-items // (GE_WARPS * B)) * per_item
        a64 = np.abs(attr.astype(np.float64))
        assert_within(dw.cpu().numpy(), dpre.T @ attr.astype(np.float64),
                      eb.T @ a64 + (L + GE_WARPS + B + 2) * U32 * (mag.T @ a64) + TINY, f"{c.id} dW")
    else:
        assert dw is None


@pytest.mark.parametrize("c", TABLE, ids=[c.id for c in TABLE])
def test_table_row(dev, c):
    """Every row: records its instantiation's name, every output element lies within the bound of the module
    docstring, and the hub plans' arrival counters are back at zero."""
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import genconv_edge_fwd_raw
    from cogdl_b200.structure import DEFAULT_CHUNK_EDGES, CSRStructure

    RATIOS.clear()
    rp, ci, n = _row_graph(c)
    x, attr, w, A, dA = _row_inputs(c, rp, ci, n)
    st = CSRStructure(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), n_cols=n,
                      chunk_edges=(c.chunk or DEFAULT_CHUNK_EDGES) if c.plan else 0)
    xd = torch.from_numpy(x).to(dev)
    if not c.aligned:    # 4 bytes off 16-byte alignment: the scalar kernel
        xd = misaligned(xd)
    attr_d, w_d = torch.from_numpy(attr).to(dev), torch.from_numpy(w).to(dev)
    beta_d = torch.tensor([c.beta], dtype=torch.float32, device=dev)
    pre, m = sa_m(x, A, ci)
    if c.family == "exact":
        cols, first = np.unique(ci, return_index=True)
        assert np.all(pre[first[cols % 7 != 0]] == 0)
    dm, flip = _m_error(pre, m, dA)
    if c.op == "fwd":
        out, lse2, q = _fwd_call(c, st, xd, attr_d, w_d, beta_d, dev)
        if st.n_rows and c.F:
            assert _cabi.last_kernel() == c.kernel
        if c.graph.startswith("bounds") or c.partials_offset:
            assert st.plan.n_chunks > 0
        _check_fwd(c, rp, out, lse2, q, m, dm)
        check_counters(st, c.id)
    else:
        out, lse2, _ = genconv_edge_fwd_raw(st, xd, attr_d, w_d, beta_d, EPS, want_lse=True)
        g = np.random.default_rng(3 + c.F).standard_normal((st.n_rows, c.F)).astype(np.float32)
        gd = torch.from_numpy(g).to(dev)
        dx, dw = _bwd_call(c, st, xd, attr_d, w_d, beta_d, gd, out, lse2, dev)
        if st.n_cols and c.F:
            assert _cabi.last_kernel() == c.kernel
        st_t, _ = st.csc()
        if c.graph.startswith("bounds") or c.graph == "wide" or c.partials_offset:
            assert st_t.plan.n_chunks > 0
        if c.graph == "wide":
            assert st_t.plan.n_chunks + n > GE_WARPS * GE_BWD_BLOCKS
            again = _bwd_call(c, st, xd, attr_d, w_d, beta_d, gd, out, lse2, dev)
            for a, b in zip((dx, dw), again):
                assert (a is None and b is None) or torch.equal(a, b), f"{c.id}: not reproducible"
        _check_bwd(c, st, rp, ci, n, attr, g, out, lse2, dx, dw, pre, m, dm, flip)
        check_counters(st, c.id)
        check_counters(st_t, c.id)
    print(" ".join(f"[{k}: worst err/bound {v:.3g}]" for k, v in RATIOS.items()))


def test_no_edge_sized_tensor(dev):
    """Arxiv shape, F = 128, D = 8: beyond the three [N, F] tensors the operator has to hold (out, the saved lse2,
    then dx), forward + backward grow max_memory_allocated by less than a quarter of one [nnz, F] tensor; and the
    forward is within 1e-5 of fp64 evaluated on the GPU.  (At arxiv's mean degree of 7.9 one [N, F] tensor is an
    eighth of an [nnz, F] one, so the node-sized tensors are counted out rather than hidden in the bound; beta is a
    constant here, as the dense d beta reduction adds node-sized temporaries of its own.)"""
    from cogdl_b200 import genconv_aggregate, synth
    from cogdl_b200.structure import CSRStructure

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, device=dev, self_loops=True)
    st = CSRStructure.from_int64(rp, col)
    del rp, col
    F, D = 128, 8
    x, attr, w = operands(st, F, D, dev, seed=0)
    st.plan, st.csc()[0].plan                          # structure built before the measurement
    xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    beta = torch.ones(1, device=dev)
    r = torch.randn(st.n_rows, F, device=dev)
    with torch.no_grad():
        genconv_aggregate(st, x, "softmax_sg", beta=1.0, edge_attr=attr, edge_weight=w)   # plan scratch sized
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = genconv_aggregate(st, xg, "softmax_sg", beta=beta, edge_attr=attr, edge_weight=wg)
    out.backward(r)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base - 3 * st.n_rows * F * 4
    assert growth < st.nnz * F * 4 / 4, (growth, st.nnz * F * 4)
    assert xg.grad is not None and wg.grad is not None
    with torch.no_grad():
        got = genconv_aggregate(st, x, "softmax_sg", beta=1.0, edge_attr=attr, edge_weight=w)
    assert row_err(got, fp64(st, x, attr, w, "softmax_sg", 1.0)) <= 1e-5


def test_errors(dev):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure("tiny", dev)
    x, attr, w = operands(st, 8, 3, dev)
    with pytest.raises(ValueError):      # both an edge term and edge features
        genconv_aggregate(st, x, "softmax", edge_term=attr @ w.T, edge_attr=attr, edge_weight=w)
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr)
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_weight=w)
    with pytest.raises(ValueError):      # nnz mismatch
        genconv_aggregate(st, x, "softmax", edge_attr=attr[:-1], edge_weight=w)
    with pytest.raises(ValueError):      # W not [F, D]
        genconv_aggregate(st, x, "softmax", edge_attr=attr, edge_weight=w.T.contiguous())
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr[:, 0], edge_weight=w)
    wide = torch.rand(st.nnz, 17, device=dev)
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_attr=wide, edge_weight=torch.randn(8, 17, device=dev))
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr.clone().requires_grad_(True), edge_weight=w)
    with pytest.raises(RuntimeError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr.cpu(), edge_weight=w)
    with pytest.raises(TypeError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr.double(), edge_weight=w)
    for aggr in ("max", "powermean"):
        with pytest.raises(NotImplementedError):
            genconv_aggregate(st, x, aggr, edge_attr=attr, edge_weight=w)


def test_reference_deepergcn_with_edge_encoder_through_install():
    """Reference DeeperGCN (softmax_sg, learnable beta, edge_attr_size=[8]) and a lone GENConv with an EdgeEncoder
    through install(genconv=True), in a child process (tests/genconv_edge_refpkg_check.py)."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.genconv_edge_refpkg_check"], cwd=ROOT, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for name in ("deepergcn", "genconv_edge"):
        m = res[name]
        assert m["logits_vs_ref_cpu"] <= 1e-4, (name, m)
        assert m["logits_vs_fp64"] <= 1e-4, (name, m)
        assert m["grads_present"], (name, m)
        assert m["edge_encoder_calls"] == 0, (name, m)
        assert "genconv_edge_" in m["last_kernel"], (name, m)
    assert max(res["genconv_edge"]["grad_errs"].values()) <= 1e-4, res["genconv_edge"]
    assert max(res["deepergcn"]["grad_errs_model_scale"].values()) <= 1e-3, res["deepergcn"]
    for case in ("bond_encoder", "attr_requires_grad"):
        assert res[case]["edge_term_kernel"], (case, res[case])

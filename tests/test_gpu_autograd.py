"""The autograd layer above the kernels, per element against fp64 on the host.

1. The Functions (SPMMFunction, EdgeSoftmaxFunction, MHSPMMFunction, ScatterMaxFunction, FusedGATFunction without
   dropout) on tests/graphs.py CASES and on boundary_csr(64) under a 64-edge hub plan, so the transpose the backward
   walks has hub chunks of its own.  Each input that can take a gradient requires it or not (every subset); the
   incoming gradient is contiguous, the stride-0 tensor `out.sum().backward()` gives, or a strided view; the feature
   input is contiguous, a strided view, or misaligned by one element.  A gradient nobody asked for comes back None
   from the Function's own backward.
2. The graph-level entry points (spmm fp32 / fp16, edge_softmax, mh_spmm, fused_gat_op, spmm_residual) on each square
   graph built from (row_ptr, col), from edge_index in CSR order and from edge_index under a seeded edge permutation
   with the weights permuted along, crossed with no / fixed / trainable weights and no / sym / row normalisation.
   Two calls on a fresh graph are bit-identical, and both are checked against fp64 built from the user's own COO
   triplets; a trainable weight gets its gradient back in the user's order.
3. GCNLayer, SAGELayer, GATLayer (fused and unfused) and fused_sage_layer on a shuffled COO graph against the same
   layer on its twin, the graph built from the stable row sort of the same edges: bit-identical outputs and gradients.

Bounds.  The fp64 reference is evaluated from the exact fp32 values the kernels read (weights after normalisation,
out_norm * x as fp32 forms it).  A sum of k terms, followed by m fp32 products (in_norm, the residual scale a, the
normalisation factors of a trainable weight) is held per element to (k + 2 + m) 2^-24 sum|terms|: each term passes
through at most k roundings in the sum, plus one per product.  The softmax and GAT bounds are those of
tests/test_gpu_dispatch.py (softmax64, softmax_bwd64); where the softmax backward reads an fp32 SDDMM result, that
result's own bound b is carried through it as dact y (b + sum_row y b).  fp16 SpMM uses the dispatch fp16 bound.
"""
import copy
import json
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.gpu_util import T, dev, misaligned, plan_structure
from tests.graphs import CASES, boundary_csr, case
from tests.test_gpu_dispatch import (SLOPE, TINY, U32, assert_within, check_softmax, es_logits, fp16_bound,
                                     gat_logits32, softmax_bwd64)

pytestmark = pytest.mark.gpu

GRAPHS = list(CASES) + ["bounds"]
SQUARE = [g for g in GRAPHS if g != "rect"]
# (incoming gradient, feature layout): each kind of either occurs once
MODES = [("rand", "contig"), ("sum", "view"), ("view", "misaligned")]


WORST = {}      # test function -> largest |got - ref| / bound seen


@pytest.fixture(scope="module", autouse=True)
def _report_worst_ratio():
    yield
    print("\nworst error / bound per test function: " + json.dumps({k: float(f"{v:.3g}") for k, v in WORST.items()}))


def within(got, ref, bnd, what):
    """assert_within, recording the largest error-to-bound ratio of the calling test function."""
    assert_within(got, ref, bnd, what)
    err = np.abs(np.asarray(got, np.float64) - ref)
    bnd = np.broadcast_to(bnd, err.shape)
    ratio = float(np.max(np.where(bnd > 0, err / np.where(bnd > 0, bnd, 1), 0))) if err.size else 0.0
    test = os.environ.get("PYTEST_CURRENT_TEST", "?").split("::")[-1].split("[")[0]
    WORST[test] = max(WORST.get(test, 0.0), ratio)


def graph_np(name):
    """(rowptr, colind, n_cols) int32 CSR of a case; "bounds" is boundary_csr(64)."""
    return boundary_csr(64) if name == "bounds" else case(name)


def structure(name, rp, ci, n_cols, dev):
    from cogdl_b200.structure import DEFAULT_CHUNK_EDGES

    return plan_structure(rp, ci, n_cols, dev, chunk=64 if name == "bounds" else DEFAULT_CHUNK_EDGES)


def place(a, kind, dev):
    """numpy a on the device: contiguous, a view of every other element of a wider last dimension, or misaligned."""
    t = T(a, dev)
    if kind == "view":
        v = torch.zeros(a.shape[:-1] + (2 * a.shape[-1],), dtype=t.dtype, device=dev)[..., ::2]
        v.copy_(t)
        return v
    return misaligned(t) if kind == "misaligned" else t


def incoming(out, kind, rng):
    """(G on the device, G as float64 numpy): random contiguous, the stride-0 ones of out.sum(), or a strided view."""
    if kind == "sum":
        return torch.ones((), dtype=out.dtype, device=out.device).expand(out.shape), np.ones(out.shape)
    g = rng.standard_normal(tuple(out.shape)).astype(np.float16 if out.dtype == torch.float16 else np.float32)
    return place(g, "view", out.device) if kind == "view" else T(g, out.device), g.astype(np.float64)


def same_bits(a, b, what):
    assert a.shape == b.shape and a.dtype == b.dtype, what
    ib = torch.int16 if a.dtype == torch.float16 else torch.int32
    assert torch.equal(a.contiguous().view(ib), b.contiguous().view(ib)), f"{what}: not bit-identical"


def mat(rows, cols, vals, shape):
    """fp64 sparse matrix of (rows, cols, vals); duplicates add up.  Magnitudes are built from |vals|, never abs() of a
    matrix, which would merge duplicate entries before taking the absolute value."""
    return sp.coo_matrix((np.asarray(vals, np.float64), (rows, cols)), shape=shape).tocsr()


def sum_ref(rows, cols, vals, X, shape):
    """(A @ X, |A| @ |X|) in fp64, A = (rows, cols, vals)."""
    X = np.asarray(X, np.float64)
    return mat(rows, cols, vals, shape) @ X, mat(rows, cols, np.abs(vals), shape) @ np.abs(X)


def bound(k, mag, m=0):
    """(k + 2 + m) 2^-24 sum|terms| (+ the smallest normal) for a sum of k terms and m fp32 products after it."""
    return (np.asarray(k, np.float64) + 2 + m) * U32 * mag + TINY


def sddmm_ref(rows, cols, A, B):
    """per edge e: (sum_f A[rows[e], f] B[cols[e], f], sum_f |...|), over the last axis."""
    t = np.asarray(A, np.float64)[rows] * np.asarray(B, np.float64)[cols]
    return t.sum(-1), np.abs(t).sum(-1)


def rows_of(rp):
    return np.repeat(np.arange(rp.shape[0] - 1), np.diff(rp))


def raw_backward(out, g):
    """The Function's own backward on g: its tuple as returned, so a gradient nobody asked for shows as None."""
    return out.grad_fn.apply(g)


def check_raw(out, g, expect, what):
    """expect[i]: None where input i must get no gradient, else the gradient autograd delivered (bit-identical)."""
    got = raw_backward(out, g)
    assert len(got) == len(expect), what
    for i, (a, b) in enumerate(zip(got, expect)):
        if b is None:
            assert a is None, f"{what}: input {i} was not asked for a gradient but got one"
        else:
            assert a is not None, f"{what}: input {i} got no gradient"
            same_bits(a.reshape(b.shape), b, f"{what}: input {i}")


# ================================================================================== 1. the Functions
SPMM_COMBOS = [  # (weights, inputs that require grad, actnn)
    ("none", "x", False), ("fixed", "x", False), ("grad", "w", False), ("grad", "xw", False),
    ("fixed", "x", True), ("grad", "w", True), ("grad", "xw", True)]


def spmm_graph(name, sym, rng):
    rp, ci, n_cols = graph_np(name)
    w = rng.standard_normal(ci.size).astype(np.float32)
    if sym:   # S = A + A^T: the CSR is its own transpose, values included
        S = sp.csr_matrix((w.astype(np.float64), ci.copy(), rp.copy()), shape=(rp.size - 1, n_cols))
        S = (S + S.T).tocsr()
        S.sort_indices()
        rp, ci, w = S.indptr.astype(np.int32), S.indices.astype(np.int32), S.data.astype(np.float32)
    return rp, ci, n_cols, w


@pytest.mark.parametrize("name,sym", [(g, s) for g in GRAPHS for s in (False, True) if not (s and g == "rect")])
@pytest.mark.parametrize("wkind,need,actnn", SPMM_COMBOS)
def test_spmm_function(dev, name, sym, wkind, need, actnn):
    from cogdl_b200.actnn.ops import dequantize_activation, quantize_activation
    from cogdl_b200.operators.spmm import SPMMFunction

    rng = np.random.default_rng(11)
    rp, ci, n_cols, w = spmm_graph(name, sym, rng)
    n, F = rp.size - 1, 36
    st = structure(name, rp, ci, n_cols, dev)
    X = rng.standard_normal((n_cols, F)).astype(np.float32)
    rows = rows_of(rp)
    vals = np.ones(ci.size, np.float32) if wkind == "none" else w
    ref, mag = sum_ref(rows, ci, vals, X, (n, n_cols))
    deg, cdeg = np.diff(rp)[:, None], np.bincount(ci, minlength=n_cols)[:, None]
    Xw = X
    if actnn and "w" in need:   # the SDDMM reads the features as the forward saved them: quantized, then dequantized
        torch.manual_seed(7)
        Xw = dequantize_activation(quantize_activation(T(X, dev), None), X.shape).cpu().numpy()
    first = None
    for gkind, xkind in MODES:
        x = place(X, xkind, dev).requires_grad_("x" in need)
        wt = None if wkind == "none" else T(w, dev).requires_grad_("w" in need)
        torch.manual_seed(7)
        out = SPMMFunction.apply(st, None, x, wt, sym, actnn)
        what = f"{name} sym={sym} {wkind}/{need} actnn={actnn} {gkind}/{xkind}"
        within(out.detach().cpu().numpy(), ref, bound(deg, mag), what + " out")
        G, g64 = incoming(out, gkind, rng)
        out.backward(G)
        if "x" in need:
            gx, gmag = sum_ref(ci, rows, vals, g64, (n_cols, n))
            within(x.grad.cpu().numpy(), gx, bound(cdeg, gmag), what + " grad x")
        else:
            assert x.grad is None
        if "w" in need:
            gw, wmag = sddmm_ref(rows, ci, g64, Xw)
            within(wt.grad.cpu().numpy(), gw, bound(F, wmag), what + " grad w")
        if first is None:
            first = (G.clone(), x.grad, None if wt is None else wt.grad)
    # the Function's own return values: None for rowptr, colind, sym, actnn and whatever was not asked for
    x = T(X, dev).requires_grad_("x" in need)
    wt = None if wkind == "none" else T(w, dev).requires_grad_("w" in need)
    torch.manual_seed(7)
    out = SPMMFunction.apply(st, None, x, wt, sym, actnn)
    check_raw(out, first[0], [None, None, first[1], first[2], None, None], f"{name} raw backward")


@pytest.mark.parametrize("name", GRAPHS)
@pytest.mark.parametrize("H", [1, 4])
@pytest.mark.parametrize("via", ["structure", "rowptr"])
def test_edge_softmax_function(dev, name, H, via):
    """Through a CSRStructure, and through the reference signature csr_edge_softmax(rowptr, h), whose structure has a
    zero stand-in for the column indices (edge softmax never reads them)."""
    from cogdl_b200.operators.edge_softmax import EdgeSoftmaxFunction, csr_edge_softmax

    rp, ci, n_cols = graph_np(name)
    rng = np.random.default_rng(20 + H)
    x = es_logits(rp, H, rng)
    st = structure(name, rp, ci, n_cols, dev)
    first = None
    for gkind, xkind in MODES:
        h = place(x, xkind, dev).requires_grad_(True)
        out = EdgeSoftmaxFunction.apply(st, h) if via == "structure" else csr_edge_softmax(T(rp, dev), h)
        what = f"{name} H={H} {via} {gkind}/{xkind}"
        y = out.detach().cpu().numpy()
        check_softmax(y, x, rp, what + " forward")
        G, g64 = incoming(out, gkind, rng)
        out.backward(G)
        ref, bnd, _, _ = softmax_bwd64(rp, y, g64, 1.0)
        within(h.grad.cpu().numpy(), ref, bnd, what + " backward")
        if first is None:
            first = (G.clone(), h.grad)
    h = T(x, dev).requires_grad_(True)
    out = EdgeSoftmaxFunction.apply(st, h) if via == "structure" else csr_edge_softmax(T(rp, dev), h)
    check_raw(out, first[0], [None, first[1], None], f"{name} raw backward")


def check_mhspmm(rp, ci, n_cols, att, feat, out, g64, g_feat, g_att, what):
    """out [n, H, F] = per head (rp, ci, att[:, h]) @ feat[:, h]; g_feat its transpose on g64; g_att the SDDMM."""
    n, H, F = rp.size - 1, feat.shape[1], feat.shape[2]
    rows = rows_of(rp)
    g64 = g64.reshape(n, H, F)
    deg, cdeg = np.diff(rp)[:, None], np.bincount(ci, minlength=n_cols)[:, None]
    for h in range(H):
        ref, mag = sum_ref(rows, ci, att[:, h], feat[:, h], (n, n_cols))
        within(out[:, h], ref, bound(deg, mag), f"{what} out head {h}")
        if g_feat is not None:
            ref, mag = sum_ref(ci, rows, att[:, h], g64[:, h], (n_cols, n))
            within(g_feat[:, h], ref, bound(cdeg, mag), f"{what} grad feat head {h}")
    if g_att is not None:
        ref, mag = sddmm_ref(rows, ci, g64, feat)
        within(g_att.reshape(ref.shape), ref, bound(F, mag), f"{what} grad attention")


NEEDS = {"feat": (True, False), "att": (False, True), "both": (True, True)}


@pytest.mark.parametrize("name", GRAPHS)
@pytest.mark.parametrize("H,F", [(4, 16), (3, 5)])
@pytest.mark.parametrize("need", list(NEEDS))
def test_mhspmm_function(dev, name, H, F, need):
    from cogdl_b200.operators.mhspmm import MHSPMMFunction

    rp, ci, n_cols = graph_np(name)
    n = rp.size - 1
    rng = np.random.default_rng(30 + H)
    att = rng.standard_normal((ci.size, H)).astype(np.float32)
    feat = rng.standard_normal((n_cols, H, F)).astype(np.float32)
    st = structure(name, rp, ci, n_cols, dev)
    nf, na = NEEDS[need]
    first = None
    for gkind, xkind in MODES:
        f = place(feat, xkind, dev).requires_grad_(nf)
        a = place(att, xkind, dev).requires_grad_(na)
        out = MHSPMMFunction.apply(st, None, f, a)
        G, g64 = incoming(out, gkind, rng)
        out.backward(G)
        check_mhspmm(rp, ci, n_cols, att, feat, out.detach().cpu().numpy(), g64,
                     f.grad.cpu().numpy() if nf else None, a.grad.cpu().numpy() if na else None,
                     f"{name} H={H} F={F} {need} {gkind}/{xkind}")
        assert (f.grad is None) != nf and (a.grad is None) != na
        if first is None:
            first = (G.clone(), f.grad, a.grad)
    out = MHSPMMFunction.apply(st, None, T(feat, dev).requires_grad_(nf), T(att, dev).requires_grad_(na))
    check_raw(out, first[0], [None, None, first[1], first[2]], f"{name} raw backward")


def scatter_max64(rp, ci, X):
    """(max, argmax) per row and column: the first edge in CSR order holding the maximum; empty rows 0 and -1."""
    n, F = rp.size - 1, X.shape[1]
    out, arg = np.zeros((n, F), np.float32), np.full((n, F), -1, np.int32)
    for r in np.nonzero(np.diff(rp))[0]:
        cols = ci[rp[r]:rp[r + 1]]
        j = np.argmax(X[cols], axis=0)          # first occurrence of the maximum
        out[r], arg[r] = X[cols][j, np.arange(F)], cols[j]
    return out, arg


@pytest.mark.parametrize("name", GRAPHS)
@pytest.mark.parametrize("F", [16, 7])
def test_scatter_max_function(dev, name, F):
    """argmax equal to the oracle's, ties (quantised values) and empty rows included; the gradient of a source element
    is the sum of g over the rows that picked it: bit-exact where one row did, within the bound where several did
    (atomics), exactly 0 where none did.  rect has more sources than rows."""
    from cogdl_b200.operators.scatter_max import ScatterMaxFunction, scatter_max_with_argmax

    rp, ci, n_cols = graph_np(name)
    n = rp.size - 1
    rng = np.random.default_rng(40 + F)
    X = (np.round(rng.standard_normal((n_cols, F)) * 4) / 4).astype(np.float32)
    ref, ref_id = scatter_max64(rp, ci, X)
    st = structure(name, rp, ci, n_cols, dev)
    _, arg = scatter_max_with_argmax(st, None, T(X, dev))
    assert np.array_equal(arg.cpu().numpy(), ref_id), f"{name}: argmax differs"
    ok = ref_id >= 0
    cols = np.broadcast_to(np.arange(F), ref_id.shape)[ok]

    def check_grad(gx, g64, what):
        want, mag, cnt = (np.zeros((n_cols, F)) for _ in range(3))
        np.add.at(want, (ref_id[ok], cols), g64[ok])
        np.add.at(mag, (ref_id[ok], cols), np.abs(g64[ok]))
        np.add.at(cnt, (ref_id[ok], cols), 1)
        got = gx.cpu().numpy()
        assert got.shape == (n_cols, F), what
        assert np.all(got[cnt == 0] == 0), f"{what}: a source no row picked has a gradient"
        assert np.array_equal(got[cnt == 1], want[cnt == 1]), f"{what}: a source one row picked is not that row's g"
        within(got, want, np.where(cnt > 1, bound(cnt, mag), 0), what + " gradient")

    for gkind, xkind in MODES:
        x = place(X, xkind, dev).requires_grad_(True)
        out = ScatterMaxFunction.apply(st, None, x)
        what = f"{name} F={F} {gkind}/{xkind}"
        assert np.array_equal(out.detach().cpu().numpy(), ref), f"{what}: max differs"
        G, g64 = incoming(out, gkind, rng)
        out.backward(G)
        check_grad(x.grad, g64, what)
    # the Function's own return values (the atomic sums may differ from the run above in their last bits)
    out = ScatterMaxFunction.apply(st, None, T(X, dev).requires_grad_(True))
    G, g64 = incoming(out, "rand", rng)
    got = raw_backward(out, G)
    assert len(got) == 3 and got[0] is None and got[1] is None
    check_grad(got[2], g64, f"{name} F={F} raw backward")


def check_gat(rp, ci, hl, hr, feat, att, out, g64, grads, what):
    """The fused GAT against fp64.  att: the fp32 attention the forward saved, held to the softmax bound of the fp32
    logits; out, d feat: the multi-head SpMM over att and over its transpose; d h_l, d h_r: the row and column sums of
    the per-edge softmax backward, whose input d att is an fp32 SDDMM carrying its own bound b (module docstring)."""
    n, H, F = feat.shape
    rows = rows_of(rp)
    z, logits = gat_logits32(rp, ci, hl, hr)
    check_softmax(att, logits, rp, what + " attention")
    check_mhspmm(rp, ci, n, att, feat, out.reshape(n, H, F), g64, grads[2], None, what)
    if grads[0] is None and grads[1] is None:
        return
    d_att, amag = sddmm_ref(rows, ci, g64.reshape(n, H, F), feat)
    b = bound(F, amag)
    dact = np.where(z > 0, 1.0, np.float64(SLOPE))
    y = att.astype(np.float64)
    d_edge, ebound, g_row, rbound = softmax_bwd64(rp, att, d_att, dact)
    yb = np.zeros((n, H))
    np.add.at(yb, rows, y * b)
    ebound = ebound + dact * y * (b + yb[rows])
    carried = np.zeros((n, H))
    np.add.at(carried, rows, dact * y * (b + yb[rows]))
    if grads[0] is not None:
        within(grads[0], g_row, rbound + carried, what + " grad h_l")
    if grads[1] is not None:
        g_col, cmag, cb = np.zeros((n, H)), np.zeros((n, H)), np.zeros((n, H))
        np.add.at(g_col, ci, d_edge)
        np.add.at(cmag, ci, np.abs(d_edge))
        np.add.at(cb, ci, ebound)
        cdeg = np.bincount(ci, minlength=n)[:, None]
        within(grads[1], g_col, cb + bound(cdeg, cmag), what + " grad h_r")


GAT_NEEDS = ["l", "r", "f", "lr", "lf", "rf", "lrf"]      # h_l, h_r, feat: every non-empty subset


def saved_attention(out):
    """The fp32 attention FusedGATFunction saved for its backward."""
    return out.grad_fn.saved_tensors[3].detach().cpu().numpy()


@pytest.mark.parametrize("name", SQUARE)
@pytest.mark.parametrize("H,F", [(4, 16), (1, 8)])
@pytest.mark.parametrize("need", GAT_NEEDS)
def test_fused_gat_function(dev, name, H, F, need):
    from cogdl_b200.operators.fused_gat import FusedGATFunction

    rp, ci, n = graph_np(name)
    rng = np.random.default_rng(50 + H)
    hl = rng.standard_normal((n, H)).astype(np.float32)
    hr = rng.standard_normal((n, H)).astype(np.float32)
    feat = rng.standard_normal((n, H, F)).astype(np.float32)
    st = structure(name, rp, ci, n, dev)
    first = None
    for gkind, xkind in MODES:
        ts = [place(a, xkind, dev).requires_grad_(c in need) for a, c in ((hl, "l"), (hr, "r"), (feat, "f"))]
        out = FusedGATFunction.apply(ts[0], ts[1], st, None, None, None, float(SLOPE), ts[2], 0.0, None)
        att = saved_attention(out)
        G, g64 = incoming(out, gkind, rng)
        out.backward(G)
        grads = [None if t.grad is None else t.grad.cpu().numpy() for t in ts]
        assert [g is not None for g in grads] == [c in need for c in "lrf"]
        check_gat(rp, ci, hl, hr, feat, att, out.detach().cpu().numpy(), g64, grads,
                  f"{name} H={H} F={F} {need} {gkind}/{xkind}")
        if first is None:
            first = (G.clone(), [t.grad for t in ts])
    ts = [T(a, dev).requires_grad_(c in need) for a, c in ((hl, "l"), (hr, "r"), (feat, "f"))]
    out = FusedGATFunction.apply(ts[0], ts[1], st, None, None, None, float(SLOPE), ts[2], 0.0, None)
    g = first[1]
    check_raw(out, first[0], [g[0], g[1], None, None, None, None, None, g[2], None, None], f"{name} raw backward")


# ================================================================================== 2. the graph-level entry points
BUILDS = ["rowptr", "coo", "shuffled"]
WEIGHTS = ["none", "fixed", "leaf"]
NORMS = ["none", "sym", "row"]


class GraphCase:
    """A Graph built one of three ways from a square case, with what its fp64 reference needs, in the user's edge order:
    row, col, w (the weights the SpMM multiplies by, after normalisation, fp32), in_norm / out_norm (fp32 or None),
    factors (the fp32 per-edge factors normalisation multiplied a trainable weight by), sym (the graph's flag), and the
    graph's CSR (rp, ci) once built: the stable sort of the user's edges by row."""

    def __init__(self, name, build, weights, norm, dev, seed=0):
        import cogdl_b200

        rp, ci, n = graph_np(name)
        E = ci.size
        row, col = rows_of(rp).astype(np.int64), ci.astype(np.int64)
        w = np.random.default_rng(seed + 5).uniform(0.25, 2.0, E).astype(np.float32)
        if build == "shuffled":
            p = np.random.default_rng(seed + 6).permutation(E)
            row, col, w = row[p], col[p], w[p]
        self.leaf = None if weights == "none" else T(w, dev).requires_grad_(weights == "leaf")
        if build == "rowptr":
            self.g = cogdl_b200.Graph(row_ptr=T(rp.astype(np.int64), dev), col=T(col, dev), edge_weight=self.leaf,
                                      num_nodes=n)
        else:
            self.g = cogdl_b200.Graph(edge_index=(T(row, dev), T(col, dev)), edge_weight=self.leaf, num_nodes=n)
        self.factors = []
        if norm != "none":
            getattr(self.g, f"{norm}_norm")()
            if build != "rowptr":      # a COO graph bakes the scaling into its weights: s[col] * w * s[row] or w * s[row]
                d = torch.zeros(n, device=dev).scatter_add_(0, T(row, dev), torch.ones(E, device=dev))
                s = d.pow(-0.5 if norm == "sym" else -1)
                s[torch.isinf(s)] = 0
                s = s.cpu().numpy()
                self.factors = [s[row], s[col]] if norm == "sym" else [s[row]]
        # read before anything builds the CSR: a COO graph's weights are still in the user's order here
        self.w = self.g.raw_edge_weight.detach().cpu().numpy().copy()
        self.in_norm = None if self.g.in_norm is None else self.g.in_norm.cpu().numpy().reshape(-1)
        self.out_norm = None if self.g.out_norm is None else self.g.out_norm.cpu().numpy().reshape(-1)
        self.sym = self.g.is_symmetric()
        self.n, self.row, self.col = n, row, col
        order = np.argsort(row, kind="stable")
        self.rp, self.ci = rp, col[order].astype(np.int32)

    def x_in(self, X):
        """The features the kernel reads: out_norm * X as fp32 forms it."""
        return X if self.out_norm is None else (self.out_norm[:, None] * X).astype(np.float32)

    def g_in(self, g, scale=None):
        """The incoming gradient the backward's SpMM reads: in_norm * g (and then * scale) as fp32 forms it."""
        g = np.asarray(g, np.float32)
        if self.in_norm is not None:
            g = (self.in_norm[:, None] * g).astype(np.float32)
        return g if scale is None else (np.float32(scale) * g).astype(np.float32)

    def spmm_ref(self, X):
        """(A @ x_in, |A| @ |x_in|, per-row term counts) for the user's triplets, with in_norm applied."""
        ref, mag = sum_ref(self.row, self.col, self.w, self.x_in(X), (self.n, self.n))
        if self.in_norm is not None:
            ref, mag = self.in_norm[:, None] * ref, self.in_norm[:, None] * mag
        return ref, mag, np.bincount(self.row, minlength=self.n)[:, None]

    def adjoint_ref(self, g):
        """The feature gradient of the SpMM on the fp32 gradient g it reads: over A itself when the graph is flagged
        symmetric (as the reference's backward takes it), else over A^T; then * out_norm.  (ref, mag, counts)."""
        src, dst = (self.row, self.col) if self.sym else (self.col, self.row)
        ref, mag = sum_ref(src, dst, self.w, g, (self.n, self.n))
        if self.out_norm is not None:
            ref, mag = self.out_norm[:, None] * ref, self.out_norm[:, None] * mag
        return ref, mag, np.bincount(src, minlength=self.n)[:, None]

    def leaf_ref(self, g, X):
        """The gradient of the trainable weight, in the user's order: SDDMM(g, x_in) times the normalisation factors."""
        ref, mag = sddmm_ref(self.row, self.col, g, self.x_in(X))
        for f in self.factors:
            ref, mag = ref * f, mag * f
        return ref, mag, len(self.factors)

    def m_out(self):
        return int(self.in_norm is not None)

    def m_adj(self):
        return int(self.out_norm is not None)


def two_calls(fn, inputs, gkind, rng):
    """fn() twice on the graph: the outputs must be bit-identical, and so must the gradients of inputs for one
    incoming gradient.  Returns (out, G as float64, gradients of the inputs that require grad)."""
    out1 = fn()
    out2 = fn()
    same_bits(out1, out2, "second call")
    G, g64 = incoming(out1, gkind, rng)
    req = [t for t in inputs if t is not None and t.requires_grad]
    g1 = torch.autograd.grad(out1, req, G, retain_graph=True)
    g2 = torch.autograd.grad(out2, req, G)
    for a, b in zip(g1, g2):
        same_bits(a, b, "gradient of the second call")
    return out1.detach(), g64, g1


def mode_of(weights):
    return MODES[WEIGHTS.index(weights)]


@pytest.mark.parametrize("name", SQUARE)
@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("weights", WEIGHTS)
@pytest.mark.parametrize("norm", NORMS)
def test_spmm_graph(dev, name, build, weights, norm):
    import cogdl_b200

    c = GraphCase(name, build, weights, norm, dev)
    rng = np.random.default_rng(60)
    X = rng.standard_normal((c.n, 24)).astype(np.float32)
    gkind, xkind = mode_of(weights)
    x = place(X, xkind, dev).requires_grad_(True)
    out, g64, grads = two_calls(lambda: cogdl_b200.spmm(c.g, x), [x, c.leaf], gkind, rng)
    what = f"{name} {build} {weights} {norm}"
    ref, mag, k = c.spmm_ref(X)
    within(out.cpu().numpy(), ref, bound(k, mag, c.m_out()), what + " out")
    gin = c.g_in(g64)
    ref, mag, k = c.adjoint_ref(gin)
    within(grads[0].cpu().numpy(), ref, bound(k, mag, c.m_adj()), what + " grad x")
    if weights == "leaf":
        ref, mag, m = c.leaf_ref(gin, X)
        within(grads[1].cpu().numpy(), ref, bound(24, mag, m), what + " grad weight")


@pytest.mark.parametrize("name", SQUARE)
@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("weights", WEIGHTS)
def test_spmm_graph_fp16(dev, name, build, weights):
    """fp16 features: the weights are rounded to fp16 for the kernel, and the reference is fp64 over the fp16 values."""
    import cogdl_b200

    c = GraphCase(name, build, weights, "none", dev)
    rng = np.random.default_rng(61)
    X = rng.standard_normal((c.n, 24)).astype(np.float16)
    gkind, xkind = mode_of(weights)
    x = place(X, xkind, dev).requires_grad_(True)
    out, g64, grads = two_calls(lambda: cogdl_b200.spmm(c.g, x), [x, c.leaf], gkind, rng)
    assert out.dtype == grads[0].dtype == torch.float16
    what = f"{name} {build} {weights} fp16"
    w16 = c.w.astype(np.float16)
    ref, mag = sum_ref(c.row, c.col, w16, X, (c.n, c.n))
    within(out.cpu().numpy(), ref, fp16_bound(ref, mag, np.bincount(c.row, minlength=c.n)[:, None]),
                  what + " out")
    src, dst = (c.row, c.col) if c.sym else (c.col, c.row)
    ref, mag = sum_ref(src, dst, w16, g64, (c.n, c.n))
    within(grads[0].cpu().numpy(), ref, fp16_bound(ref, mag, np.bincount(src, minlength=c.n)[:, None]),
                  what + " grad x")
    if weights == "leaf":
        ref, mag = sddmm_ref(c.row, c.col, g64, X)
        within(grads[1].cpu().numpy(), ref, fp16_bound(ref, mag, 24), what + " grad weight")


@pytest.mark.parametrize("name", SQUARE)
@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("weights", WEIGHTS)
@pytest.mark.parametrize("norm", NORMS)
def test_spmm_residual_graph(dev, name, build, weights, norm):
    """a * spmm(graph, x) + b * z: the k edge terms and b z form one sum of k + 1 terms, then the products by in_norm
    and a."""
    import cogdl_b200

    a, b = 0.9, 0.1
    a32, b32 = np.float64(np.float32(a)), np.float64(np.float32(b))
    c = GraphCase(name, build, weights, norm, dev)
    rng = np.random.default_rng(62)
    X = rng.standard_normal((c.n, 24)).astype(np.float32)
    Z = rng.standard_normal((c.n, 24)).astype(np.float32)
    gkind, xkind = mode_of(weights)
    x = place(X, xkind, dev).requires_grad_(True)
    z = place(Z, xkind, dev).requires_grad_(True)
    out, g64, grads = two_calls(lambda: cogdl_b200.spmm_residual(c.g, x, z, a, b), [x, z, c.leaf], gkind, rng)
    what = f"{name} {build} {weights} {norm}"
    ref, mag, k = c.spmm_ref(X)
    bz = b32 * Z.astype(np.float64)
    within(out.cpu().numpy(), a32 * ref + bz, bound(k + 1, a32 * mag + np.abs(bz), c.m_out() + 1),
                  what + " out")
    gin = c.g_in(g64)
    ref, mag, k = c.adjoint_ref(gin)
    within(grads[0].cpu().numpy(), a32 * ref, bound(k, a32 * mag, c.m_adj() + 1), what + " grad x")
    within(grads[1].cpu().numpy(), b32 * g64, bound(1, np.abs(b32 * g64)), what + " grad z")
    if weights == "leaf":
        ref, mag, m = c.leaf_ref(c.g_in(g64, a), X)
        within(grads[2].cpu().numpy(), ref, bound(24, mag, m), what + " grad weight")


@pytest.mark.parametrize("name", SQUARE)
@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("dim", [1, 2])
def test_edge_softmax_graph(dev, name, build, dim):
    """As in the reference, the values are taken in the graph's CSR order once it is built (the call builds it): on a
    shuffled COO graph, position p is the p-th edge of the stable row sort of the user's edges."""
    import cogdl_b200

    c = GraphCase(name, build, "none", "none", dev)
    rng = np.random.default_rng(63)
    x = es_logits(c.rp, 3, rng)[:, :1] if dim == 1 else es_logits(c.rp, 3, rng)
    x = np.ascontiguousarray(x)
    h = T(x.reshape(-1) if dim == 1 else x, dev).requires_grad_(True)
    out, g64, grads = two_calls(lambda: cogdl_b200.edge_softmax(c.g, h), [h], "rand", rng)
    assert out.dim() == dim
    what = f"{name} {build} dim={dim}"
    y = out.cpu().numpy().reshape(x.shape)
    check_softmax(y, x, c.rp, what + " forward")
    ref, bnd, _, _ = softmax_bwd64(c.rp, y, g64.reshape(x.shape), 1.0)
    within(grads[0].cpu().numpy().reshape(x.shape), ref, bnd, what + " backward")


@pytest.mark.parametrize("name", SQUARE)
@pytest.mark.parametrize("build", BUILDS)
@pytest.mark.parametrize("H", [1, 4])
def test_mh_spmm_graph(dev, name, build, H):
    """H > 1: the multi-head SpMM; H = 1: an SpMM with the attention as the edge weight inside local_graph() (flagged
    asymmetric, so its backward takes the transpose).  Either way the attention is taken in the graph's CSR order."""
    import cogdl_b200

    c = GraphCase(name, build, "none", "none", dev)
    rng = np.random.default_rng(64)
    F = 12
    att = rng.standard_normal((c.ci.size, H)).astype(np.float32)
    feat = rng.standard_normal((c.n, H, F)).astype(np.float32)
    a = T(att, dev).requires_grad_(True)
    f = T(feat, dev).requires_grad_(True)
    out, g64, grads = two_calls(lambda: cogdl_b200.mh_spmm(c.g, a, f), [a, f], "rand", rng)
    assert out.shape == (c.n, H * F)
    check_mhspmm(c.rp, c.ci, c.n, att, feat, out.cpu().numpy().reshape(c.n, H, F), g64,
                 grads[1].cpu().numpy(), grads[0].cpu().numpy(), f"{name} {build} H={H}")
    assert c.g.is_symmetric() == c.sym, "local_graph() leaked the symmetric flag"


@pytest.mark.parametrize("name", SQUARE)
@pytest.mark.parametrize("build", BUILDS)
def test_fused_gat_op_graph(dev, name, build):
    import cogdl_b200

    c = GraphCase(name, build, "none", "none", dev)
    rng = np.random.default_rng(65)
    H, F = 4, 8
    hl = rng.standard_normal((c.n, H)).astype(np.float32)
    hr = rng.standard_normal((c.n, H)).astype(np.float32)
    feat = rng.standard_normal((c.n, H, F)).astype(np.float32)
    ts = [T(v, dev).requires_grad_(True) for v in (hl, hr, feat)]
    att = []

    def call():
        o = cogdl_b200.fused_gat_op(ts[0], ts[1], c.g, float(SLOPE), ts[2])
        att.append(saved_attention(o))
        return o

    out, g64, grads = two_calls(call, ts, "rand", rng)
    assert np.array_equal(att[0], att[1])
    check_gat(c.rp, c.ci, hl, hr, feat, att[0], out.cpu().numpy(), g64, [g.cpu().numpy() for g in grads],
              f"{name} {build}")


# ================================================================================== 3. layers on a shuffled COO graph
LAYERS = ["gcn", "gcn-fused", "sage-mean", "sage-mean-fused", "sage-sum", "sage-sum-fused", "sage-max",
          "sage-max-fused", "gat", "gat-fused", "gat1", "gat1-fused", "fused_sage-mean", "fused_sage-sum",
          "fused_sage-max"]


def layer_graphs(name, dev):
    """(shuffled COO graph, its twin: the stable row sort of the same edges and weights, as COO, so normalisation bakes
    the same fp32 weights into both, edge by edge), the twin's CSR as numpy."""
    import cogdl_b200

    rp, ci, n = graph_np(name)
    E = ci.size
    row, col = rows_of(rp).astype(np.int64), ci.astype(np.int64)
    w = np.random.default_rng(7).uniform(0.25, 2.0, E).astype(np.float32)
    p = np.random.default_rng(8).permutation(E)
    row, col, w = row[p], col[p], w[p]
    o = np.argsort(row, kind="stable")
    graphs = [cogdl_b200.Graph(edge_index=(T(r, dev), T(c_, dev)), edge_weight=T(w_, dev), num_nodes=n)
              for r, c_, w_ in ((row, col, w), (row[o], col[o], w[o]))]
    return graphs, n


class DirectSAGE(torch.nn.Module):
    """fused_sage_layer called directly, with SAGELayer's parameters."""

    def __init__(self, aggr):
        super().__init__()
        self.aggr = aggr
        self.fc = torch.nn.Linear(256, 64)

    def forward(self, graph, x):
        from cogdl_b200.operators.fused_sage import fused_sage_layer

        return fused_sage_layer(graph, x, self.fc.weight, self.fc.bias, self.aggr, relu=self.aggr != "max")


def make_layer(kind):
    from cogdl_b200.layers import GATLayer, GCNLayer, SAGELayer

    torch.manual_seed(3)
    fused = kind.endswith("-fused")
    base = kind.replace("-fused", "")
    if base == "gcn":
        return GCNLayer(128, 64, activation="relu", fused=fused)
    if base.startswith("sage-"):
        aggr = base.split("-")[1]
        return SAGELayer(128, 64, aggr=aggr, activation=None if aggr == "max" else "relu", fused=fused)
    if base.startswith("gat"):
        return GATLayer(128, 16, nhead=1 if base == "gat1" else 4, attn_drop=0.0, fused=fused)
    return DirectSAGE(base.split("-")[1])


@pytest.mark.parametrize("name", ["two_hubs", "bounds"])
@pytest.mark.parametrize("kind", LAYERS)
def test_layer_on_shuffled_coo_graph(dev, name, kind):
    """Outputs and every parameter and input gradient bit-identical between the shuffled COO graph and its twin: the
    same edges in each row in the same order, so every fp32 sum sees the same terms in the same order.  The input
    gradient of max aggregation passes through the scatter_max backward's atomics: there the two runs may differ by
    twice the section-1 bound of the atomic sum, plus one rounding each of the self term's addition."""
    graphs, n = layer_graphs(name, dev)
    if kind.startswith("gcn"):
        for g in graphs:
            g.sym_norm()
    layers = [make_layer(kind).to(dev)]
    layers.append(copy.deepcopy(layers[0]))
    X = torch.randn(n, 128, generator=torch.Generator().manual_seed(9)).to(dev)
    G = None
    res = []
    for g, layer in zip(graphs, layers):
        x = X.clone().requires_grad_(True)
        out = layer(g, x)
        G = torch.randn(out.shape, generator=torch.Generator().manual_seed(10)).to(dev) if G is None else G
        out.backward(G)
        res.append((out.detach(), x.grad, [p.grad for p in layer.parameters()]))
    (o1, gx1, p1), (o2, gx2, p2) = res
    same_bits(o1, o2, f"{kind} output")
    for i, (a, b) in enumerate(zip(p1, p2)):
        same_bits(a, b, f"{kind} parameter {i} gradient")
    if not kind.endswith("max") and "max-" not in kind:
        same_bits(gx1, gx2, f"{kind} input gradient")
        return
    from cogdl_b200.operators.scatter_max import scatter_max_with_argmax

    _, arg = scatter_max_with_argmax(graphs[1].structure(), None, X)
    d = (G @ layers[0].fc.weight[:, 128:]).detach().double().cpu().numpy()     # the gradient reaching the aggregation
    arg = arg.cpu().numpy()
    ok = arg >= 0
    cols = np.broadcast_to(np.arange(128), arg.shape)[ok]
    mag, cnt = np.zeros((n, 128)), np.zeros((n, 128))
    np.add.at(mag, (arg[ok], cols), np.abs(d[ok]))
    np.add.at(cnt, (arg[ok], cols), 1)
    a, b = gx1.cpu().numpy(), gx2.cpu().numpy()
    assert np.array_equal(a[cnt <= 1], b[cnt <= 1]), f"{kind}: input gradient differs where no atomics add up"
    within(a, b.astype(np.float64), np.where(cnt > 1, 2 * bound(cnt, mag) + 2 * U32 * np.abs(b), 0),
                  f"{kind} input gradient")

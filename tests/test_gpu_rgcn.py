"""R-GCN fan-out aggregation and edge dot (cogdl_b200/csrc/rgcn.cu), rgcn_aggregate / rgcn_conv and the reference
RGCN through install(rgcn=True).

- Each row of tests/rgcn_table.py records exactly the kernel it names.  The aggregation (and its per-basis form) is
  bit-identical, for every basis b, to this package's SpMM with per-slot values fl(w * coef[type, b]) on the same
  structure, and within 1e-5 of fp64 measured against the sum of |terms|; the edge dot is within the suite's
  (k + 2 + m) 2^-24 sum|terms| bound of fp64.  Two runs give the same bits.
- rgcn_conv and rgcn_aggregate: the output and d x, d coef, d weight against fp64 autograd of the relational sum, on a
  cogdl_b200.Graph built from a shuffled COO whose edge types stay paired with their edges; reproducible bits; types
  out of range raise before any launch; no host synchronisation after the first call on a graph.
- The reference RGCN / LinkPredictRGCN through install(rgcn=True), in a child process (tests/rgcn_refpkg_check.py).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.gpu_util import bits, dev, misaligned, rel
from tests.graphs import boundary_csr, case
from tests.rgcn_table import TABLE
from tests.test_gpu_autograd import bound, rows_of

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TOL = 1e-5


def row_inputs(c, dev):
    from cogdl_b200.structure import CSRStructure

    rp, ci, n_cols = boundary_csr(64) if c.graph == "bounds" else case(c.graph)
    st = CSRStructure(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), n_cols=n_cols,
                      chunk_edges=64)
    rng = np.random.default_rng(900 + c.F + 31 * c.B + c.T)
    f32 = lambda *s: rng.standard_normal(s).astype(np.float32)  # noqa: E731
    nnz = ci.shape[0]
    etype = rng.integers(0, c.T, nnz).astype(np.int32)
    w = (rng.random(nnz) + 0.1).astype(np.float32)
    coef = f32(c.T, c.B)
    return rp, ci, n_cols, st, etype, w, coef, rng


def dev_t(a, dev, aligned=True):
    t = torch.from_numpy(np.ascontiguousarray(a)).to(dev)
    return t if aligned else misaligned(t)


@pytest.mark.parametrize("c", TABLE, ids=lambda c: c.id)
def test_row_bit_identical_to_per_basis_spmm_and_near_fp64(dev, c):
    import cogdl_b200
    from cogdl_b200.operators._raw import rgcn_aggr_raw, rgcn_edge_dot_raw, spmm_raw

    rp, ci, n_cols, st, etype, w, coef, rng = row_inputs(c, dev)
    n, nnz = rp.shape[0] - 1, ci.shape[0]
    rows = rows_of(rp)
    et, wt, ct = dev_t(etype, dev), dev_t(w, dev), dev_t(coef, dev)
    if c.op == "dot":
        G = rng.standard_normal((n, c.B, c.F)).astype(np.float32)
        X = rng.standard_normal((n_cols, c.F)).astype(np.float32)
        Gt, Xt = dev_t(G, dev, c.aligned), dev_t(X, dev, c.aligned)
        p = rgcn_edge_dot_raw(st, wt, Gt, Xt)
        assert cogdl_b200._cabi.last_kernel().startswith(c.kernel + " ") or nnz == 0, cogdl_b200._cabi.last_kernel()
        assert torch.equal(bits(p), bits(rgcn_edge_dot_raw(st, wt, Gt, Xt))), "two runs differ"
        terms = G.astype(np.float64)[rows] * X.astype(np.float64)[ci][:, None, :]
        ref = w[:, None].astype(np.float64) * terms.sum(-1)
        mag = w[:, None].astype(np.float64) * np.abs(terms).sum(-1)
        got = p.double().cpu().numpy()
        bad = np.argwhere(~(np.abs(got - ref) <= bound(c.F + 5, mag, 1)))
        assert bad.size == 0, f"{c.id}: {len(bad)} dot products off fp64, first at {tuple(bad[0])}"
        return
    per_basis = c.op == "per_basis"
    X = rng.standard_normal((n_cols, c.B, c.F) if per_basis else (n_cols, c.F)).astype(np.float32)
    Xt = dev_t(X, dev, c.aligned)
    y = rgcn_aggr_raw(st, et, wt, ct, Xt, per_basis=per_basis)
    assert y.shape == (n, c.B, c.F)
    if nnz:
        assert cogdl_b200._cabi.last_kernel().startswith(c.kernel + " "), cogdl_b200._cabi.last_kernel()
    assert torch.equal(bits(y), bits(rgcn_aggr_raw(st, et, wt, ct, Xt, per_basis=per_basis))), "two runs differ"
    deg = np.diff(rp)
    X64 = X.astype(np.float64)
    for b in range(c.B):
        v = wt * ct[et.long(), b]                     # fl(w * coef[type, b]), as the kernel forms it
        xb = Xt[:, b].contiguous() if per_basis else Xt
        want = spmm_raw(st, v, xb)
        mism = (bits(y[:, b]) != bits(want)).nonzero()
        assert mism.numel() == 0, f"{c.id}: basis {b}: {mism.shape[0]} elements differ from the SpMM, first at " \
                                  f"{tuple(mism[0].tolist())}"
        vals = w.astype(np.float64) * coef.astype(np.float64)[etype, b]
        xs = (X64[:, b] if per_basis else X64)[ci]
        ref = np.zeros((n, c.F))
        mag = np.zeros((n, c.F))
        np.add.at(ref, rows, vals[:, None] * xs)
        np.add.at(mag, rows, np.abs(vals[:, None] * xs))
        got = y[:, b].double().cpu().numpy()
        scale = np.maximum(np.abs(ref), mag)
        bad = np.argwhere(~(np.abs(got - ref) <= TOL * scale + 1e-30))
        assert bad.size == 0, f"{c.id}: basis {b}: {len(bad)} elements off fp64 (max degree {deg.max()})"


# ------------------------------------------------------------------ graph-level entry points

N, E, T, B, F_IN, F_OUT = 300, 2400, 5, 3, 24, 16


def kg(dev, seed=3, weighted=True):
    """A shuffled COO with edge types (type 0 absent, a hub row) as host arrays, and a cogdl_b200.Graph built from it
    on the device."""
    import cogdl_b200

    g = torch.Generator().manual_seed(seed)
    row = torch.cat([torch.randint(0, N, (E,), generator=g), torch.zeros(200, dtype=torch.int64)])
    col = torch.randint(0, N, (row.numel(),), generator=g)
    typ = torch.randint(1, T, (row.numel(),), generator=g)
    w = torch.rand(row.numel(), generator=g) + 0.5 if weighted else None
    perm = torch.randperm(row.numel(), generator=g)
    row, col, typ = row[perm], col[perm], typ[perm]
    w = None if w is None else w[perm]
    graph = cogdl_b200.Graph(edge_index=(row.to(dev), col.to(dev)), edge_weight=None if w is None else w.to(dev),
                             edge_attr=typ.to(dev), num_nodes=N)
    return row, col, typ, w, graph


def params(dev, seed=4):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(N, F_IN, generator=g)
    alpha = torch.randn(T, B, generator=g)
    V = torch.randn(B, F_IN, F_OUT, generator=g) / 5
    dout = torch.randn(N, F_OUT, generator=g)
    return x, alpha, V, dout


def test_rgcn_conv_and_aggregate_against_fp64_autograd(dev):
    import cogdl_b200
    from tests.rgcn_ref import relational_sum, row_norm_weights, type_weights

    row, col, typ, w, graph = kg(dev)
    graph.row_norm()
    x, alpha, V, dout = params(dev)
    xd, ad, Vd = (t.to(dev).requires_grad_(True) for t in (x, alpha, V))
    out = cogdl_b200.rgcn_conv(graph, xd, ad, Vd)
    gx, ga, gV = torch.autograd.grad(out, [xd, ad, Vd], dout.to(dev))

    w_hat = row_norm_weights(row, N, w)
    x64, a64, V64 = (t.double().requires_grad_(True) for t in (x, alpha, V))
    ref = relational_sum(row, col, typ, w_hat, x64, type_weights(a64, V64, T))
    rx, ra, rV = torch.autograd.grad(ref, [x64, a64, V64], dout.double())
    for name, got, want in (("out", out, ref), ("dx", gx, rx), ("dalpha", ga, ra), ("dV", gV, rV)):
        assert rel(got, want) <= TOL, (name, rel(got, want))

    # the aggregation alone: agg[i, b] = sum_t alpha[t, b] (A_t x)[i], with its own backward
    agg = cogdl_b200.rgcn_aggregate(graph, xd, ad)
    g_agg = torch.randn(agg.shape, generator=torch.Generator().manual_seed(9)).to(dev)
    hx, ha = torch.autograd.grad(agg, [xd, ad], g_agg)
    x64b, a64b = x.double().requires_grad_(True), alpha.double().requires_grad_(True)
    ragg = torch.stack([relational_sum(row, col, typ, w_hat * a64b[typ, b], x64b,
                                       torch.eye(F_IN, dtype=torch.float64).expand(T, F_IN, F_IN)) for b in range(B)], 1)
    rhx, rha = torch.autograd.grad(ragg, [x64b, a64b], g_agg.double().cpu())
    for name, got, want in (("agg", agg, ragg), ("agg dx", hx, rhx), ("agg dalpha", ha, rha)):
        assert rel(got, want) <= TOL, (name, rel(got, want))


def test_rgcn_conv_is_reproducible_and_types_stay_with_their_edges(dev):
    import cogdl_b200

    x, alpha, V, dout = params(dev)

    def run(graph):
        xd, ad, Vd = (t.to(dev).requires_grad_(True) for t in (x, alpha, V))
        out = cogdl_b200.rgcn_conv(graph, xd, ad, Vd)
        return [out.detach()] + list(torch.autograd.grad(out, [xd, ad, Vd], dout.to(dev)))

    row, col, typ, w, g1 = kg(dev)
    a = run(g1)
    b = run(g1)
    assert all(torch.equal(bits(u), bits(v)) for u, v in zip(a, b))
    # the same edges in CSR order: the graph's stable sort gives the same slots, so the same bits
    order = torch.sort(row, stable=True).indices
    g2 = cogdl_b200.Graph(edge_index=(row[order].to(dev), col[order].to(dev)), edge_weight=w[order].to(dev),
                          edge_attr=typ[order].to(dev), num_nodes=N)
    c = run(g2)
    assert all(torch.equal(bits(u), bits(v)) for u, v in zip(a, c))


def test_bad_types_and_operands_raise_before_any_launch(dev):
    import cogdl_b200

    x, alpha, V, _ = params(dev)
    xd, ad, Vd = x.to(dev), alpha.to(dev), V.to(dev)
    row, col, typ, w, graph = kg(dev)
    graph.edge_attr = graph.edge_attr.clone()
    with pytest.raises(ValueError, match="out of range"):
        cogdl_b200.rgcn_conv(graph, xd, ad[:3], Vd)          # types up to 4, 3 relations
    row2, col2, typ2, w2, g_neg = kg(dev, seed=5)
    g_neg.edge_attr = torch.where(torch.arange(typ2.numel(), device=dev) == 7, -1, g_neg.edge_attr)
    with pytest.raises(ValueError, match="negative"):
        cogdl_b200.rgcn_aggregate(g_neg, xd, ad)
    with pytest.raises(RuntimeError):
        cogdl_b200.rgcn_aggregate(graph, x, ad)
    with pytest.raises(TypeError):
        cogdl_b200.rgcn_aggregate(graph, xd.double(), ad)
    _, _, _, _, g3 = kg(dev, seed=6)
    g3.edge_weight = g3.raw_edge_weight.clone().requires_grad_(True)
    with pytest.raises(ValueError, match="require grad"):
        cogdl_b200.rgcn_aggregate(g3, xd, ad)
    g3.grb_adj = torch.eye(N, device=dev)
    with pytest.raises(ValueError):
        cogdl_b200.rgcn_aggregate(g3, xd, ad)


def test_no_launch_for_an_out_of_range_type(dev):
    """The host-side size check runs before the aggregation: nothing is launched for a table that is too small."""
    import cogdl_b200

    x, alpha, V, _ = params(dev)
    _, _, _, _, graph = kg(dev)
    cogdl_b200.rgcn_conv(graph, x.to(dev), alpha.to(dev), V.to(dev))     # builds and caches the structure
    torch.cuda.synchronize()
    before = cogdl_b200._cabi.launch_count()
    with pytest.raises(ValueError, match="out of range"):
        cogdl_b200.rgcn_conv(graph, x.to(dev), alpha[:2].to(dev), V.to(dev))
    assert cogdl_b200._cabi.launch_count() == before


def test_empty_graph_gives_zeros(dev):
    import cogdl_b200

    graph = cogdl_b200.Graph(edge_index=(torch.zeros(0, dtype=torch.int64, device=dev),) * 2,
                             edge_attr=torch.zeros(0, dtype=torch.int64, device=dev), num_nodes=4)
    x = torch.randn(4, 8, device=dev)
    agg = cogdl_b200.rgcn_aggregate(graph, x, torch.randn(3, 2, device=dev))
    assert agg.shape == (4, 2, 8) and not agg.any()


def test_no_host_sync_after_the_first_call(dev):
    import cogdl_b200

    x, alpha, V, dout = params(dev)
    _, _, _, _, graph = kg(dev)
    graph.row_norm()
    xd, ad, Vd = (t.to(dev).requires_grad_(True) for t in (x, alpha, V))
    g = dout.to(dev)
    out = cogdl_b200.rgcn_conv(graph, xd, ad, Vd)
    torch.autograd.grad(out, [xd, ad, Vd], g)                       # builds the transpose and the type index
    agg = cogdl_b200.rgcn_aggregate(graph, xd, ad)
    torch.autograd.grad(agg, [xd, ad], torch.ones_like(agg))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        out = cogdl_b200.rgcn_conv(graph, xd, ad, Vd)
        torch.autograd.grad(out, [xd, ad, Vd], g)
        agg = cogdl_b200.rgcn_aggregate(graph, xd, ad)
        torch.autograd.grad(agg, [xd, ad], torch.ones_like(agg))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_reference_rgcn_through_install():
    """RGCN / LinkPredictRGCN through install(rgcn=True): at T = 1 within 1e-5 of the reference's own CPU run (output
    and parameter gradients), at T > 1 within 1e-5 of the fp64 relational sum, on shuffled-COO cogdl.data.Graphs;
    fallbacks run the original and uninstall_rgcn() restores it."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.rgcn_refpkg_check"], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["untouched_without_flag"] and res["rebound"] and res["restored"], res
    assert res["patched"] == ["cogdl.layers.rgcn_layer.RGCNLayer.forward"], res
    assert max(res["t1_vs_ref_cpu"].values()) <= 1e-5, res
    assert max(res["tn_vs_fp64"].values()) <= 1e-5, res
    assert res["grads_present"], res
    assert res["loss_finite"] and res["structures_built_per_step"] == 1, res
    assert res["fallbacks"] == ["cpu", "bdd"], res

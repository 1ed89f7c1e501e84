"""Simple-HGN attention (cogdl_b200/csrc/simple_hgn.cu), cogdl_b200.hgn_attention and install_simple_hgn.

- Every row of tests/hgn_table.py records the kernels it names, and every element of every output lies within a
  per-element bound (u = 2^-24; the helpers are those of tests/test_gpu_dispatch.py, whose docstring derives them):
  * the logits are reproduced bit for bit in numpy, fl(fl(h_l[row] + h_r[col]) + h_e[type]) and then the fp32 product
    with the slope where negative, and the attention |att| is checked against their fp64 softmax (check_softmax);
    the sign bits of att are the dropout mask of gat_dropout_ref.keep_mask exactly;
  * mix = fl(fl(fl(a keep_scale) (1 - alpha)) + fl(res alpha)) (fl(a keep_scale) taken as 0 where dropped) is all
    separately rounded products and sums, so it equals a numpy emulation over the kernel's own |att| bit for bit;
    the inference call (no attention output) gives the same mix bit for bit;
  * out: the multi-head SpMM bound over the kernel's mix, deg u sum |mix h|;
  * d m = mhsddmm(d out, h): F u sum |g h|; d res = fl(d m alpha) bit for bit;
  * d edge and d h_l (g_row): softmax_bwd64 on |att| with g = fl(d m fl(grad_scale)) (0 where dropped) and the
    LeakyReLU derivative at the exact pre-activation (the slope at exactly 0: the first edge of every row);
  * d h: the transposed multi-head SpMM bound, coldeg u sum |mix d out|;
  * d h_r: the column sums of the kernel's d edge, coldeg u sum |d edge| (cogdl_b200_edge_colsum_f32, hub columns
    under the transpose's plan on the bounds_t rows);
  * d h_e: the per-type sums of the kernel's d edge, (deg_t + 2) u sum |d edge|, exactly 0 for types no edge carries.
  Inputs: h_r ~ U(-20, 90), h_e holding one type near -60 and one near +30 (the largest row's first chunk entirely of
  the dominated type, so whole chunks underflow beside the row maximum), the first edge of every row at a
  pre-activation of exactly +0, and T above the largest type used.  With alpha = 1, d h_l, d h_r and d h_e are exactly
  0.  The worst error / bound ratio of every check is printed.
- The same seed gives the same bits, d h_e included.
- The rebound layer (on a stand-in with myGATConv's parameters) reproduces tests/golden/simple_hgn.npz from a shuffled
  COO, its types reordered with the edges; types, tables, devices and dtypes that have no kernel raise before any
  launch; uninstall_simple_hgn restores the original forward.
- With the example staged in oracle/_ref/examples, its unmodified myGATConv under the hook against its original forward,
  in a child process (tests/simple_hgn_refpkg_check.py).
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import test_gpu_dispatch
from tests.gat_dropout_ref import keep_mask
from tests.gpu_util import dev
from tests.graphs import boundary_csc, boundary_csr, case
from tests.hgn_table import ALPHA, CHUNK, MAX_TABLE, TABLE
from tests.simple_hgn_ref import HgnConvStandIn, aggregate_fp64, hgn_attention_fp64
from tests.test_gpu_dispatch import assert_within, check_softmax, softmax_bwd64
from tests.test_gpu_dispatch_message import col_sum, edge_rows, seg_reduce

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "simple_hgn.npz")
SLOPE, F = 0.2, 4
U32 = 2.0 ** -24
TINY = float(np.finfo(np.float32).tiny)


def close(a, b, what):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    if b.numel() == 0:
        return
    scale = float(b.abs().max())
    err = (a - b).abs() / torch.clamp(b.abs(), min=scale).clamp_min(1e-30)
    assert float(err.max()) <= 1e-5, f"{what}: {float(err.max()):.2e}"


def _graph(c):
    if c.graph == "bounds":
        return boundary_csr(CHUNK)
    if c.graph == "bounds_t":
        return boundary_csc(CHUNK)
    return case(c.graph)


def row_inputs(c, dev, seed=0):
    """The row's graph and inputs (module docstring).  h_l, h_r and h_e lie on a 2^-10 grid, so h_l of a row's first
    edge can cancel h_r + h_e exactly."""
    from cogdl_b200.structure import CSRStructure, RgcnStructure

    rp, ci, n_cols = _graph(c)
    st = CSRStructure(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), n_cols=n_cols,
                      chunk_edges=CHUNK if c.plan else 0)
    rng = np.random.default_rng(1000 + c.H + 7 * c.T + seed)
    n, nnz, deg = rp.shape[0] - 1, ci.shape[0], np.diff(rp)
    grid = lambda a: (np.round(np.asarray(a) * 1024) / 1024).astype(np.float32)  # noqa: E731
    used = max(c.T - 1, 1)                                  # type T - 1 carries no edge (T > 1)
    etype = rng.integers(0, used, nnz).astype(np.int32)
    he = grid(rng.standard_normal((c.T, c.H)))
    he[0] = grid(-60 + rng.standard_normal(c.H))
    if used > 1:
        he[1] = grid(30 + rng.standard_normal(c.H))
    big = int(np.argmax(deg)) if n else 0
    if n and deg[big] > CHUNK:                              # the largest row's first chunk: the dominated type only
        etype[rp[big]:rp[big] + CHUNK] = 0
        if used > 1:
            etype[rp[big] + CHUNK] = 1
    hr = grid(rng.uniform(-20, 90, (n_cols, c.H)))
    hl = grid(rng.standard_normal((n, c.H)))
    first = rp[:-1][deg > 0]
    hl[deg > 0] = -(hr[ci[first]] + he[etype[first]])       # exact on the grid: pre-activation +0
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    ins = {"h": t(rng.standard_normal((n_cols, c.H, F)).astype(np.float32)), "h_l": t(hl), "h_r": t(hr), "h_e": t(he),
           "res": t(rng.random((nnz, c.H)).astype(np.float32)) if c.res else None}
    g = t(rng.standard_normal((n, c.H, F)).astype(np.float32))
    return rp, ci, st, RgcnStructure(st, torch.from_numpy(etype).to(dev)), etype, ins, g


def run(rs, ins, c, seed):
    from cogdl_b200.operators._raw import attn_dropout_args
    from cogdl_b200.operators.simple_hgn import HgnAttentionFunction

    leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items() if v is not None}
    drop = None
    if c.p:
        drop_below, scale = attn_dropout_args(c.p)
        drop = (seed, drop_below, scale)
    out, att = HgnAttentionFunction.apply(rs, leaves["h"], leaves["h_l"], leaves["h_r"], leaves["h_e"],
                                          leaves.get("res"), SLOPE, drop, c.alpha)
    return out, att, leaves


def np_bits(a):
    return np.ascontiguousarray(a, np.float32).view(np.uint32)


@pytest.mark.parametrize("c", TABLE, ids=lambda c: c.id)
def test_row_against_fp64(dev, c):
    import cogdl_b200

    from cogdl_b200.operators._raw import attn_dropout_args, hgn_attn_bwd_raw, hgn_attn_raw, mhsddmm_raw

    test_gpu_dispatch.RATIOS.clear()
    rp, ci, st, rs, etype, ins, g = row_inputs(c, dev)
    seed = 12345 + c.H
    # the kernels the row names: the attention stage and its backward, each recorded by its own call
    drop = (seed, *attn_dropout_args(c.p)) if c.p else None
    mix, att = hgn_attn_raw(st, rs.type, ins["h_l"], ins["h_r"], ins["h_e"], SLOPE, True, drop, ins["res"], c.alpha)
    note2 = cogdl_b200._cabi.last_kernel()
    mix_inf, att_inf = hgn_attn_raw(st, rs.type, ins["h_l"], ins["h_r"], ins["h_e"], SLOPE, False, drop, ins["res"],
                                    c.alpha)
    assert att_inf is None and note2 == cogdl_b200._cabi.last_kernel()
    hgn_attn_bwd_raw(st, rs.type, att, torch.ones_like(att), ins["h_l"], ins["h_r"], ins["h_e"], SLOPE, 1.0)
    for mode, note in ((2, note2), (3, cogdl_b200._cabi.last_kernel())):
        if ci.shape[0] > 0:
            parts = [p.replace(" cp.async.bulk tiles", "") for p in note.split(" + ")]
            want = [c.kernel(mode)] + ([c.stats(mode)] if c.stats(mode) and st.plan.n_chunks > 0 else [])
            assert sorted(parts) == sorted(want), (note, want)
    if c.graph.startswith("bounds") and c.plan:
        assert st.plan.n_chunks > 0 and st.csc()[0].plan.n_chunks > 0
    n, n_cols, nnz, H = rp.shape[0] - 1, ins["h"].shape[0], ci.shape[0], c.H
    rows = edge_rows(rp)
    np_ = {k: v.cpu().numpy() for k, v in ins.items() if v is not None}
    gn = g.cpu().numpy()
    slope = np.float32(SLOPE)
    # logits, bit for bit as the kernels form them
    z = (np_["h_l"][rows] + np_["h_r"][ci]) + np_["h_e"][etype]
    assert np.all(z[rp[:-1][np.diff(rp) > 0]] == 0)
    logit = np.where(z > 0, z, z * slope).astype(np.float32)
    att_n, mix_n = att.cpu().numpy(), mix.cpu().numpy()
    check_softmax(np.abs(att_n), logit, rp, f"{c.id} attention")
    dropped = np.signbit(att_n)
    if c.p:
        assert np.array_equal(dropped, ~keep_mask(seed, nnz, H, c.p)), "the sign bits are not the dropout mask"
    else:
        assert not dropped.any()
    # mix, bit for bit over the kernel's own attention; the inference call writes the same bits
    scale = drop[2] if drop else 1.0                     # a Python float: the kernels take fl(scale)
    keep_scale = np.float32(scale)
    want_mix = np.where(dropped, np.float32(0), (np.abs(att_n) * keep_scale).astype(np.float32)).astype(np.float32)
    if c.res:
        alpha32 = np.float32(c.alpha)
        keep32 = np.float32(np.float32(1) - alpha32)
        want_mix = ((want_mix * keep32).astype(np.float32) + (np_["res"] * alpha32).astype(np.float32))
    assert np.array_equal(np_bits(mix_n), np_bits(want_mix)), f"{c.id}: mix differs from its fp32 emulation"
    assert torch.equal(mix_inf.view(torch.int32), mix.view(torch.int32)), f"{c.id}: the inference call's mix differs"

    # the layer: forward and backward through the autograd function
    out, mix_a, leaves = run(rs, ins, c, seed)
    assert torch.equal(mix_a.view(torch.int32), mix.view(torch.int32))
    out.backward(g)
    h64 = np_["h"].astype(np.float64)
    terms = mix_n[:, :, None].astype(np.float64) * h64[ci]                       # [nnz, H, F]
    deg = np.diff(rp).astype(np.float64)[:, None]
    assert_within(out.detach().cpu().numpy().reshape(n, H * F), seg_reduce(np.add, terms.reshape(nnz, H * F), rp),
                  deg * U32 * seg_reduce(np.add, np.abs(terms).reshape(nnz, H * F), rp) + TINY, f"{c.id} out")
    coldeg = np.bincount(ci, minlength=n_cols).astype(np.float64)[:, None]
    dterms = mix_n[:, :, None].astype(np.float64) * gn[rows].astype(np.float64)
    assert_within(leaves["h"].grad.cpu().numpy().reshape(n_cols, H * F),
                  col_sum(dterms.reshape(nnz, H * F), ci, n_cols),
                  coldeg * U32 * col_sum(np.abs(dterms).reshape(nnz, H * F), ci, n_cols) + TINY, f"{c.id} d h")
    # d m, as the backward forms it, then the attention backward on it
    dm = mhsddmm_raw(st, g, ins["h"]).cpu().numpy()
    sd = gn[rows].astype(np.float64) * h64[ci]
    assert_within(dm, sd.sum(-1), F * U32 * np.abs(sd).sum(-1) + TINY, f"{c.id} d m")
    if c.res:
        assert np.array_equal(np_bits(leaves["res"].grad.cpu().numpy()), np_bits(dm * np.float32(c.alpha))), "d res"
    gs = np.float32((1.0 - (c.alpha if c.res else 0.0)) * scale)    # the layer's grad_scale, rounded once
    d_edge, g_row = hgn_attn_bwd_raw(st, rs.type, att, torch.from_numpy(dm).to(dev), ins["h_l"], ins["h_r"],
                                     ins["h_e"], SLOPE, float(gs))
    gk = np.where(dropped, np.float32(0), (dm * gs).astype(np.float32))
    dact = np.where(z > 0, 1.0, np.float64(slope))
    ref, bound, grow, gbound = softmax_bwd64(rp, np.abs(att_n), gk, dact)
    de = d_edge.cpu().numpy()
    assert_within(de, ref, bound, f"{c.id} d edge")
    assert_within(leaves["h_l"].grad.cpu().numpy(), grow, gbound, f"{c.id} d h_l")
    assert torch.equal(leaves["h_l"].grad, g_row)
    # d h_r: the column sums of the kernel's d edge; d h_e: its per-type sums
    de64 = de.astype(np.float64)
    assert_within(leaves["h_r"].grad.cpu().numpy(), col_sum(de64, ci, n_cols),
                  coldeg * U32 * col_sum(np.abs(de64), ci, n_cols) + TINY, f"{c.id} d h_r")
    tdeg = np.bincount(etype, minlength=c.T).astype(np.float64)[:, None]
    dhe = leaves["h_e"].grad.cpu().numpy()
    assert_within(dhe, col_sum(de64, etype, c.T), (tdeg + 2) * U32 * col_sum(np.abs(de64), etype, c.T) + TINY,
                  f"{c.id} d h_e")
    unused = tdeg[:, 0] == 0
    assert unused.any() or c.T == 1
    assert np.all(dhe[unused] == 0), f"{c.id}: d h_e of a type no edge carries is not 0"
    if c.res and c.alpha == 1.0:
        for k in ("h_l", "h_r", "h_e"):
            assert int(torch.count_nonzero(leaves[k].grad)) == 0, f"{c.id}: d {k} is not 0 at alpha = 1"
    print(" ".join(f"[{k}: worst err/bound {v:.3g}]" for k, v in test_gpu_dispatch.RATIOS.items()))


def test_backward_kernel_and_kept_set(dev):
    """The backward's attention pass is the row's MODE 3 kernel, and the saved attention's sign bits are the dropped
    set of keep_mask exactly."""
    import cogdl_b200
    from cogdl_b200.operators._raw import attn_dropout_args, hgn_attn_bwd_raw, hgn_attn_raw

    c = next(r for r in TABLE if r.graph == "two_hubs" and r.H == 8 and r.p and r.res)
    rp, ci, st, rs, etype, ins, g = row_inputs(c, dev)
    drop_below, scale = attn_dropout_args(c.p)
    mix, att = hgn_attn_raw(st, rs.type, ins["h_l"], ins["h_r"], ins["h_e"], SLOPE, True, (77, drop_below, scale),
                            ins["res"], ALPHA)
    dropped = (att.view(torch.int32) < 0).cpu().numpy()
    assert np.array_equal(~dropped, keep_mask(77, ci.shape[0], c.H, c.p))
    hgn_attn_bwd_raw(st, rs.type, att, torch.ones_like(att), ins["h_l"], ins["h_r"], ins["h_e"], SLOPE, 1.0)
    note = cogdl_b200._cabi.last_kernel()
    assert c.stats(3) in note and c.kernel(3) in note, note


def test_same_seed_same_bits(dev):
    c = next(r for r in TABLE if r.graph == "two_hubs" and r.H == 8 and r.p and r.res)
    _, _, _, rs, _, ins, g = row_inputs(c, dev)
    got = []
    for _ in range(2):
        out, att, leaves = run(rs, ins, c, 99)
        out.backward(g)
        got.append([out, att] + [leaves[k].grad for k in ("h", "h_l", "h_r", "h_e", "res")])
    for a, b in zip(*got):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))


def _graph_from_coo(row, col, n, dev):
    import cogdl_b200

    return cogdl_b200.Graph(edge_index=(row.to(dev), col.to(dev)), num_nodes=n)


def _stand_ins(d, dev):
    convs = [HgnConvStandIn(6, 5, 16, 8, 8, attn_drop=0.0, activation=torch.tanh),
             HgnConvStandIn(6, 5, 64, 8, 8, attn_drop=0.0, residual=True, activation=torch.tanh, alpha=ALPHA),
             HgnConvStandIn(6, 5, 64, 3, 1, attn_drop=0.0)]
    for k, conv in enumerate(convs, 1):
        with torch.no_grad():
            for name, prm in conv.named_parameters():
                prm.copy_(torch.from_numpy(d[f"c{k}_{name}"]))
    return [c.to(dev) for c in convs]


def test_rebound_layer_reproduces_the_golden_file(dev):
    import cogdl_b200

    d = dict(np.load(GOLDEN))
    convs = _stand_ins(d, dev)
    cogdl_b200.install_simple_hgn(HgnConvStandIn)
    try:
        n = d["x"].shape[0]
        graph = _graph_from_coo(torch.from_numpy(d["row"]), torch.from_numpy(d["col"]), n, dev)
        graph.edge_type = torch.from_numpy(d["type"]).to(dev)        # COO order: the hook reorders it
        x = torch.from_numpy(d["x"]).to(dev).requires_grad_(True)
        out1, att1 = convs[0](graph, x)
        out2, att2 = convs[1](graph, out1, res_attn=att1)
        out3, att3 = convs[2](graph, out2)
        assert torch.equal(graph.edge_type.cpu(), torch.from_numpy(d["type"][d["order"]]))
        ((out2 * torch.from_numpy(d["g2"]).to(dev)).sum() + (out3 * torch.from_numpy(d["g3"]).to(dev)).sum()).backward()
        for k, (o, a) in enumerate(((out1, att1), (out2, att2), (out3, att3)), 1):
            close(o, torch.from_numpy(d[f"out{k}"]), f"out{k}")
            close(a, torch.from_numpy(d[f"att{k}"]), f"att{k}")        # the fixture's attention is in CSR order
        close(x.grad, torch.from_numpy(d["grad_x"]), "grad x")
        for k, conv in enumerate(convs, 1):
            for name, prm in conv.named_parameters():
                ref = torch.from_numpy(d[f"grad_c{k}_{name}"])
                a, b = prm.grad.double().cpu(), ref.double()
                assert float((a - b).abs().max()) <= 2e-5 * max(float(b.abs().max()), 1e-30), f"grad c{k}.{name}"
    finally:
        cogdl_b200.uninstall_simple_hgn(HgnConvStandIn)


def test_coo_types_follow_their_edges(dev):
    """hgn_attention on a graph built from a shuffled COO, with types reordered as the CSR build reorders the edges,
    equals the restatement on CSR-ordered inputs."""
    import cogdl_b200

    g = torch.Generator().manual_seed(5)
    n, e, H, T = 200, 2500, 4, 5
    row, col = torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g)
    etype = torch.randint(0, T, (e,), generator=g)
    graph = _graph_from_coo(row, col, n, dev)
    order = torch.sort(row, stable=True).indices
    rp = graph.row_indptr.cpu().numpy()
    ci = graph.col_indices.cpu().numpy()
    assert np.array_equal(ci, col[order].numpy())
    h, hl, hr, he = (torch.randn(*s, generator=g).to(dev) for s in ((n, H, F), (n, H), (n, H), (T, H)))
    out, att = cogdl_b200.hgn_attention(graph, h, hl, hr, he, etype[order].to(dev), SLOPE)
    _, m = hgn_attention_fp64(rp, ci, etype[order].numpy(), hl.double(), hr.double(), he.double(), SLOPE)
    close(att, m, "attention")
    close(out, aggregate_fp64(rp, ci, m, h.double()), "out")


def test_errors_raise_before_any_launch(dev):
    import cogdl_b200

    rp, ci, n = case("hub")
    graph = cogdl_b200.Graph(row_ptr=torch.from_numpy(rp), col=torch.from_numpy(ci), num_nodes=n).to(dev)
    H = 8
    h, hl, hr = torch.randn(n, H, F, device=dev), torch.randn(n, H, device=dev), torch.randn(n, H, device=dev)
    he = torch.randn(5, H, device=dev)
    et = torch.randint(0, 5, (ci.shape[0],), device=dev)
    cogdl_b200.hgn_attention(graph, h, hl, hr, he, et, SLOPE)      # builds and caches what the calls below share
    before = cogdl_b200._cabi.launch_count()
    bad = et.clone()
    bad[3] = 5
    with pytest.raises(ValueError):
        cogdl_b200.hgn_attention(graph, h, hl, hr, he, bad, SLOPE)
    bad[3] = -1
    with pytest.raises(ValueError):
        cogdl_b200.hgn_attention(graph, h, hl, hr, he, bad, SLOPE)
    with pytest.raises(ValueError):
        cogdl_b200.hgn_attention(graph, h, hl, hr, torch.randn(MAX_TABLE // H + 1, H, device=dev), et, SLOPE)
    with pytest.raises(RuntimeError):
        cogdl_b200.hgn_attention(graph, h.cpu(), hl, hr, he, et, SLOPE)
    with pytest.raises(TypeError):
        cogdl_b200.hgn_attention(graph, h, hl.double(), hr, he, et, SLOPE)
    assert cogdl_b200._cabi.launch_count() == before


def test_uninstall_restores_the_original(dev):
    import cogdl_b200

    original = HgnConvStandIn.forward
    assert cogdl_b200.install_simple_hgn(HgnConvStandIn)
    assert HgnConvStandIn.forward is not original
    cogdl_b200.uninstall_simple_hgn(HgnConvStandIn)
    assert HgnConvStandIn.forward is original


def test_example_layer_under_the_hook(dev):
    from tests.refpkg import reference_dir

    conv = os.path.join(ROOT, "oracle", "_ref", "examples", "simple_hgn", "conv.py")
    if reference_dir() is None or not os.path.exists(conv):
        pytest.skip("the reference package or the staged example (oracle/_ref) is not present")
    r = subprocess.run([sys.executable, "-m", "tests.simple_hgn_refpkg_check"], cwd=ROOT, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
    assert "simple_hgn refpkg ok" in r.stdout

"""Simple-HGN attention (cogdl_b200/csrc/simple_hgn.cu), cogdl_b200.hgn_attention and install_simple_hgn.

- Every row of tests/hgn_table.py records the kernels it names, and the output, the returned attention and the
  gradients of h, h_l, h_r, h_e and res_attn are within |a - b| <= 1e-5 max(|b|, scale) of the fp64 restatement
  (tests/simple_hgn_ref.py), scale the largest |b| of the tensor; the kept set is gat_dropout_ref.keep_mask exactly;
  the same seed gives the same bits, d h_e included.
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

from tests.gat_dropout_ref import keep_mask
from tests.graphs import boundary_csr, case
from tests.hgn_table import CHUNK, MAX_TABLE, TABLE
from tests.simple_hgn_ref import HgnConvStandIn, aggregate_fp64, hgn_attention_fp64

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "simple_hgn.npz")
SLOPE, ALPHA, F = 0.2, 0.05, 4


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import cogdl_b200

    assert cogdl_b200._cabi.load().cogdl_b200_check_device() == 0, cogdl_b200._cabi.last_error()
    return torch.device("cuda:0")


def close(a, b, what):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    if b.numel() == 0:
        return
    scale = float(b.abs().max())
    err = (a - b).abs() / torch.clamp(b.abs(), min=scale).clamp_min(1e-30)
    assert float(err.max()) <= 1e-5, f"{what}: {float(err.max()):.2e}"


def row_inputs(c, dev, seed=0):
    from cogdl_b200.structure import CSRStructure, RgcnStructure

    rp, ci, n_cols = boundary_csr(CHUNK) if c.graph == "bounds" else case(c.graph)
    st = CSRStructure(torch.from_numpy(rp).to(dev), torch.from_numpy(ci).to(dev), n_cols=n_cols,
                      chunk_edges=CHUNK if c.plan else 0)
    rng = np.random.default_rng(1000 + c.H + 7 * c.T + seed)
    n, nnz = rp.shape[0] - 1, ci.shape[0]
    etype = rng.integers(0, c.T, nnz).astype(np.int32)
    t = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(np.float32)).to(dev)  # noqa: E731
    ins = {"h": t(n_cols, c.H, F), "h_l": t(n, c.H), "h_r": t(n_cols, c.H), "h_e": t(c.T, c.H),
           "res": torch.from_numpy(rng.random((nnz, c.H)).astype(np.float32)).to(dev) if c.res else None}
    return rp, ci, st, RgcnStructure(st, torch.from_numpy(etype).to(dev)), etype, ins, t(n, c.H, F)


def run(rs, ins, c, seed):
    from cogdl_b200.operators._raw import attn_dropout_args
    from cogdl_b200.operators.simple_hgn import HgnAttentionFunction

    leaves = {k: v.clone().requires_grad_(True) for k, v in ins.items() if v is not None}
    drop = None
    if c.p:
        drop_below, scale = attn_dropout_args(c.p)
        drop = (seed, drop_below, scale)
    out, att = HgnAttentionFunction.apply(rs, leaves["h"], leaves["h_l"], leaves["h_r"], leaves["h_e"],
                                          leaves.get("res"), SLOPE, drop, ALPHA)
    return out, att, leaves


@pytest.mark.parametrize("c", TABLE, ids=lambda c: c.id)
def test_row_against_fp64(dev, c):
    import cogdl_b200

    from cogdl_b200.operators._raw import attn_dropout_args, hgn_attn_bwd_raw, hgn_attn_raw

    rp, ci, st, rs, etype, ins, g = row_inputs(c, dev)
    seed = 12345 + c.H
    # the kernels the row names: the attention stage and its backward, each recorded by its own call
    drop = (seed, *attn_dropout_args(c.p)) if c.p else None
    _, att0 = hgn_attn_raw(st, rs.type, ins["h_l"], ins["h_r"], ins["h_e"], SLOPE, True, drop, ins["res"], ALPHA)
    for mode in (2, 3):
        if mode == 3:
            hgn_attn_bwd_raw(st, rs.type, att0, torch.ones_like(att0), ins["h_l"], ins["h_r"], ins["h_e"], SLOPE, 1.0)
        note = cogdl_b200._cabi.last_kernel()
        if ci.shape[0] > 0:
            parts = [p.replace(" cp.async.bulk tiles", "") for p in note.split(" + ")]
            want = [c.kernel(mode)] + ([c.stats(mode)] if c.stats(mode) and st.plan.n_chunks > 0 else [])
            assert sorted(parts) == sorted(want), (note, want)
    out, att, leaves = run(rs, ins, c, seed)
    out.backward(g)
    keep = keep_mask(seed, ci.shape[0], c.H, c.p) if c.p else None
    d = {k: v.detach().double().requires_grad_(True) for k, v in ins.items() if v is not None}
    _, m = hgn_attention_fp64(rp, ci, etype, d["h_l"], d["h_r"], d["h_e"], SLOPE, keep, c.p, d.get("res"), ALPHA)
    ref = aggregate_fp64(rp, ci, m, d["h"])
    ref.backward(g.double())
    close(out, ref, "out")
    close(att, m, "attention")
    if keep is not None:
        kept = (att != 0) if not c.res else None
        if kept is not None:
            assert torch.equal(kept.cpu(), torch.from_numpy(keep) & (m.detach().cpu() != 0)), "kept set"
    for k in d:
        close(leaves[k].grad, d[k].grad, f"d {k}")


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

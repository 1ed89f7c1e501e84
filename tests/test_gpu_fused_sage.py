"""Fused GraphSAGE layer (aggregation + neighbour half of fc in the wgmma epilogue) against an fp64 evaluation of
the reference order fc(cat[x, agg(x)]) (cogdl/layers/sage_layer.py:69-87), agg from the oracle:
element-wise |a-b| <= 1e-5 * max(|b|, row scale).  The layout and aggregated-tile cases isolate the pieces
(operand layout, the aggregation written into the tile) so a failure names its cause."""
import numpy as np
import pytest
import torch

import oracle
from tests.gpu_util import dev, plan_structure, row_err
from tests.graphs import case

pytestmark = pytest.mark.gpu
TOL = 1e-5
AGGS = ["sum_weighted", "sum_unweighted", "mean_baked", "mean_in_norm", "max"]


@pytest.fixture(scope="module", autouse=True)
def _no_cudnn_tf32():
    torch.backends.cudnn.allow_tf32 = False


def inputs(kind, rp, ci, dev, g):
    """(val, row_scale, raw aggr) for one aggregation kind; mean = sum with 1/deg baked in or as the row scale."""
    n = rp.shape[0] - 1
    deg = np.diff(rp).astype(np.float32)
    inv = np.where(deg > 0, np.float32(1) / np.maximum(deg, 1), np.float32(0)).astype(np.float32)
    if kind == "sum_weighted":
        return torch.rand(ci.shape[0], device=dev, generator=g), None, "sum"
    if kind == "mean_baked":
        return torch.from_numpy(np.repeat(inv, np.diff(rp))).to(dev), None, "sum"
    if kind == "mean_in_norm":
        return None, torch.from_numpy(inv).to(dev).view(n, 1), "sum"
    return None, None, "max" if kind == "max" else "sum"


def oracle_agg(rp, ci, val, row_scale, aggr, x):
    xn = x.cpu().numpy()
    if aggr == "max":
        return torch.from_numpy(oracle.scatter_max_fwd(rp, ci, xn)[0])
    a = oracle.spmm_csr(rp, ci, None if val is None else val.cpu().numpy(), xn)
    if row_scale is not None:
        a = row_scale.cpu().numpy().astype(np.float32) * a          # fp32 product, as `in_norm * x`
    return torch.from_numpy(a)


def ref_layer(x, agg, W, b, relu):
    n = agg.shape[0]
    h = torch.cat([x[:n].double().cpu(), agg.double()], dim=1) @ W.double().cpu().t()
    if b is not None:
        h = h + b.double().cpu()
    return torch.relu(h) if relu else h


def unfused_agg(st, val, row_scale, aggr, x):
    from cogdl_b200.operators._raw import scatter_max_fwd_raw, spmm_raw

    if aggr == "max":
        return scatter_max_fwd_raw(st, x)[0]
    a = spmm_raw(st, val, x)
    return a if row_scale is None else row_scale * a


@pytest.mark.parametrize("aggr", ["sum", "max"])
def test_identity_graph_layout(dev, aggr):
    """A = I, W_self = 0, W_neigh = I, b = 0: OUT must be x itself (operand layout, accumulator read-back, S add)."""
    from cogdl_b200.operators.fused_sage import fused_sage_raw

    n = 300                                               # 3 tiles, the last one partial
    rp = np.arange(n + 1, dtype=np.int32)
    ci = np.arange(n, dtype=np.int32)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(n, 128, device=dev, generator=g)
    st = plan_structure(rp, ci, n, dev, chunk=64)
    eye = torch.cat([torch.zeros(128, 128, device=dev), torch.eye(128, device=dev)], dim=1)
    for fout in (128, 16, 40, 7, 100):                     # N padding and the masked / unvectorised stores
        out = fused_sage_raw(st, None, None, x, eye[:fout].contiguous(), None, aggr, False)
        assert out.shape == (n, fout)
        assert row_err(out, x[:, :fout]) <= 1e-6, f"operand layout / read-back broken at Fout={fout}"
    W = torch.randn(100, 256, device=dev, generator=g) / 16
    b = torch.randn(100, device=dev, generator=g)
    out = fused_sage_raw(st, None, None, x, W, b, aggr, True)
    assert row_err(out, ref_layer(x, x.cpu(), W, b, True)) <= TOL


@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "two_hubs", "empty_graph"])
@pytest.mark.parametrize("kind", AGGS)
@pytest.mark.parametrize("fout", [128, 40])
def test_fused_sage_matches_reference_order_fp64(dev, name, kind, fout):
    from cogdl_b200.operators.fused_sage import fused_sage_raw

    rp, ci, n_cols = case(name)
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(n_cols, 128, device=dev, generator=g)          # mixed signs: max must not clamp at 0
    val, row_scale, aggr = inputs(kind, rp, ci, dev, g)
    W = torch.randn(fout, 256, device=dev, generator=g) / 16
    b = torch.randn(fout, device=dev, generator=g)
    agg = oracle_agg(rp, ci, val, row_scale, aggr, x)
    for chunk in (64, 16):
        st = plan_structure(rp, ci, n_cols, dev, chunk=chunk)
        for relu in (False, True):
            out = fused_sage_raw(st, val, row_scale, x, W, b, aggr, relu)
            assert row_err(out, ref_layer(x, agg, W, b, relu)) <= TOL, (chunk, relu)
        assert int(st.plan.counters.abs().sum()) == 0


@pytest.mark.parametrize("name", ["ragged", "hub", "two_hubs"])
@pytest.mark.parametrize("kind", AGGS)
def test_aggregated_tile_is_the_unfused_aggregation(dev, name, kind):
    """W_self = 0, W_neigh = I, b = 0: the output is the aggregated tile, re-assembled from its three bf16 terms."""
    from cogdl_b200.operators.fused_sage import fused_sage_raw

    rp, ci, n_cols = case(name)
    g = torch.Generator(device=dev).manual_seed(3)
    x = torch.randn(n_cols, 128, device=dev, generator=g)
    val, row_scale, aggr = inputs(kind, rp, ci, dev, g)
    eye = torch.cat([torch.zeros(128, 128, device=dev), torch.eye(128, device=dev)], dim=1)
    for chunk in (64, 16):
        st = plan_structure(rp, ci, n_cols, dev, chunk=chunk)
        out = fused_sage_raw(st, val, row_scale, x, eye, None, aggr, False)
        assert row_err(out, unfused_agg(st, val, row_scale, aggr, x)) <= 1e-6, chunk
        assert int(st.plan.counters.abs().sum()) == 0


def symmetric_csr(name):
    rp, ci, n = case(name)
    row = np.repeat(np.arange(n), np.diff(rp))
    a = np.unique(np.concatenate([row * n + ci, ci.astype(np.int64) * n + row]))
    r, c = a // n, a % n
    rp2 = np.zeros(n + 1, np.int64)
    rp2[1:] = np.cumsum(np.bincount(r, minlength=n))
    return rp2, c.astype(np.int64), n


def make_graph(form, dev):
    """'sym': a symmetric structure as a CSR-only Graph (symmetric flag; mean goes through in_norm);
    'asym': a non-symmetric COO Graph flagged asymmetric (mean bakes 1/deg into the weights)."""
    import cogdl_b200

    if form == "sym":
        rp, col, n = symmetric_csr("two_hubs")
        return cogdl_b200.Graph(row_ptr=torch.from_numpy(rp).to(dev), col=torch.from_numpy(col).to(dev), num_nodes=n)
    rp, ci, n = case("two_hubs")
    row = torch.from_numpy(np.repeat(np.arange(n), np.diff(rp))).to(dev)
    gr = cogdl_b200.Graph(edge_index=(row, torch.from_numpy(ci.astype(np.int64)).to(dev)), num_nodes=n)
    gr.set_asymmetric()
    return gr


def pair(dev, in_feats=128, out_feats=64, **kw):
    from cogdl_b200.layers import SAGELayer

    torch.manual_seed(0)
    a = SAGELayer(in_feats, out_feats, **kw).to(dev)
    b = SAGELayer(in_feats, out_feats, fused=True, **kw).to(dev)
    b.load_state_dict(a.state_dict())
    return a, b


def check_layers(a, b, gr_a, gr_b, x, fused_expected=True):
    import cogdl_b200

    xa = x.detach().clone().requires_grad_(True)
    xb = x.detach().clone().requires_grad_(True)
    ya = a(gr_a, xa)
    yb = b(gr_b, xb)
    # with hub rows the fused layer records its pre-pass first: the fused kernel is the last launch named
    last = cogdl_b200._cabi.last_kernel().split(" + ")[-1]
    assert last.startswith("cogdl_b200::fg::fused_layer_kernel<sage-") == fused_expected, cogdl_b200._cabi.last_kernel()
    assert row_err(yb, ya) <= 2e-5
    gout = torch.randn_like(ya)
    ya.backward(gout)
    yb.backward(gout)
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert row_err(pb.grad.reshape(1, -1), pa.grad.reshape(1, -1)) <= 1e-4
    assert row_err(xb.grad, xa.grad) <= 1e-4


@pytest.mark.parametrize("aggr", ["mean", "sum", "max"])
@pytest.mark.parametrize("form", ["sym", "asym"])
def test_sage_layer_module_and_autograd(dev, aggr, form):
    a, b = pair(dev, aggr=aggr, activation="relu")
    gr_a, gr_b = make_graph(form, dev), make_graph(form, dev)
    x = torch.randn(gr_a.num_nodes, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(4))
    check_layers(a, b, gr_a, gr_b, x)


@pytest.mark.parametrize("kw,fused_expected", [
    ({"in_feats": 32}, False),
    ({"out_feats": 256}, False),
    ({"normalize": True}, True),          # fused aggregation + GEMM; normalize then ReLU after the kernel
    ({"norm": "layernorm"}, True),
])
def test_sage_layer_fallbacks_match_unfused(dev, kw, fused_expected):
    kw = dict(kw)
    fin, fout = kw.pop("in_feats", 128), kw.pop("out_feats", 64)
    a, b = pair(dev, fin, fout, aggr="mean", activation="relu", **kw)
    gr_a, gr_b = make_graph("asym", dev), make_graph("asym", dev)
    x = torch.randn(gr_a.num_nodes, fin, device=dev, generator=torch.Generator(device=dev).manual_seed(5))
    check_layers(a, b, gr_a, gr_b, x, fused_expected)


def test_sage_layer_minibatch_from_the_device_sampler(dev):
    """A sampled mini-batch as the reference's Graphsage trains it: CSR-only graph (rows of the batch, padded with
    empty rows to the sampled node count), aggr="mean" -> in_norm path."""
    import cogdl_b200
    from cogdl_b200 import synth
    from cogdl_b200.sampling import sample_adj

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0)
    ip, ix = rp.to(dev), col.to(dev)
    batch = torch.arange(0, n, 37, device=dev)
    out_ptr, out_idx, nodes, _ = sample_adj(ip, ix, batch, 10, False, seed=7)
    m = nodes.numel()
    row_ptr = torch.cat([out_ptr, out_ptr[-1:].expand(m - batch.numel())])
    feats = torch.randn(n, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(6))
    x = feats[nodes]
    graphs = [cogdl_b200.Graph(row_ptr=row_ptr, col=out_idx, num_nodes=m) for _ in range(2)]
    a, b = pair(dev, 128, 128, aggr="mean", activation="relu")
    check_layers(a, b, graphs[0], graphs[1], x)


@pytest.mark.parametrize("aggr", ["mean", "max"])
def test_fused_sage_full_arxiv_shape(dev, aggr):
    """C4 size: the whole arxiv-shaped graph, 128 -> 128 with bias and ReLU (mean as 1/deg row scale)."""
    from cogdl_b200 import synth
    from cogdl_b200.operators.fused_sage import fused_sage_raw

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0)
    rp32, ci32 = rp.numpy().astype(np.int32), col.numpy().astype(np.int32)
    st = plan_structure(rp32, ci32, n, dev, chunk=64)
    gen = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(n, 128, device=dev, generator=gen)
    W = torch.randn(128, 256, device=dev, generator=gen) / 16
    b = torch.randn(128, device=dev, generator=gen) * 0.1
    val, row_scale, raw = inputs("mean_in_norm" if aggr == "mean" else "max", rp32, ci32, dev, gen)
    out = fused_sage_raw(st, val, row_scale, x, W, b, raw, True)
    ref = ref_layer(x, oracle_agg(rp32, ci32, val, row_scale, raw, x), W, b, True)
    assert row_err(out, ref) <= TOL

"""Fused GCN layer (wgmma epilogue, SURVEY 8f-3) against an fp64 evaluation of the REFERENCE order
act(A.(X.W^T + b)) (cogdl/layers/gcn_layer.py:51-64): element-wise |a-b| <= 1e-5 * max(|b|, row scale).
The first three cases isolate the pieces (operand layout of A, of W, the accumulator read-back) so a
failure names its cause."""
import numpy as np
import pytest
import torch

from tests.gpu_util import dev, plan_structure, row_err
from tests.graphs import case

pytestmark = pytest.mark.gpu
TOL = 1e-5


def ref_layer(rp, ci, val, x, W, b, relu):
    n = rp.shape[0] - 1
    A = torch.sparse_csr_tensor(torch.from_numpy(rp.astype(np.int64)), torch.from_numpy(ci.astype(np.int64)),
                                torch.ones(ci.shape[0], dtype=torch.float64) if val is None else val.double().cpu(),
                                size=(n, x.shape[0]))
    h = x.double().cpu() @ W.double().cpu().t()
    if b is not None:
        h = h + b.double().cpu()
    out = A @ h
    return torch.relu(out) if relu else out


def test_identity_graph_is_a_plain_gemm(dev):
    """A = I: OUT = X.W^T + b -- exercises the operand layouts, descriptors and the accumulator fragment layout only."""
    from cogdl_b200.operators.fused_gcn import fused_gcn_raw

    n = 300                                               # 3 tiles, the last one partial
    rp = np.arange(n + 1, dtype=np.int32)
    ci = np.arange(n, dtype=np.int32)
    g = torch.Generator(device=dev).manual_seed(0)
    x = torch.randn(n, 128, device=dev, generator=g)
    st = plan_structure(rp, ci, n, dev, chunk=64)
    eye = torch.eye(128, device=dev)
    out = fused_gcn_raw(st, None, x, eye, None, False)     # W = I: OUT must be X itself (three-term split is exact)
    # (bit-exact if the tensor core adds the three terms without dropping bits; only 1e-6 is REQUIRED)
    assert row_err(out, x) <= 1e-6, f"A-operand layout / accumulator read-back broken: max diff {float((out - x).abs().max())}"
    W = torch.randn(128, 128, device=dev, generator=g) / 11.3
    b = torch.randn(128, device=dev, generator=g)
    out = fused_gcn_raw(st, None, x, W, b, False)
    assert row_err(out, ref_layer(rp, ci, None, x, W, b, False)) <= TOL
    for fout in (16, 40, 7, 100):                          # N padding and the masked / unvectorised stores
        Wn, bn = W[:fout].contiguous(), b[:fout].contiguous()
        out = fused_gcn_raw(st, None, x, Wn, bn, True)
        assert out.shape == (n, fout)
        assert row_err(out, ref_layer(rp, ci, None, x, Wn, bn, True)) <= TOL, fout


@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "two_hubs", "empty_graph"])
@pytest.mark.parametrize("fout", [128, 40])
@pytest.mark.parametrize("weighted", [True, False])
def test_fused_layer_matches_reference_order_fp64(dev, name, fout, weighted):
    from cogdl_b200.operators.fused_gcn import fused_gcn_raw
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n_cols = case(name)
    if n_cols != rp.shape[0] - 1:
        pytest.skip("square graphs")
    n = rp.shape[0] - 1
    g = torch.Generator(device=dev).manual_seed(1)
    x = torch.randn(n_cols, 128, device=dev, generator=g)
    val = torch.rand(ci.shape[0], device=dev, generator=g) if weighted else None
    W = torch.randn(fout, 128, device=dev, generator=g) / 11.3
    b = torch.randn(fout, device=dev, generator=g)
    for chunk in (64, 16):
        st = plan_structure(rp, ci, n_cols, dev, chunk=chunk)
        for relu in (False, True):
            out = fused_gcn_raw(st, val, x, W, b, relu)
            assert row_err(out, ref_layer(rp, ci, val, x, W, b, relu)) <= TOL, (chunk, relu)
            out = fused_gcn_raw(st, val, x, W, b, relu, cache_rowsum=False)      # hub weight sums inside the kernel
            assert row_err(out, ref_layer(rp, ci, val, x, W, b, relu)) <= TOL, (chunk, relu, "no cached row sums")
        # W = I, no bias: the fused kernel's aggregated tile is the SpMM output (re-assembled from its three bf16 terms)
        if fout == 128:
            out = fused_gcn_raw(st, val, x, torch.eye(128, device=dev), None, False)
            assert row_err(out, spmm_raw(st, val, x)) <= 1e-6, chunk
        assert int(st.plan.counters.abs().sum()) == 0


def test_fused_layer_module_and_autograd_names_pre_pass_and_layer(dev):
    """GCNLayer(fused=True) against the unfused layer, forward and gradients; on a graph with hub rows the layer records
    both of its launches: the SpMM's hub pre-pass, then the fused kernel."""
    import cogdl_b200
    from cogdl_b200.layers import GCNLayer

    rp, ci, n_cols = case("two_hubs")
    n = n_cols
    # The graph is made symmetric, as the Graph default assumes (both backward paths use A for A^T).  It is given
    # with COO rows so that sym_norm() bakes the scaling into the edge weights, the form the fused layer takes: a
    # CSR-only graph keeps it in in/out norms, and GCNLayer then runs the unfused path.
    rows = np.repeat(np.arange(n), np.diff(rp))
    pairs = np.unique(np.concatenate([np.stack([rows, ci], 1), np.stack([ci, rows], 1)]), axis=0)
    gr = cogdl_b200.Graph(edge_index=(torch.from_numpy(pairs[:, 0]).to(dev), torch.from_numpy(pairs[:, 1]).to(dev)),
                          num_nodes=n)
    gr.sym_norm()
    assert gr.in_norm is None and gr.out_norm is None
    torch.manual_seed(0)
    a = GCNLayer(128, 64, activation="relu").to(dev)
    b = GCNLayer(128, 64, activation="relu", fused=True).to(dev)
    b.load_state_dict(a.state_dict())
    x = torch.randn(n, 128, device=dev, requires_grad=True)
    x2 = x.detach().clone().requires_grad_(True)
    ya, yb = a(gr, x), b(gr, x2)
    # the graph has hub rows: the SpMM hub pre-pass, then the fused kernel
    launches = cogdl_b200._cabi.last_kernel().split(" + ")
    assert len(launches) == 2 and launches[0].startswith("cogdl_b200::stream_kernel<"), launches
    assert launches[1].startswith("cogdl_b200::fg::fused_layer_kernel<gcn,"), launches
    assert row_err(yb, ya) <= 2e-5
    g = torch.randn_like(ya)
    ya.backward(g)
    yb.backward(g)
    for pa, pb in zip(a.parameters(), b.parameters()):
        assert row_err(pb.grad.reshape(1, -1), pa.grad.reshape(1, -1)) <= 1e-4
    assert row_err(x2.grad, x.grad) <= 1e-4


def test_fused_layer_full_arxiv_shape(dev):
    """C2 size: the whole arxiv-shaped graph, sym-normalised weights, 128 -> 128 with bias and ReLU."""
    import cogdl_b200
    from cogdl_b200 import synth
    from cogdl_b200.operators.fused_gcn import fused_gcn_raw

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0)
    w = synth.sym_norm_weights(rp, col)
    g = cogdl_b200.Graph(row_ptr=rp, col=col, edge_weight=w, num_nodes=n).to(dev)
    st = g.structure()
    gen = torch.Generator(device=dev).manual_seed(2)
    x = torch.randn(n, 128, device=dev, generator=gen)
    W = torch.randn(128, 128, device=dev, generator=gen) / 11.3
    b = torch.randn(128, device=dev, generator=gen) * 0.1
    out = fused_gcn_raw(st, g.raw_edge_weight, x, W, b, True)
    ref = ref_layer(rp.numpy().astype(np.int32), col.numpy().astype(np.int32), w, x, W, b, True)
    assert row_err(out, ref) <= TOL

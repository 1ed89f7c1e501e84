"""GENConv aggregation kernels (cogdl_b200/csrc/softmax_aggr.cu) and genconv_aggregate against the fp64 restatement
of tests/genconv_ref.py (itself pinned to the reference GENConv by tests/test_cpu_genconv_golden.py)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import graphs
from tests.genconv_ref import genconv_aggregate_fp64
from tests.gpu_util import dev, plan_structure, row_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def structure(name, dev, chunk=None):
    from cogdl_b200.structure import DEFAULT_CHUNK_EDGES

    rp, ci, n_cols = graphs.case(name)
    return plan_structure(rp, ci, n_cols, dev, chunk=DEFAULT_CHUNK_EDGES if chunk is None else chunk), rp, ci, n_cols


@pytest.mark.parametrize("chunk", [None, 16])
@pytest.mark.parametrize("edge", [False, True])
@pytest.mark.parametrize("F", [7, 16, 64, 128, 256])
@pytest.mark.parametrize("name", list(graphs.CASES))
def test_forward_matches_fp64(dev, name, F, edge, chunk):
    from cogdl_b200 import genconv_aggregate

    st, rp, ci, n_cols = structure(name, dev, chunk)
    g = torch.Generator(device=dev).manual_seed(F)
    x = torch.randn(n_cols, F, device=dev, generator=g)
    a = 0.5 * torch.randn(st.nnz, F, device=dev, generator=g) if edge else None
    for beta in (0.0, 0.5, 1.0, 4.0):
        got = genconv_aggregate(st, x, "softmax_sg", beta=beta, edge_term=a)
        want = genconv_aggregate_fp64(st.rowptr, st.colind, x, "softmax_sg", beta=beta, edge_term=a)
        assert got.shape == (st.n_rows, F)
        assert row_err(got, want) <= 1e-5, f"beta={beta}"
    for aggr in ("softmax", "mean", "sum") + (() if edge else ("max", "powermean")):
        got = genconv_aggregate(st, x, aggr, edge_term=a, p=2.0)
        want = genconv_aggregate_fp64(st.rowptr, st.colind, x, aggr, edge_term=a, p=2.0)
        assert row_err(got, want) <= 1e-5, aggr


def test_large_logits(dev):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure("two_hubs", dev)
    g = torch.Generator(device=dev).manual_seed(3)
    x = 4.0 * torch.rand(st.n_cols, 128, device=dev, generator=g)
    beta = torch.full((1,), 20.0, device=dev)                     # beta * m up to 80
    got = genconv_aggregate(st, x, "softmax_sg", beta=beta)
    assert torch.isfinite(got).all()
    assert row_err(got, genconv_aggregate_fp64(st.rowptr, st.colind, x, "softmax_sg", beta=20.0)) <= 1e-5


@pytest.mark.parametrize("aggr", ["softmax_sg", "softmax", "mean", "sum"])
@pytest.mark.parametrize("edge", [False, True])
@pytest.mark.parametrize("name", ["ragged", "hub", "two_hubs", "rect"])
def test_gradients_match_fp64_autograd(dev, name, edge, aggr):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev)
    F = 64
    g = torch.Generator(device=dev).manual_seed(11)
    x = torch.randn(st.n_cols, F, device=dev, generator=g)
    a = 0.5 * torch.randn(st.nnz, F, device=dev, generator=g) if edge else None
    r = torch.randn(st.n_rows, F, device=dev, generator=g)
    beta = torch.full((1,), 1.5, device=dev)

    def grads(fn, dtype):
        xs = x.clone().to(dtype).requires_grad_(True)
        as_ = None if a is None else a.clone().to(dtype).requires_grad_(True)
        bs = beta.clone().to(dtype).requires_grad_(aggr == "softmax_sg")
        out = fn(xs, as_, bs)
        (out * r.to(dtype)).sum().backward()
        return xs.grad, None if as_ is None else as_.grad, bs.grad

    got = grads(lambda x_, a_, b_: genconv_aggregate(st, x_, aggr, beta=b_, edge_term=a_), torch.float32)
    want = grads(lambda x_, a_, b_: genconv_aggregate_fp64(st.rowptr, st.colind, x_, aggr, beta=b_, edge_term=a_),
                 torch.float64)
    assert row_err(got[0], want[0]) <= 1e-4
    if edge:
        assert row_err(got[1], want[1]) <= 1e-4
    if aggr == "softmax_sg":
        assert row_err(got[2], want[2]) <= 1e-4
    else:
        assert got[2] is None


@pytest.mark.parametrize("name", ["hub", "two_hubs"])
def test_forward_backward_bitwise_reproducible(dev, name):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev, 16)
    g = torch.Generator(device=dev).manual_seed(5)
    x0 = torch.randn(st.n_cols, 128, device=dev, generator=g)
    a0 = torch.randn(st.nnz, 128, device=dev, generator=g)
    r = torch.randn(st.n_rows, 128, device=dev, generator=g)

    def once():
        x, a = x0.clone().requires_grad_(True), a0.clone().requires_grad_(True)
        b = torch.full((1,), 0.8, device=dev, requires_grad=True)
        out = genconv_aggregate(st, x, "softmax_sg", beta=b, edge_term=a)
        (out * r).sum().backward()
        return out.detach(), x.grad, a.grad, b.grad

    first, second = once(), once()
    assert all(torch.equal(u, v) for u, v in zip(first, second))


def test_kernel_notes(dev):
    from cogdl_b200 import _cabi, genconv_aggregate

    st, *_ = structure("hub", dev)
    x = torch.randn(st.n_cols, 128, device=dev, requires_grad=True)
    genconv_aggregate(st, x, "softmax_sg", beta=torch.ones(1, device=dev))
    assert _cabi.last_kernel() == "cogdl_b200::softmax_aggr_fwd_kernel<float4,no_edge_term,no_Q>"
    genconv_aggregate(st, x, "softmax_sg", beta=torch.ones(1, device=dev, requires_grad=True))
    assert _cabi.last_kernel() == "cogdl_b200::softmax_aggr_fwd_kernel<float4,no_edge_term,Q>"
    genconv_aggregate(st, x[:, :7].contiguous(), "softmax")
    assert _cabi.last_kernel() == "cogdl_b200::softmax_aggr_fwd_kernel<float,no_edge_term,no_Q>"


def test_errors(dev):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure("tiny", dev)
    x = torch.randn(st.n_cols, 8, device=dev)
    with pytest.raises(RuntimeError):
        genconv_aggregate(st, x.cpu(), "softmax_sg", beta=1.0)
    with pytest.raises(TypeError):
        genconv_aggregate(st, x.half(), "softmax_sg", beta=1.0)
    with pytest.raises(ValueError):
        genconv_aggregate(st, x[:-1], "softmax_sg", beta=1.0)
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_term=torch.randn(st.nnz + 1, 8, device=dev))
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax_sg")
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "median")
    for aggr in ("max", "powermean"):
        with pytest.raises(NotImplementedError):
            genconv_aggregate(st, x, aggr, edge_term=torch.randn(st.nnz, 8, device=dev))


def test_full_arxiv_shape_forward(dev):
    """The whole arxiv-shaped graph (the benchmark's) at F = 128, fp64 evaluation on the GPU."""
    from cogdl_b200 import genconv_aggregate, synth
    from cogdl_b200.structure import CSRStructure

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, device=dev, self_loops=True)
    st = CSRStructure.from_int64(rp, col)
    x = torch.randn(st.n_cols, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    got = genconv_aggregate(st, x, "softmax_sg", beta=1.0)
    want = genconv_aggregate_fp64(st.rowptr, st.colind, x, "softmax_sg", beta=1.0)
    assert row_err(got, want) <= 1e-5


def test_reference_deepergcn_through_install():
    """Reference DeeperGCN (softmax_sg) and a GENConv with an EdgeEncoder through install(genconv=True), in a child
    process (tests/genconv_refpkg_check.py): logits vs the reference CPU run, gradients vs fp64."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.genconv_refpkg_check"], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["untouched_without_flag"], "install() without genconv=True must leave GENConv.forward alone"
    assert res["rebound"] and res["patched"][-1] == "cogdl.layers.deepergcn_layer.GENConv.forward"
    for name in ("deepergcn", "genconv_edge"):
        m = res[name]
        assert m["logits_vs_ref_cpu"] <= 1e-4, (name, m)
        assert m["logits_vs_fp64"] <= 1e-4, (name, m)
        assert m["grads_present"], (name, m)
    # GENConv alone: every gradient within 1e-4 of its own scale
    assert max(res["genconv_edge"]["grad_errs"].values()) <= 1e-4, res["genconv_edge"]
    # DeeperGCN: each ResGNNLayer starts with a BatchNorm, so the biases in front of one have an exact gradient of 0
    # and the layers below it a nearly cancelled one; those are measured against the model's largest gradient.  fp32
    # cancellation through the BatchNorms leaves 1.5e-4 of that scale (measured), hence 1e-3 here
    assert max(res["deepergcn"]["grad_errs_model_scale"].values()) <= 1e-3, res["deepergcn"]
    assert res["max_edge_ran_original"], res

"""DisenGCN routing kernels (cogdl_b200/csrc/disen_routing.cu), DisenRouteFunction and disen_routing against the fp64
restatement of tests/disengcn_ref.py (itself pinned to the reference DisenGCNLayer by test_cpu_disengcn_golden.py)."""
import json
import os
import subprocess
import sys

import pytest
import torch

from tests import graphs
from tests.disengcn_ref import disen_routing_fp64, normalize_channels_fp64, route_step_fp64
from tests.gpu_util import dev, misaligned, plan_structure, row_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SQUARE = [name for name in graphs.CASES if name != "rect"]


def route_err(got, want, norm):
    """row_err() of u = out |u| rather than of out, with the fp64 |u| [n, K] of the step that made `want`.  The last
    normalisation multiplies any rounding of u by 1 / |u|: where a + c nearly cancels (|u| -> 0: routinely for
    d = 1, where c = +-1) out is ill-conditioned in the layer itself, not in the kernel.  Channels whose fp64 |u|
    is below 1e-6 decide their direction by rounding and are left out."""
    n, F = want.shape
    K = norm.shape[1]
    keep = (norm.double().cpu() >= 1e-6)[..., None]
    scale = norm.double().cpu()[..., None] * keep
    u_got = torch.where(keep, got.detach().double().cpu().reshape(n, K, -1) * scale, 0.0)
    u_want = torch.where(keep, want.detach().double().cpu().reshape(n, K, -1) * scale, 0.0)
    return row_err(u_got.reshape(n, F), u_want.reshape(n, F))


def structure(name, dev, chunk=None):
    from cogdl_b200.structure import DEFAULT_CHUNK_EDGES

    rp, ci, n_cols = graphs.case(name)
    return plan_structure(rp, ci, n_cols, dev, chunk=DEFAULT_CHUNK_EDGES if chunk is None else chunk)


def unit_channels(n, K, d, dev, gen):
    return normalize_channels_fp64(torch.randn(n, K * d, device=dev, generator=gen), K).float()


@pytest.mark.parametrize("chunk", [None, 16])
@pytest.mark.parametrize("d", [1, 2, 4, 8, 16, 32])
@pytest.mark.parametrize("name", SQUARE)
def test_step_matches_fp64(dev, name, d, chunk):
    from cogdl_b200.operators._raw import disen_route_fwd_raw

    st = structure(name, dev, chunk)
    gen = torch.Generator(device=dev).manual_seed(d)
    for K in sorted({1, 3, 8, 256 // d}):                 # F from d up to 256; K = 3 leaves idle lanes
        q, c = unit_channels(st.n_rows, K, d, dev, gen), unit_channels(st.n_rows, K, d, dev, gen)
        for tau in (0.1, 1.0, 5.0):
            want, norm = route_step_fp64(st.rowptr, st.colind, q, c, K, tau, with_norm=True)
            for saved in (False, True):
                out, lse2, r = disen_route_fwd_raw(st, q, c, K, tau, want_saved=saved)
                assert out.shape == (st.n_rows, K * d)
                assert route_err(out, want, norm) <= 1e-5, (K, tau, saved)
                if saved:
                    # NaN where the reference has it (a zero-norm channel of c spreads to the rows routing to it);
                    # elsewhere |u| <= 2, an absolute bound
                    rn, nn = r.double().cpu(), norm.cpu()
                    assert torch.equal(rn.isnan(), nn.isnan()), (K, tau, "NaN pattern")
                    assert float((rn - nn).abs().nan_to_num(0.0).max()) <= 2e-5, (K, tau, "r")
            if d >= 4:
                out, _, _ = disen_route_fwd_raw(st, misaligned(q), misaligned(c), K, tau)
                assert route_err(out, want, norm) <= 1e-5, (K, tau, "misaligned")


@pytest.mark.parametrize("K,d", [(16, 4), (8, 8), (4, 2), (3, 32)])
@pytest.mark.parametrize("name", SQUARE)
def test_disen_routing_seven_iterations(dev, name, K, d):
    from cogdl_b200 import disen_routing

    st = structure(name, dev)
    h = torch.randn(st.n_rows, K * d, device=dev, generator=torch.Generator(device=dev).manual_seed(K * d))
    # tau = 0.1 multiplies any rounding of q by 1/tau = 10 in the next step's logits, seven times over: the plain
    # fp32 torch restatement of the layer is itself up to 7e-5 from fp64 here (measured), so that tau gets 1e-4
    for tau, bar in ((0.1, 1e-4), (1.0, 1e-5), (5.0, 1e-5)):
        got = disen_routing(st, h, K, 7, tau)
        assert route_err(got, *disen_routing_fp64(st.rowptr, st.colind, h, K, 7, tau, with_norm=True)) <= bar, tau
    assert row_err(disen_routing(st, h, K, 0, 1.0), normalize_channels_fp64(h, K)) <= 1e-6   # no iterations: c


@pytest.mark.parametrize("K,d", [(16, 4), (8, 8), (8, 2), (2, 32)])
@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "two_hubs"])
def test_step_gradients_match_fp64_autograd(dev, name, K, d):
    from cogdl_b200.operators.disen_routing import DisenRouteFunction

    st = structure(name, dev)
    gen = torch.Generator(device=dev).manual_seed(7)
    q0, c0 = unit_channels(st.n_rows, K, d, dev, gen), unit_channels(st.n_rows, K, d, dev, gen)
    r = torch.randn(st.n_rows, K * d, device=dev, generator=gen)

    def grads(fn, dtype):
        q, c = q0.clone().to(dtype).requires_grad_(True), c0.clone().to(dtype).requires_grad_(True)
        (fn(q, c) * r.to(dtype)).sum().backward()
        return q.grad, c.grad

    for tau in (0.5, 1.0):
        got = grads(lambda q, c: DisenRouteFunction.apply(st, q, c, K, tau), torch.float32)
        want = grads(lambda q, c: route_step_fp64(st.rowptr, st.colind, q, c, K, tau), torch.float64)
        assert row_err(got[0], want[0]) <= 1e-4, ("dq", tau)
        assert row_err(got[1], want[1]) <= 1e-4, ("dc", tau)


@pytest.mark.parametrize("K,d", [(16, 4), (8, 8), (4, 16)])
@pytest.mark.parametrize("name", ["ragged", "hub", "two_hubs"])
def test_layer_chain_gradients_match_fp64_autograd(dev, name, K, d):
    """T = 7 steps behind h = leaky_relu(x W + b): gradients of x, W and b.  d = 2 is left to the one-step test: over
    seven steps two-dimensional channels pass near |u| = 0 often enough that the plain fp32 torch restatement's own
    gradients are 4e-4 to 2e-3 from fp64 (measured), so that chain says nothing about the kernels."""
    from cogdl_b200 import disen_routing

    st = structure(name, dev)
    gen = torch.Generator(device=dev).manual_seed(9)
    x0 = torch.randn(st.n_rows, 24, device=dev, generator=gen)
    W0 = 0.3 * torch.randn(24, K * d, device=dev, generator=gen)
    b0 = 0.1 * torch.randn(K * d, device=dev, generator=gen)
    r = torch.randn(st.n_rows, K * d, device=dev, generator=gen)

    def grads(route, dtype):
        x, W, b = (t.clone().to(dtype).requires_grad_(True) for t in (x0, W0, b0))
        h = torch.nn.functional.leaky_relu(x @ W + b)
        (route(h) * r.to(dtype)).sum().backward()
        return x.grad, W.grad, b.grad

    got = grads(lambda h: disen_routing(st, h, K, 7, 1.0), torch.float32)
    want = grads(lambda h: disen_routing_fp64(st.rowptr, st.colind, h, K, 7, 1.0), torch.float64)
    for name_, g, w in zip(("x", "W", "b"), got, want):
        assert row_err(g, w) <= 1e-4, name_


@pytest.mark.parametrize("name", ["hub", "two_hubs"])
def test_forward_backward_bitwise_reproducible(dev, name):
    from cogdl_b200 import disen_routing

    st = structure(name, dev, 16)
    gen = torch.Generator(device=dev).manual_seed(5)
    h0 = torch.randn(st.n_rows, 64, device=dev, generator=gen)
    r = torch.randn(st.n_rows, 64, device=dev, generator=gen)

    def once(K):
        h = h0.clone().requires_grad_(True)
        out = disen_routing(st, h, K, 7, 1.0)
        (out * r).sum().backward()
        return out.detach(), h.grad

    for K in (16, 8, 32):                       # d = 4, 8 (float4 lanes) and 2 (scalar lanes)
        first, second = once(K), once(K)
        assert all(torch.equal(u, v) for u, v in zip(first, second)), K


def test_kernel_notes(dev):
    from cogdl_b200 import _cabi, disen_routing

    st = structure("hub", dev)
    h = torch.randn(st.n_rows, 64, device=dev, requires_grad=True)
    with torch.no_grad():
        disen_routing(st, h, 16, 1, 1.0)
    assert _cabi.last_kernel() == "cogdl_b200::disen_route_fwd_kernel<float4,GROUP=16>"
    # autograd runs the backward on its own thread, and the note is per thread: call the backward here
    from cogdl_b200.operators._raw import disen_route_bwd_raw, disen_route_fwd_raw

    c = h.detach()
    out, lse2, r = disen_route_fwd_raw(st, c, c, 16, 1.0, want_saved=True)
    disen_route_bwd_raw(st, c, c, 16, 1.0, torch.ones_like(out), out, lse2, r)
    assert _cabi.last_kernel() == ("cogdl_b200::disen_route_bwd_row_kernel<float4,GROUP=16> + "
                                   "cogdl_b200::disen_route_bwd_col_kernel<float4,GROUP=16>")
    with torch.no_grad():
        disen_routing(st, h[:, :16].contiguous(), 8, 1, 1.0)
    assert _cabi.last_kernel() == "cogdl_b200::disen_route_fwd_kernel<float,GROUP=16>"
    with torch.no_grad():
        disen_routing(st, torch.randn(st.n_rows, 512, device=dev), 16, 1, 1.0)
    assert _cabi.last_kernel() == "cogdl_b200::disen_route_fwd_kernel<float4,GROUP=32>"


def test_errors(dev):
    from cogdl_b200 import disen_routing

    st = structure("tiny", dev)
    h = torch.randn(st.n_rows, 32, device=dev)
    with pytest.raises(RuntimeError, match="CUDA"):
        disen_routing(st, h.cpu(), 8, 1, 1.0)
    with pytest.raises(TypeError):
        disen_routing(st, h.half(), 8, 1, 1.0)
    rect = structure("rect", dev)
    with pytest.raises(RuntimeError, match="square"):
        disen_routing(rect, torch.randn(rect.n_rows, 32, device=dev), 8, 1, 1.0)
    with pytest.raises(RuntimeError, match="d=3 is not supported"):
        disen_routing(st, torch.randn(st.n_rows, 24, device=dev), 8, 1, 1.0)
    with pytest.raises(RuntimeError, match="tau"):
        disen_routing(st, h, 8, 1, 0.0)
    with pytest.raises(ValueError):
        disen_routing(st, h, 5, 1, 1.0)


@pytest.mark.parametrize("K", [16, 8])
def test_full_arxiv_shape(dev, K):
    """The whole arxiv-shaped graph (no self loops) at F = 64, T = 7, against fp64 evaluated on the GPU."""
    from cogdl_b200 import disen_routing, synth
    from cogdl_b200.structure import CSRStructure

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, device=dev, self_loops=False)
    st = CSRStructure.from_int64(rp, col)
    h = torch.randn(n, 64, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    got = disen_routing(st, h, K, 7, 1.0)
    assert route_err(got, *disen_routing_fp64(st.rowptr, st.colind, h, K, 7, 1.0, with_norm=True)) <= 1e-5


def test_reference_disengcn_through_install():
    """The reference DisenGCN (K = [16, 8], hidden 64, 7 iterations) through install(disengcn=True), in a child
    process (tests/disengcn_refpkg_check.py): logits vs the reference CPU run and fp64, gradients vs fp64."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.disengcn_refpkg_check"], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["untouched_without_flag"], "install() without disengcn=True must leave DisenGCNLayer.forward alone"
    assert res["rebound"] and res["patched"][-1] == "cogdl.layers.disengcn_layer.DisenGCNLayer.forward"
    assert res["logits_vs_ref_cpu"] <= 1e-4, res
    assert res["logits_vs_fp64"] <= 1e-4, res
    assert res["grads_present"], res
    assert max(res["grad_errs"].values()) <= 1e-4, res
    assert res["misses_per_step"][0] >= 1 and res["misses_per_step"][1:] == [0, 0], res
    assert res["uncovered_ran_original"] == ["cpu", "d3"], res
    assert res["restored"], res

"""CompGCN composition aggregation (cogdl_b200/csrc/comp_aggr.cu), CompAggrFunction and compgcn_aggregate against the
fp64 restatement of tests/compgcn_ref.py (itself pinned to the reference CompGCNLayer by test_cpu_compgcn_golden.py)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import graphs
from tests.compgcn_ref import compgcn_aggregate_fp64
from tests.gpu_util import dev, misaligned, row_err

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HUBS = ["hub", "two_hubs"]


def abs_problem(opn, x, rel):
    """(|x|, r) such that every term phi(|x|, r) is |phi| summed without cancellation: r = |rel| for mult, -|rel| for
    sub."""
    ra = rel.double().abs()
    return x.double().abs(), (ra if opn == "mult" else -ra)


def typed_coo(name, T, dev, seed=0):
    """A test graph as CompGCN's typed COO: the CSR's edges with random types in [0, T), shuffled so neither half
    is a CSR prefix.  N covers the rows and the columns.  Returns (row, col, type, N)."""
    rp, ci, n_cols = graphs.case(name)
    n = rp.size - 1
    rng = np.random.default_rng(seed + 7)
    row = np.repeat(np.arange(n), np.diff(rp))
    perm = rng.permutation(row.size)
    typ = rng.integers(0, T, row.size)
    to = lambda a: torch.from_numpy(np.ascontiguousarray(a).astype(np.int64)).to(dev)  # noqa: E731
    return to(row[perm]), to(ci[perm]), to(typ), max(n, n_cols)


@pytest.mark.parametrize("chunk", [None, 16])
@pytest.mark.parametrize("opn", ["sub", "mult"])
@pytest.mark.parametrize("T", [1, 3, 475])
@pytest.mark.parametrize("F", [1, 7, 16, 100, 128, 256])
@pytest.mark.parametrize("name", list(graphs.CASES))
def test_forward_matches_fp64(dev, name, F, T, opn, chunk):
    from cogdl_b200 import compgcn_aggregate

    row, col, typ, N = typed_coo(name, T, dev)
    gen = torch.Generator(device=dev).manual_seed(F * 1000 + T)
    x = torch.randn(N, F, device=dev, generator=gen)
    rel = torch.randn(T, F, device=dev, generator=gen)
    a_in, a_out = compgcn_aggregate((row, col), typ, x, rel, opn, chunk_edges=chunk)
    w_in, w_out = compgcn_aggregate_fp64(row, col, typ, x, rel, opn)
    b_in, b_out = compgcn_aggregate_fp64(row, col, typ, *abs_problem(opn, x, rel), opn)
    assert a_in.shape == a_out.shape == (N, F)
    assert row_err(a_in, w_in, b_in) <= 1e-5 and row_err(a_out, w_out, b_out) <= 1e-5


@pytest.mark.parametrize("opn", ["sub", "mult"])
@pytest.mark.parametrize("F", [7, 16, 100, 256])
@pytest.mark.parametrize("name", HUBS + ["ragged"])
def test_misaligned_inputs(dev, name, F, opn):
    from cogdl_b200 import compgcn_aggregate

    row, col, typ, N = typed_coo(name, 5, dev)
    gen = torch.Generator(device=dev).manual_seed(F)
    x = misaligned(torch.randn(N, F, device=dev, generator=gen))
    rel = misaligned(torch.randn(5, F, device=dev, generator=gen))
    a_in, a_out = compgcn_aggregate((row, col), typ, x, rel, opn, chunk_edges=16)
    w_in, w_out = compgcn_aggregate_fp64(row, col, typ, x, rel, opn)
    b_in, b_out = compgcn_aggregate_fp64(row, col, typ, *abs_problem(opn, x, rel), opn)
    assert row_err(a_in, w_in, b_in) <= 1e-5 and row_err(a_out, w_out, b_out) <= 1e-5


def _grads(aggregate, x0, rel0, G):
    """(dx, drel) of sum(agg_in * G[0] + agg_out * G[1]) with (agg_in, agg_out) = aggregate(x, rel)."""
    x, rel = x0.clone().requires_grad_(True), rel0.clone().requires_grad_(True)
    a_in, a_out = aggregate(x, rel)
    ((a_in * G[0]).sum() + (a_out * G[1]).sum()).backward()
    return x.grad, rel.grad


@pytest.mark.parametrize("chunk", [None, 16])
@pytest.mark.parametrize("opn", ["sub", "mult"])
@pytest.mark.parametrize("F", [7, 100, 128])
@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "two_hubs", "rect"])
def test_gradients_match_fp64_autograd(dev, name, F, opn, chunk):
    """T = 3 on the hub graphs: every type has ~1000-2700 edges, so its dR' row spans many hub chunks."""
    from cogdl_b200 import compgcn_aggregate
    from cogdl_b200.structure import DEFAULT_CHUNK_EDGES

    row, col, typ, N = typed_coo(name, 3, dev)
    gen = torch.Generator(device=dev).manual_seed(F + 1)
    x = torch.randn(N, F, device=dev, generator=gen)
    rel = torch.randn(3, F, device=dev, generator=gen)
    G = torch.randn(2, N, F, device=dev, generator=gen)
    dx, drel = _grads(lambda a, b: compgcn_aggregate((row, col), typ, a, b, opn, chunk_edges=chunk), x, rel, G)
    fp64 = lambda a, b: compgcn_aggregate_fp64(row, col, typ, a, b, opn)  # noqa: E731
    ex, erel = _grads(fp64, x.double(), rel.double(), G.double())
    bx, brel = _grads(fp64, *abs_problem(opn, x, rel), G.double().abs())
    assert row_err(dx, ex, bx) <= 1e-5
    assert row_err(drel, erel, brel) <= 1e-5
    if name in HUBS:
        assert int(torch.bincount(typ).min()) > 10 * (chunk or DEFAULT_CHUNK_EDGES)


@pytest.mark.parametrize("opn", ["sub", "mult"])
@pytest.mark.parametrize("name", HUBS)
def test_forward_backward_bitwise_reproducible(dev, name, opn):
    from cogdl_b200 import compgcn_aggregate
    from cogdl_b200.structure import clear_structure_cache

    row, col, typ, N = typed_coo(name, 3, dev)
    gen = torch.Generator(device=dev).manual_seed(3)
    x, rel = torch.randn(N, 100, device=dev, generator=gen), torch.randn(3, 100, device=dev, generator=gen)
    G = torch.randn(2, N, 100, device=dev, generator=gen)
    runs = []
    for _ in range(2):
        clear_structure_cache()      # the second run builds its structures afresh too
        xx, rr = x.clone().requires_grad_(True), rel.clone().requires_grad_(True)
        a_in, a_out = compgcn_aggregate((row, col), typ, xx, rr, opn, chunk_edges=16)
        ((a_in * G[0]).sum() + (a_out * G[1]).sum()).backward()
        runs.append((a_in.detach(), a_out.detach(), xx.grad, rr.grad))
    for a, b in zip(*runs):
        assert torch.equal(a, b)


def test_inputs_untouched_and_cpu_types(dev):
    """The edge tensors are neither reordered nor written; host edge types give the same result."""
    from cogdl_b200 import compgcn_aggregate

    row, col, typ, N = typed_coo("two_hubs", 4, dev)
    saved = [t.clone() for t in (row, col, typ)]
    versions = [t._version for t in (row, col, typ)]
    x = torch.randn(N, 32, device=dev)
    rel = torch.randn(4, 32, device=dev)
    a = compgcn_aggregate((row, col), typ, x, rel, "mult")
    b = compgcn_aggregate((row, col), typ.cpu(), x, rel, "mult")
    for t, s, v in zip((row, col, typ), saved, versions):
        assert torch.equal(t, s) and t._version == v
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])


def test_structure_cached_per_graph(dev):
    from cogdl_b200 import compgcn_aggregate
    from cogdl_b200.structure import comp_cache_stats

    row, col, typ, N = typed_coo("ragged", 3, dev)
    x, rel = torch.randn(N, 8, device=dev), torch.randn(3, 8, device=dev)
    before = dict(comp_cache_stats)
    for _ in range(3):
        compgcn_aggregate((row, col), typ, x, rel, "sub")
    assert comp_cache_stats["miss"] - before["miss"] == 1
    assert comp_cache_stats["hit"] - before["hit"] == 2
    typ.add_(0)                      # an in-place write bumps the version: rebuilt
    compgcn_aggregate((row, col), typ, x, rel, "sub")
    assert comp_cache_stats["miss"] - before["miss"] == 2


@pytest.mark.parametrize("E", [0, 1])
def test_empty_half_gives_zeros(dev, E):
    from cogdl_b200 import compgcn_aggregate

    N = 6
    row = torch.tensor([2, 3][:E], dtype=torch.int64, device=dev)
    col = torch.tensor([4, 1][:E], dtype=torch.int64, device=dev)
    typ = torch.tensor([1, 0][:E], dtype=torch.int64, device=dev)
    x = torch.randn(N, 5, device=dev, requires_grad=True)
    rel = torch.randn(2, 5, device=dev, requires_grad=True)
    a_in, a_out = compgcn_aggregate((row, col), typ, x, rel, "mult")
    assert torch.equal(a_in, torch.zeros_like(a_in))
    w_in, w_out = compgcn_aggregate_fp64(row, col, typ, x, rel, "mult")
    assert row_err(a_out, w_out) <= 1e-6
    (a_in.sum() + a_out.sum()).backward()
    assert x.grad.shape == x.shape and rel.grad.shape == rel.shape


def test_errors_raise_before_launch(dev):
    from cogdl_b200 import _cabi, compgcn_aggregate

    lib = _cabi.load()
    row, col, typ, N = typed_coo("tiny", 3, dev)
    x, rel = torch.randn(N, 8, device=dev), torch.randn(3, 8, device=dev)
    compgcn_aggregate((row, col), typ, x, rel, "sub")      # builds and caches the structure of (row, col, typ)
    torch.cuda.synchronize()
    n0 = lib.cogdl_b200_launch_count()
    with pytest.raises(ValueError, match="edge type"):
        compgcn_aggregate((row, col), typ, x, rel[:2], "sub")              # type 2 >= T = 2
    with pytest.raises(ValueError, match="out of range"):
        compgcn_aggregate((row, col.clone().fill_(N)), typ, x, rel, "sub")  # col == N
    with pytest.raises(ValueError, match="out of range"):
        compgcn_aggregate((row.clone().fill_(-1), col), typ, x, rel, "sub")
    with pytest.raises(ValueError, match="negative"):
        compgcn_aggregate((row, col), typ.clone().fill_(-1), x, rel, "sub")
    with pytest.raises(ValueError, match="opn"):
        compgcn_aggregate((row, col), typ, x, rel, "corr")
    with pytest.raises(TypeError):
        compgcn_aggregate((row, col), typ, x.double(), rel, "sub")
    with pytest.raises(RuntimeError, match="CUDA"):
        compgcn_aggregate((row.cpu(), col.cpu()), typ.cpu(), x.cpu(), rel.cpu(), "sub")
    assert lib.cogdl_b200_launch_count() == n0
    # the C entry point's own checks
    from cogdl_b200.operators._raw import _scratch
    from cogdl_b200.structure import CompStructure, _ptr, _stream

    # the type-grouped structure of the hub graph: its 3 rows are all hubs, so its plan has no segments and only
    # fits a 3-row call
    row, col, typ, N = typed_coo("hub", 3, dev)
    x = torch.randn(N, 8, device=dev)
    st, tcol, tw = CompStructure(row, col, typ, N).by_type(3)
    assert st.plan.n_hub_rows == 3 and st.plan.n_segs == 0
    plan, keep = st.plan_struct(_scratch("comp_aggr", st, 8))
    g = torch.empty(2 * N, 8, device=dev)
    y = torch.empty(4, 8, device=dev)
    n0 = lib.cogdl_b200_launch_count()
    for op, F, n_rows, msg in ((7, 8, 3, b"unknown op"), (0, 0, 3, b"F must be"), (0, 8, 4, b"does not match")):
        assert lib.cogdl_b200_comp_aggr_f32(_ptr(st.rowptr), _ptr(st.colind), _ptr(tcol), _ptr(tw), _ptr(g), 2 * N,
                                            _ptr(x), N, _ptr(y), n_rows, F, op, plan, _stream(dev)) != 0
        assert msg in lib.cogdl_b200_last_error()
    assert lib.cogdl_b200_launch_count() == n0
    del keep


def test_kernel_notes(dev):
    from cogdl_b200 import _cabi, compgcn_aggregate
    from cogdl_b200.operators._raw import comp_aggr_raw

    row, col, typ, N = typed_coo("hub", 3, dev)
    x, rel = torch.randn(N, 100, device=dev), torch.randn(3, 100, device=dev)
    compgcn_aggregate((row, col), typ, x, rel, "mult")
    assert _cabi.last_kernel() == ("cogdl_b200::stream_kernel<float4,NV=1,comp_mult,SRC_ONE,U=4,MINB=1,prefetch> "
                                   "block=128")
    compgcn_aggregate((row, col), typ, torch.randn(N, 7, device=dev), torch.randn(3, 7, device=dev), "sub")
    assert _cabi.last_kernel() == "cogdl_b200::stream_kernel<float,NV=1,comp_sub,SRC_ONE,U=4,MINB=1,prefetch> block=128"
    # the backward passes, called on this thread (autograd runs backward on its own)
    from cogdl_b200.structure import comp_structure_for

    cs = comp_structure_for(row, col, typ, N)
    t, ttype, tw = cs.transpose()
    comp_aggr_raw(t, ttype, tw, torch.randn(2 * N, 256, device=dev), rel.new_ones(3, 256), "mult")
    assert _cabi.last_kernel() == ("cogdl_b200::stream_kernel<float4,NV=2,comp_mult,SRC_ONE,U=2,MINB=1,prefetch> "
                                   "block=128")
    st, tcol, tw = cs.by_type(3)
    comp_aggr_raw(st, None, tw, torch.randn(2 * N, 100, device=dev), None, "copy")
    assert _cabi.last_kernel() == ("cogdl_b200::stream_kernel<float4,NV=1,weighted,SRC_ONE,U=4,MINB=1,prefetch> "
                                   "block=128")


def test_reference_compgcn_through_install():
    """The reference LinkPredictCompGCN through install(compgcn=True), in a child process
    (tests/compgcn_refpkg_check.py): predict() and loss() vs the reference CPU run, gradients vs fp64, dropout masks,
    structure reuse, uncovered cases and uninstall."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.compgcn_refpkg_check"], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["untouched_without_flag"], "install() without compgcn=True must leave CompGCNLayer.forward alone"
    assert res["rebound"] and res["patched"][-1] == "cogdl.models.nn.compgcn.CompGCNLayer.forward"
    assert res["predict_vs_ref_cpu"] <= 1e-4, res
    assert res["loss_vs_ref_cpu"] <= 1e-4, res
    assert res["grads_present"], res
    assert max(res["grad_errs"].values()) <= 1e-4, res
    assert max(res["zero_grads_vs_scale"].values()) <= 1e-5, res
    assert res["node_vs_fp64"] <= 1e-4, res
    # the original GPU forward sums with float atomics; a different mask would differ by O(1)
    assert res["dropout_fused_vs_original_gpu"] <= 1e-4, res
    assert res["graph_untouched"], res
    assert res["structures_built_2layer"] == 1 and res["structures_rebuilt_on_repeat"] == 0, res
    assert res["uncovered_ran_original"] == ["cpu", "corr"], res
    assert res["restored"], res

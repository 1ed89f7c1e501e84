"""cogdl_b200_spmm_residual_f32 and cogdl_b200.spmm_residual, one row of tests/spmm_residual_table.py each.

- Forward: bit-identical to this package's SpMM followed by the unfused torch sequence `a * (r * y) + b * z` on the
  same device (same plan, same panel count), and the call records exactly the kernel the row names.
- Gradients of x, z and the edge values (SpmmResidualFunction, backward over the cached transpose) per element within
  1e-5 * max(|ref|, the largest |ref| of its row, the sum of its terms' magnitudes) of fp64: an fp32 sum of terms that
  cancel is off by a few ulp of its largest terms, not of its result.
- Every row with hub chunks leaves the plan's arrival counters at zero.
- Y overlapping X, Z or the row scale is rejected with EINVAL.
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.gpu_util import bits, dev, misaligned, plan_structure
from tests.graphs import boundary_csr, case
from tests.spmm_residual_table import TABLE

pytestmark = pytest.mark.gpu

A_COEF, B_COEF = 0.9, 0.1       # (1 - alpha, alpha) of alpha = 0.1: 0.9 is not an fp32 value, so the rounding shows


def graph_of(c):
    return boundary_csr(c.chunk) if c.graph == "bounds" else case(c.graph)


def inputs(c, dev):
    rp, ci, n_cols = graph_of(c)
    n = rp.shape[0] - 1
    rng = np.random.default_rng(300 + c.F)
    X = torch.from_numpy(rng.standard_normal((n_cols, c.F)).astype(np.float32)).to(dev)
    Z = torch.from_numpy(rng.standard_normal((n, c.F)).astype(np.float32)).to(dev) if c.z else None
    r = torch.from_numpy(rng.random(n).astype(np.float32) + 0.25).to(dev) if c.row_scale else None
    val = torch.from_numpy(rng.random(ci.shape[0]).astype(np.float32)).to(dev) if c.weighted else None
    if not c.aligned:
        X = misaligned(X)
    return rp, ci, n_cols, X, Z, r, val


@pytest.mark.parametrize("c", TABLE, ids=lambda c: c.id)
def test_forward_is_the_unfused_sequence_bit_for_bit(dev, c):
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import spmm_raw, spmm_residual_raw

    rp, ci, n_cols, X, Z, r, val = inputs(c, dev)
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    y = spmm_residual_raw(st, val, X, Z, A_COEF, B_COEF, r, panels=c.panels)
    assert _cabi.last_kernel() == c.kernel, f"{c.id}: launched {_cabi.last_kernel()!r}"
    t = spmm_raw(st, val, X, panels=c.panels)
    if r is not None:
        t = r.view(-1, 1) * t
    t = A_COEF * t
    if Z is not None:
        t = t + B_COEF * Z
    mism = (bits(y) != bits(t)).nonzero()
    assert mism.numel() == 0, f"{c.id}: {mism.shape[0]} elements differ from the unfused sequence, first at " \
                              f"{tuple(mism[0].tolist())}: {y[tuple(mism[0])].item()!r} vs {t[tuple(mism[0])].item()!r}"
    if st.chunk_edges > 0 and st.plan.n_chunks > 0:
        assert int(st.plan.counters.abs().sum()) == 0


def rel_close(got, ref, what, mag=None):
    got = got.detach().double().cpu().numpy()
    scale = np.maximum(np.abs(ref), np.abs(ref).max(axis=-1, keepdims=True) if ref.ndim == 2 else np.abs(ref))
    if mag is not None:
        scale = np.maximum(scale, mag)
    err = np.abs(got - ref)
    bad = np.argwhere(~(err <= 1e-5 * scale + 1e-30))
    assert bad.size == 0, f"{what}: {len(bad)} elements off, first at {tuple(bad[0])}: {got[tuple(bad[0])]!r} vs " \
                          f"{ref[tuple(bad[0])]!r}"


@pytest.mark.parametrize("c", TABLE, ids=lambda c: c.id)
def test_gradients_match_fp64(dev, c):
    from cogdl_b200.operators.spmm_residual import SpmmResidualFunction

    rp, ci, n_cols, X, Z, r, val = inputs(c, dev)
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    n = rp.shape[0] - 1
    x = X.detach().clone().requires_grad_(True)
    z = Z.detach().clone().requires_grad_(True) if Z is not None else None
    v = val.detach().clone().requires_grad_(True) if val is not None else None
    y = SpmmResidualFunction.apply(st, x, z, v, A_COEF, B_COEF, r, False)
    g = torch.from_numpy(np.random.default_rng(7 + c.F).standard_normal((n, c.F)).astype(np.float32)).to(dev)
    y.backward(g)
    g64 = g.double().cpu().numpy()
    r64 = np.ones(n) if r is None else r.double().cpu().numpy()
    gr = np.float64(np.float32(A_COEF)) * r64[:, None] * g64
    w64 = np.ones(ci.shape[0]) if val is None else val.double().cpu().numpy()
    A = sp.csr_matrix((w64, ci.copy(), rp.copy()), shape=(n, n_cols))
    rel_close(x.grad, A.T @ gr, f"{c.id} dx", abs(A).T @ np.abs(gr))
    if z is not None:
        rel_close(z.grad, np.float64(np.float32(B_COEF)) * g64, f"{c.id} dz")
    if v is not None:
        rows = np.repeat(np.arange(n), np.diff(rp))
        X64 = X.double().cpu().numpy()
        dv = np.einsum("ef,ef->e", gr[rows], X64[ci])
        got = v.grad.detach().double().cpu().numpy()
        scale = np.maximum(np.abs(dv), np.einsum("ef,ef->e", np.abs(gr[rows]), np.abs(X64[ci])))
        bad = np.argwhere(~(np.abs(got - dv) <= 1e-5 * scale + 1e-30))
        assert bad.size == 0, f"{c.id} dval: {len(bad)} off, first {bad[0]}"


def test_symmetric_backward_runs_over_the_matrix_itself(dev):
    """sym=True: d x = a * A (r * g), as SPMMFunction does for a graph flagged symmetric (the reference's APPNP flags
    its dropped-weight adjacency so)."""
    from cogdl_b200.operators.spmm_residual import SpmmResidualFunction
    from tests.spmm_residual_table import RCase

    c = RCase("two_hubs", 40, "", row_scale=True)
    rp, ci, n_cols, X, Z, r, val = inputs(c, dev)
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    x = X.detach().clone().requires_grad_(True)
    g = torch.randn(rp.shape[0] - 1, 40, device=dev)
    SpmmResidualFunction.apply(st, x, Z, val, A_COEF, B_COEF, r, True).backward(g)
    A = sp.csr_matrix((val.double().cpu().numpy(), ci.copy(), rp.copy()), shape=(n_cols, n_cols))
    gr = np.float64(np.float32(A_COEF)) * r.double().cpu().numpy()[:, None] * g.double().cpu().numpy()
    rel_close(x.grad, A @ gr, "sym dx", abs(A) @ np.abs(gr))


def test_aliased_output_is_rejected(dev):
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import _scratch
    from cogdl_b200.structure import _ptr, _stream

    rp, ci, n = boundary_csr(64)
    st = plan_structure(rp, ci, n, dev, chunk=64)
    X = torch.randn(n, 32, device=dev)
    Z = torch.randn(n, 32, device=dev)
    plan, keep = st.plan_struct(_scratch("spmm", st, 32))
    Xbig = torch.randn(2 * n, 32, device=dev)
    Y = torch.empty(n, 32, device=dev)
    # (Y, X, x_rows, Z, row_scale): Y is X; Y is Z; Y starts one row into X; Y ends inside Z; Y starts inside X at an
    # offset given by X's row count; row_scale lies inside Y
    for Ya, Xa, xr, Za, Ra in ((X, X, n, Z, None), (Z, X, n, Z, None), (X[1:], X, n, None, None),
                               (Z[3:], X, n, Z[:-3], None), (Xbig[n // 2:3 * n // 2], Xbig, 2 * n, None, None),
                               (Y, X, n, Z, Y.view(-1)[7:7 + n])):
        with pytest.raises(_cabi.CogdlB200Error) as e:
            _cabi.call("cogdl_b200_spmm_residual_f32", _ptr(st.rowptr), _ptr(st.colind), None, _ptr(Xa), xr, _ptr(Za),
                       0.5, 0.5, _ptr(Ra), _ptr(Ya), Ya.shape[0], 32, 0, plan, _stream(dev))
        assert e.value.code == _cabi.EINVAL
    del keep


def test_operator_matches_the_unfused_graph_api(dev):
    """cogdl_b200.spmm_residual on a Graph with in_norm / out_norm (sym_norm of a CSR-built graph) is bit-identical to
    a * cogdl_b200.spmm(graph, x) + b * z; CPU input raises."""
    import cogdl_b200
    from cogdl_b200 import synth

    rp, col = synth.powerlaw_csr(3000, 40000, seed=3)
    g = cogdl_b200.Graph(row_ptr=rp, col=col).to(dev)
    g.sym_norm()
    assert g.in_norm is not None and g.out_norm is not None
    x, z = torch.randn(3000, 64, device=dev), torch.randn(3000, 64, device=dev)
    got = cogdl_b200.spmm_residual(g, x, z, 1 - 0.1, 0.1)
    want = (1 - 0.1) * cogdl_b200.spmm(g, x) + 0.1 * z
    assert torch.equal(bits(got), bits(want))
    with pytest.raises(RuntimeError):
        cogdl_b200.spmm_residual(g, x.cpu(), z.cpu(), 0.9, 0.1)

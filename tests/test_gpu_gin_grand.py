"""cogdl_b200_spmm_residual_dcoef_f32 / gin_aggregate (GIN) and cogdl_b200_spmm_accum_f32 / random_propagate (GRAND).

- Each row of tests/gin_grand_table.py: bit-identical to this package's SpMM followed by the unfused torch sequence on
  the same device (same plan, same panel count) -- `a * (r * y) + b_dev * z` for the device coefficient, `acc_in + r * y`
  and `div_(order + 1.0)` on the last hop for the accumulation -- records exactly the kernel the row names, and is within
  the suite's (k + 2 + m) 2^-24 sum|terms| bound of fp64.
- gin_aggregate: the output and d x bit-identical to autograd through `(1 + eps) * x + cogdl_b200.spmm(graph, x)`; d eps
  and d val within the fp64 bound.  eps trainable, fixed and -1; graphs symmetric or not, with and without in_norm /
  out_norm, on every square test graph (the boundary-degree graph under a 64-edge hub plan, empty rows); inputs
  contiguous, strided and misaligned.
- random_propagate: bit-identical to the reference loop on this package's spmm for order in {0, 1, 2, 8}.
- Neither call synchronises with the host.
- The reference GIN, GINE and Grand through install(gin=True, grand=True), in a child process
  (tests/gin_grand_refpkg_check.py).
"""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.gin_grand_table import TABLE
from tests.gpu_util import bits, dev, misaligned, plan_structure
from tests.graphs import boundary_csr, case
from tests.test_gpu_autograd import (GraphCase, MODES, SQUARE, bound, incoming, place, same_bits, sum_ref, within)

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
A_COEF, B_COEF, ORDER = 0.8, 1.3, 8
ORDERS = (0, 1, 2, 8)


def row_inputs(c, dev):
    rp, ci, n_cols = boundary_csr(c.chunk) if c.graph == "bounds" else case(c.graph)
    n = rp.shape[0] - 1
    rng = np.random.default_rng(700 + c.F)
    f32 = lambda *s: torch.from_numpy(rng.standard_normal(s).astype(np.float32)).to(dev)  # noqa: E731
    X = f32(n_cols, c.F)
    Z = f32(n, c.F) if c.z else None
    r = torch.from_numpy(rng.random(n).astype(np.float32) + 0.25).to(dev) if c.row_scale else None
    val = torch.from_numpy(rng.random(ci.shape[0]).astype(np.float32)).to(dev) if c.weighted else None
    if not c.aligned:
        X = misaligned(X)
    return rp, ci, n_cols, n, X, Z, r, val


def check_bits(c, y, t):
    mism = (bits(y) != bits(t)).nonzero()
    assert mism.numel() == 0, f"{c.id}: {mism.shape[0]} elements differ from the unfused sequence, first at " \
                              f"{tuple(mism[0].tolist())}: {y[tuple(mism[0])].item()!r} vs {t[tuple(mism[0])].item()!r}"


def check_fp64(c, got, ref, mag, k, m):
    got = got.double().cpu().numpy()
    bnd = bound(k, mag, m)
    bad = np.argwhere(~(np.abs(got - ref) <= bnd))
    assert bad.size == 0, f"{c.id}: {len(bad)} elements off fp64, first at {tuple(bad[0])}"


@pytest.mark.parametrize("c", TABLE, ids=lambda c: c.id)
def test_row_is_the_unfused_sequence_bit_for_bit_and_near_fp64(dev, c):
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import spmm_accum_raw, spmm_raw, spmm_residual_dcoef_raw
    from cogdl_b200.operators.grand import div_scale

    rp, ci, n_cols, n, X, Z, r, val = row_inputs(c, dev)
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    t = spmm_raw(st, val, X, panels=c.panels)
    if r is not None:
        t = r.view(-1, 1) * t
    w64 = np.ones(ci.shape[0]) if val is None else val.double().cpu().numpy()
    A = sp.csr_matrix((w64, ci.copy(), rp.copy()), shape=(n, n_cols))
    X64 = X.double().cpu().numpy()
    r64 = np.ones((n, 1)) if r is None else r.double().cpu().numpy()[:, None]
    k = np.diff(rp)[:, None]
    if c.epi == "dcoef":
        b_dev = torch.full((1,), B_COEF, dtype=torch.float32, device=dev)
        y = spmm_residual_dcoef_raw(st, val, X, Z, A_COEF, b_dev, r, panels=c.panels)
        assert _cabi.last_kernel() == c.kernel, f"{c.id}: launched {_cabi.last_kernel()!r}"
        t = A_COEF * t
        if Z is not None:
            t = t + b_dev * Z
        check_bits(c, y, t)
        a64, b64 = float(np.float32(A_COEF)), float(np.float32(B_COEF))
        ref, mag = a64 * r64 * (A @ X64), a64 * r64 * (abs(A) @ np.abs(X64))
        if Z is not None:
            Z64 = Z.double().cpu().numpy()
            ref, mag = ref + b64 * Z64, mag + np.abs(b64 * Z64)
        check_fp64(c, y, ref, mag, k + 1, 3)
    else:
        S = torch.from_numpy(np.random.default_rng(800 + c.F).standard_normal((n, c.F)).astype(np.float32)).to(dev)
        acc = S.clone() if c.in_place else torch.empty_like(S)
        xn = spmm_accum_raw(st, val, X, acc, None if c.in_place else S, r, c.last, div_scale(ORDER), panels=c.panels)
        assert _cabi.last_kernel() == c.kernel, f"{c.id}: launched {_cabi.last_kernel()!r}"
        ref_acc = S.clone()
        ref_acc.add_(t)
        if c.last:
            ref_acc.div_(ORDER + 1.0)
            assert xn is None
        else:
            check_bits(c, xn, t)
        check_bits(c, acc, ref_acc)
        S64 = S.double().cpu().numpy()
        ref, mag = S64 + r64 * (A @ X64), np.abs(S64) + r64 * (abs(A) @ np.abs(X64))
        if c.last:
            ref, mag = ref / (ORDER + 1), mag / (ORDER + 1)
        check_fp64(c, acc, ref, mag, k + 1, 2 + int(c.last) + 1)   # + 1: the fp32 reciprocal's own rounding
    if st.chunk_edges > 0 and st.plan.n_chunks > 0:
        assert int(st.plan.counters.abs().sum()) == 0


def test_accum_entry_rejects_overlapping_outputs(dev):
    from cogdl_b200.operators._raw import spmm_accum_raw

    rp, ci, n_cols = case("two_hubs")
    st = plan_structure(rp, ci, n_cols, dev, chunk=64)
    n = rp.shape[0] - 1
    X = torch.randn(n, 16, device=dev)
    acc = torch.zeros(n, 16, device=dev)
    for kw in ({"xn": X}, {"xn": acc}):
        with pytest.raises(RuntimeError, match="overlaps"):
            spmm_accum_raw(st, None, X, acc, **kw)
    with pytest.raises(RuntimeError, match="ACC overlaps X"):
        spmm_accum_raw(st, None, X, X, last=True)
    for bad in (torch.empty(n, 8, device=dev), torch.empty(n, 32, device=dev)[:, ::2],
                torch.empty(n, 16, device=dev, dtype=torch.float64)):
        with pytest.raises(ValueError, match="xn must be"):
            spmm_accum_raw(st, None, X, acc, xn=bad)


def test_random_propagate_order_zero_is_detached(dev):
    import cogdl_b200

    c = GraphCase("two_hubs", "rowptr", "fixed", "sym", dev)
    x = torch.randn(c.n, 16, device=dev, requires_grad=True)
    got = cogdl_b200.random_propagate(c.g, x, 0)
    assert not got.requires_grad and got.data_ptr() == x.data_ptr()


GIN_EPS = {"train": (0.25, True, "leaf"), "fixed": (0.25, False, "none"), "minus1": (-1.0, False, "fixed")}


@pytest.mark.parametrize("name", SQUARE)
@pytest.mark.parametrize("build", ["rowptr", "shuffled"])
@pytest.mark.parametrize("norm", ["none", "sym", "row"])
@pytest.mark.parametrize("eps_kind", list(GIN_EPS))
def test_gin_aggregate_is_the_reference_expression(dev, name, build, norm, eps_kind):
    """Forward and d x bit-identical to autograd through `(1 + eps) * x + spmm(graph, x)` on this package's spmm (fp32
    addition commutes); d eps and d val within the fp64 bound."""
    import cogdl_b200

    eps0, train, weights = GIN_EPS[eps_kind]
    c = GraphCase(name, build, weights, norm, dev)
    gkind, xkind = MODES[(list(GIN_EPS).index(eps_kind) + ["none", "sym", "row"].index(norm)) % 3]
    rng = np.random.default_rng(90)
    X = rng.standard_normal((c.n, 24)).astype(np.float32)
    x = place(X, xkind, dev).requires_grad_(True)
    eps = torch.full((1,), eps0, dtype=torch.float32, device=dev).requires_grad_(train)
    inputs = [t for t in (x, eps, c.leaf) if t is not None and t.requires_grad]

    out = cogdl_b200.gin_aggregate(c.g, x, eps)
    ref_out = (1 + eps) * x + cogdl_b200.spmm(c.g, x)
    same_bits(out, ref_out, "forward")
    G, g64 = incoming(out, gkind, rng)
    grads = torch.autograd.grad(out, inputs, G, retain_graph=True)   # a COO graph shares its weight gather
    ref_grads = torch.autograd.grad(ref_out, inputs, G)
    same_bits(grads[0], ref_grads[0], "d x")

    b64 = float(np.float32(np.float32(1) + np.float32(eps0)))
    what = f"{name} {build} {norm} {eps_kind}"
    ref, mag, k = c.spmm_ref(X)
    bx = b64 * X.astype(np.float64)
    within(out.detach().cpu().numpy(), ref + bx, bound(k + 1, mag + np.abs(bx), c.m_out() + 1), what + " out")
    ref, mag, k = c.adjoint_ref(c.g_in(g64))
    bg = b64 * g64
    within(grads[0].cpu().numpy(), ref + bg, bound(k + 1, mag + np.abs(bg), c.m_adj() + 1), what + " d x")
    i = 1
    if train:
        t = g64 * X.astype(np.float64)
        within(grads[1].cpu().numpy(), np.array([t.sum()]), bound(t.size, np.array([np.abs(t).sum()])), what + " d eps")
        i += 1
    if weights == "leaf":
        ref, mag, m = c.leaf_ref(c.g_in(g64), X)
        within(grads[i].cpu().numpy(), ref, bound(24, mag, m), what + " d val")


def test_gin_aggregate_python_eps_and_unneeded_gradients(dev):
    import cogdl_b200
    from cogdl_b200.operators.gin import GinAggregateFunction

    c = GraphCase("two_hubs", "rowptr", "fixed", "none", dev)
    x = torch.randn(c.n, 16, device=dev)
    same_bits(cogdl_b200.gin_aggregate(c.g, x, 0.1), (1 + 0.1) * x + cogdl_b200.spmm(c.g, x), "python eps")
    st = c.g.structure()
    b = torch.full((1,), 1.5, device=dev, requires_grad=True)
    xr = x.clone().requires_grad_(True)
    out = GinAggregateFunction.apply(st, xr, None, b, c.g.raw_edge_weight, None, c.sym)
    (dx,) = torch.autograd.grad(out, [xr], torch.ones_like(out))
    assert dx is not None and b.grad is None


def reference_rand_prop(graph, x, order):
    """Grand.rand_prop after drop_node (cogdl/models/nn/grand.py:98-104) on this package's spmm."""
    import cogdl_b200

    y = x
    for _ in range(order):
        x = cogdl_b200.spmm(graph, x).detach_()
        y.add_(x)
    return y.div_(order + 1.0).detach_()


@pytest.mark.parametrize("order", ORDERS)
@pytest.mark.parametrize("name,norm,F", [("two_hubs", "sym", 40), ("ragged", "row", 128), ("bounds", "sym", 47),
                                         ("bounds", "none", 256)])
def test_random_propagate_is_the_reference_loop(dev, order, name, norm, F):
    import cogdl_b200

    c = GraphCase(name, "rowptr", "fixed", norm, dev)
    x = torch.from_numpy(np.random.default_rng(91).standard_normal((c.n, F)).astype(np.float32)).to(dev)
    got = cogdl_b200.random_propagate(c.g, x, order)
    kernel = cogdl_b200._cabi.last_kernel()
    ref = reference_rand_prop(c.g, x.clone(), order)
    if order == 0:
        assert got.data_ptr() == x.data_ptr() and not got.requires_grad
    else:   # the fused hop where it is measured to win (F <= 128, a multiple of 4), the SpMM + add_ loop elsewhere
        assert ("accum_kernel" in kernel) == (F <= 128 and F % 4 == 0), kernel
    same_bits(got, ref, f"{name} {norm} F={F} order={order}")


def test_no_host_synchronisation(dev):
    import cogdl_b200

    c = GraphCase("two_hubs", "rowptr", "leaf", "row", dev)   # row norm: not symmetric, the backward takes A^T
    x = torch.randn(c.n, 64, device=dev, requires_grad=True)
    eps = torch.zeros(1, device=dev, requires_grad=True)
    for _ in range(2):           # the first round builds the CSR, the hub plan and the transpose
        torch.cuda.set_sync_debug_mode("error" if _ else "default")
        try:
            out = cogdl_b200.gin_aggregate(c.g, x, eps)
            torch.autograd.grad(out, [x, eps, c.leaf], torch.ones_like(out))
            cogdl_b200.random_propagate(c.g, x.detach(), 8)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_reference_gin_and_grand_through_install():
    """GIN / GINE layers and the GIN model, and Grand.rand_prop / forward, through install(gin=True, grand=True): equal
    to the same reference code without the flags at the same seed, within 1e-5 of the golden file; the fallback cases
    and uninstall leave the originals in charge."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.gin_grand_refpkg_check"], cwd=ROOT, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["untouched_without_flag"] and res["rebound"] and res["restored"], res
    assert res["patched"] == ["cogdl.layers.gin_layer.GINLayer.forward", "cogdl.layers.gine_layer.GINELayer.forward",
                              "cogdl.models.nn.grand.Grand.rand_prop"], res
    assert res["bit_identical"] and all(res["bit_identical"].values()), res
    assert max(res["model_rel"].values()) <= 1e-5, res
    assert max(res["vs_golden"].values()) <= 1e-5, res
    assert all(res["fused_kernels"].values()), res
    assert all(res["fallbacks"].values()), res

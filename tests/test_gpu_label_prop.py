"""cogdl_b200_label_prop_f32 and cogdl_b200.label_propagate, one row of tests/label_prop_table.py each.

- Each row: bit-identical to this package's SpMM followed by the unfused torch sequence `a * (r * y) + b * z`,
  torch.clamp and the index_put of the pinned rows on the same device (same plan, same panel count), the call records
  exactly the kernel the row names, and the result is within 1e-5 * (the sum of its terms' magnitudes) of fp64.
- Edge cases: pinned rows equal Z bitwise (NaN and -0.0 included), NaN passes the clamp, -0.0 against lo = 0, lo > hi,
  empty rows, every row pinned and none.
- The loop: label_propagate is bit-identical to the unfused outcome_correlation loop on this package's spmm, for nprop
  in {0, 1, 50}, with the clamp, with the pinned rows and at alpha = 1 (b = 0).
"""
import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.gpu_util import bits, dev, misaligned, plan_structure
from tests.graphs import boundary_csr, case
from tests.label_prop_table import TABLE

pytestmark = pytest.mark.gpu

A_COEF, B_COEF = 0.8, 1 - 0.8   # alpha = 0.8 of the smooth phase, (1 - alpha) rounded in fp64 first, as Python does
CLAMP_LO, CLAMP_HI = -0.75, 0.5


def inputs(c, dev):
    rp, ci, n_cols = boundary_csr(c.chunk) if c.graph == "bounds" else case(c.graph)
    n = rp.shape[0] - 1
    rng = np.random.default_rng(500 + c.F)
    X = torch.from_numpy(rng.standard_normal((n_cols, c.F)).astype(np.float32)).to(dev)
    Z = torch.from_numpy(rng.standard_normal((n, c.F)).astype(np.float32)).to(dev) if c.z else None
    r = torch.from_numpy(rng.random(n).astype(np.float32) + 0.25).to(dev) if c.row_scale else None
    val = torch.from_numpy(rng.random(ci.shape[0]).astype(np.float32)).to(dev) if c.weighted else None
    nid = torch.from_numpy(np.flatnonzero(rng.random(n) < 0.35)).to(dev) if c.pin else None
    if not c.aligned:
        X = misaligned(X)
    return rp, ci, n_cols, X, Z, r, val, nid


def unfused(st, val, X, Z, r, a, b, clamp, nid, panels=0):
    """This package's spmm, then the reference's eager sequence one operation at a time."""
    from cogdl_b200.operators._raw import spmm_raw

    t = spmm_raw(st, val, X, panels=panels)
    if r is not None:
        t = r.view(-1, 1) * t
    t = a * t
    if Z is not None:
        t += b * Z
    if clamp is not None:
        t = torch.clamp(t, clamp[0], clamp[1])
    if nid is not None:
        t[nid] = Z[nid]
    return t


@pytest.mark.parametrize("c", TABLE, ids=lambda c: c.id)
def test_step_is_the_unfused_sequence_bit_for_bit_and_near_fp64(dev, c):
    from cogdl_b200 import _cabi
    from cogdl_b200.operators.label_prop import label_prop_raw, pin_mask

    rp, ci, n_cols, X, Z, r, val, nid = inputs(c, dev)
    st = plan_structure(rp, ci, n_cols, dev, c.plan, c.chunk)
    n = rp.shape[0] - 1
    clamp = (CLAMP_LO, CLAMP_HI) if c.clamp else None
    pin = pin_mask(n, nid, dev) if nid is not None else None
    y = label_prop_raw(st, val, X, Z, A_COEF, B_COEF, r, pin, clamp, panels=c.panels)
    assert _cabi.last_kernel() == c.kernel, f"{c.id}: launched {_cabi.last_kernel()!r}"
    t = unfused(st, val, X, Z, r, A_COEF, B_COEF, clamp, nid, c.panels)
    mism = (bits(y) != bits(t)).nonzero()
    assert mism.numel() == 0, f"{c.id}: {mism.shape[0]} elements differ from the unfused sequence, first at " \
                              f"{tuple(mism[0].tolist())}: {y[tuple(mism[0])].item()!r} vs {t[tuple(mism[0])].item()!r}"
    if st.chunk_edges > 0 and st.plan.n_chunks > 0:
        assert int(st.plan.counters.abs().sum()) == 0

    # fp64 restatement: the same formula with every operation exact, bounded by the magnitudes of its terms
    w64 = np.ones(ci.shape[0]) if val is None else val.double().cpu().numpy()
    A = sp.csr_matrix((w64, ci.copy(), rp.copy()), shape=(n, n_cols))
    X64 = X.double().cpu().numpy()
    r64 = np.ones(n) if r is None else r.double().cpu().numpy()
    a64, b64 = float(np.float32(A_COEF)), float(np.float32(B_COEF))
    ref = a64 * r64[:, None] * (A @ X64)
    mag = np.abs(a64) * r64[:, None] * (abs(A) @ np.abs(X64))
    if Z is not None:
        Z64 = Z.double().cpu().numpy()
        ref, mag = ref + b64 * Z64, mag + np.abs(b64 * Z64)
    if clamp is not None:
        ref = np.clip(ref, float(np.float32(clamp[0])), float(np.float32(clamp[1])))
    if nid is not None:
        ref[nid.cpu().numpy()] = Z64[nid.cpu().numpy()]
    got = y.double().cpu().numpy()
    bad = np.argwhere(~(np.abs(got - ref) <= 1e-5 * np.maximum(mag, np.abs(ref)) + 1e-30))
    assert bad.size == 0, f"{c.id}: {len(bad)} elements off fp64, first at {tuple(bad[0])}"


def special_inputs(dev, F=40, plan="default"):
    """A hub graph with empty rows, X and Z holding NaN, +-inf and -0.0."""
    rp, ci, n = case("two_hubs")
    st = plan_structure(rp, ci, n, dev, plan, 64)
    g = torch.Generator().manual_seed(11)
    X = torch.randn(n, F, generator=g)
    Z = torch.randn(n, F, generator=g)
    X[3, :5] = float("nan")
    X[7, 5:9] = float("inf")
    Z[:, 10:12] = -0.0
    Z[5, 12] = float("nan")
    return rp, ci, n, st, X.to(dev), Z.to(dev)


@pytest.mark.parametrize("F", [40, 47])
def test_edge_cases_match_torch(dev, F):
    from cogdl_b200.operators.label_prop import label_prop_raw, pin_mask

    rp, ci, n, st, X, Z = special_inputs(dev, F)
    empty = torch.from_numpy(np.flatnonzero(np.diff(rp) == 0)).to(dev)
    assert empty.numel() > 0
    hubs = torch.from_numpy(np.argsort(-np.diff(rp))[:2].copy()).to(dev)
    nid = torch.cat([hubs, empty[: empty.numel() // 2], torch.arange(0, n, 5, device=dev)])
    # a = -1 turns an empty row's zero sum into -0.0, and b * -0.0 adds -0.0 to it: -0.0 meets lo = 0
    for a, b, clamp in ((A_COEF, B_COEF, (0.0, 1.0)), (-1.0, 1.0, (0.0, 1.0)), (A_COEF, B_COEF, (0.5, -0.5)),
                        (A_COEF, B_COEF, (-1.0, 1.0)), (A_COEF, 0.0, None)):
        for pinned in (None, nid, torch.arange(n, device=dev), torch.zeros(0, dtype=torch.int64, device=dev)):
            pin = None if pinned is None else pin_mask(n, pinned, dev)
            y = label_prop_raw(st, None, X, Z, a, b, None, pin, clamp)
            t = unfused(st, None, X, Z, None, a, b, clamp, pinned)
            assert torch.equal(bits(y), bits(t)), (a, b, clamp, None if pinned is None else pinned.numel())
            if pinned is not None and pinned.numel() > 0:
                assert torch.equal(bits(y[pinned]), bits(Z[pinned]))
    pre = unfused(st, None, X, Z, None, -1.0, 1.0, None, None)
    assert bool(torch.isnan(pre).any()) and bool(((pre == 0) & torch.signbit(pre)).any())
    y = label_prop_raw(st, None, X, Z, A_COEF, B_COEF, None, None, (0.5, -0.5))
    assert bool(((y == -0.5) | torch.isnan(y)).all())
    assert torch.equal(torch.isnan(y), torch.isnan(unfused(st, None, X, Z, None, A_COEF, B_COEF, None, None)))


def test_rejects_aliasing_and_pins_without_z(dev):
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import _scratch
    from cogdl_b200.structure import _ptr, _stream

    rp, ci, n, st, X, Z = special_inputs(dev, 32)
    pin = torch.ones(n, dtype=torch.uint8, device=dev)
    Y = torch.empty_like(Z)
    plan, keep = st.plan_struct(_scratch("spmm", st, 32))
    for Ya, Za, P in ((X, Z, None), (Z, Z, None), (Y, None, pin)):
        with pytest.raises(_cabi.CogdlB200Error) as e:
            _cabi.call("cogdl_b200_label_prop_f32", _ptr(st.rowptr), _ptr(st.colind), None, _ptr(X), n, _ptr(Za), 0.5,
                       0.5, None, _ptr(P), 1, -1.0, 1.0, _ptr(Ya), n, 32, 0, plan, _stream(dev))
        assert e.value.code == _cabi.EINVAL
    del keep


def outcome_loop(graph, labels, alpha, nprop, post, alpha_term=True):
    """Correct & Smooth's propagation loop, one eager operation at a time, on this package's spmm."""
    import cogdl_b200

    out = labels.clone()
    for _ in range(nprop):
        out = alpha * cogdl_b200.spmm(graph, out)
        out += ((1 - alpha) if alpha_term else 1) * labels
        out = post(out)
    return out


@pytest.mark.parametrize("built", ["csr", "coo"])
@pytest.mark.parametrize("nprop", [0, 1, 50])
def test_label_propagate_is_the_reference_loop(dev, built, nprop):
    import cogdl_b200
    from cogdl_b200 import synth

    rp, col = synth.powerlaw_csr(4000, 60000, seed=5)
    if built == "csr":
        g = cogdl_b200.Graph(row_ptr=rp, col=col).to(dev)
    else:
        row = torch.repeat_interleave(torch.arange(4000), rp[1:] - rp[:-1])
        g = cogdl_b200.Graph(edge_index=(row, col)).to(dev)
    g.sym_norm()
    gen = torch.Generator().manual_seed(nprop)
    labels = torch.softmax(torch.randn(4000, 47, generator=gen), -1).to(dev)
    nid = torch.randperm(4000, generator=gen)[:1500].to(dev)
    with torch.no_grad():
        for alpha in (0.8, 1.0):
            for alpha_term in (True, False):
                def reset(x):
                    x[nid] = labels[nid]
                    return x

                cases = ((dict(lower=0, upper=1), lambda x: torch.clamp(x, 0, 1)),
                         (dict(lower=-1.0, upper=1.0), lambda x: torch.clamp(x, -1.0, 1.0)), (dict(pinned=nid), reset))
                for kw, post in cases:
                    got = cogdl_b200.label_propagate(g, labels, alpha, nprop, alpha_term=alpha_term, **kw)
                    want = outcome_loop(g, labels, alpha, nprop, post, alpha_term)
                    assert torch.equal(bits(got), bits(want)), (built, nprop, alpha, alpha_term, kw.keys())
                    assert got.data_ptr() != labels.data_ptr()


def test_label_propagate_rejects(dev):
    import cogdl_b200
    from cogdl_b200 import synth

    rp, col = synth.powerlaw_csr(500, 4000, seed=2)
    g = cogdl_b200.Graph(row_ptr=rp, col=col).to(dev)
    labels = torch.rand(500, 7, device=dev)
    with pytest.raises(RuntimeError):
        cogdl_b200.label_propagate(g, labels.cpu(), 0.5, 3)
    with pytest.raises(TypeError):
        cogdl_b200.label_propagate(g, labels.double(), 0.5, 3)
    with pytest.raises(RuntimeError):
        cogdl_b200.label_propagate(g, labels.clone().requires_grad_(True), 0.5, 3)
    with torch.no_grad():
        out = cogdl_b200.label_propagate(g, labels.clone().requires_grad_(True), 0.5, 3, lower=0, upper=1)
    assert out.shape == labels.shape

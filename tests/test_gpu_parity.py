"""GPU parity tests: every C-ABI op (through the Python operator layer) against the CPU oracle on
the same seeded inputs.  Bar (north star): integer outputs bit-exact; fp32 within 1e-5 relative.

`rel` below is max|a-b| / max|b| (error relative to the result's scale), the tolerance stated in
each test.  SpMM rows that are not split by the hub plan are additionally required to be
BIT-IDENTICAL to the oracle (= reference CPU spmm_cpu order: CSR order, separate mul and add).
"""
import numpy as np
import pytest
import torch

import oracle
from tests.gpu_util import T, dev, plan_structure, rel
from tests.graphs import CASES, case

pytestmark = pytest.mark.gpu

TOL = 1e-5


# ------------------------------------------------------------------------------------ SpMM
@pytest.mark.parametrize("name", list(CASES))
@pytest.mark.parametrize("F", [128, 16, 40, 7, 256, 1, 64, 33, 300, 9, 17, 65, 1433])
@pytest.mark.parametrize("weighted", [True, False])
def test_spmm_matches_oracle(dev, name, F, weighted):
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n_cols = case(name)
    rng = np.random.default_rng(1)
    X = rng.standard_normal((n_cols, F)).astype(np.float32)
    val = rng.random(ci.shape[0]).astype(np.float32) if weighted else None
    ref = oracle.spmm_csr(rp, ci, val, X)
    # chunk 0: no hub plan -> strictly sequential -> bit exact everywhere; seg_cost 0: a plan without segments, so
    # every width runs the row kernel with hub chunks
    for chunk, seg_cost in ((0, None), (256, None), (256, 0)):
        st = plan_structure(rp, ci, n_cols, dev, chunk=chunk, seg_cost=seg_cost)
        y = spmm_raw(st, None if val is None else T(val, dev), T(X, dev)).cpu().numpy()
        assert y.shape == ref.shape
        deg = np.diff(rp)
        unsplit = deg <= chunk if chunk else np.ones_like(deg, bool)
        assert np.array_equal(y[unsplit], ref[unsplit]), f"unsplit rows must be bit-identical (chunk={chunk})"
        assert rel(y, ref) <= TOL


def test_spmm_deterministic_with_hubs(dev):
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n_cols = case("hub")
    rng = np.random.default_rng(2)
    X, val = T(rng.standard_normal((n_cols, 128)).astype(np.float32), dev), T(rng.random(ci.shape[0]).astype(np.float32), dev)
    st = plan_structure(rp, ci, n_cols, dev)
    assert st.plan.n_hub_rows == 1 and st.plan.n_chunks == 6
    y0 = spmm_raw(st, val, X)
    for _ in range(5):
        assert torch.equal(spmm_raw(st, val, X), y0)
    assert int(st.plan.counters.abs().sum()) == 0  # arrival counters are left clean


def test_spmm_half(dev):
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n_cols = case("hub")
    rng = np.random.default_rng(3)
    X = rng.standard_normal((n_cols, 128)).astype(np.float16)
    val = rng.random(ci.shape[0]).astype(np.float16)
    ref = oracle.spmm_csr(rp, ci, val.astype(np.float32), X.astype(np.float32))
    st = plan_structure(rp, ci, n_cols, dev)
    y = spmm_raw(st, T(val, dev), T(X, dev))
    assert y.dtype == torch.float16
    # fp16 storage, fp32 accumulate: error budget = one fp16 rounding of the result
    assert rel(y.float().cpu().numpy(), ref) <= 2e-3


def test_spmm_two_source(dev):
    from cogdl_b200.operators._raw import spmm_2src_raw

    rp, ci, n_cols = case("rect")
    rng = np.random.default_rng(4)
    X = rng.standard_normal((n_cols, 128)).astype(np.float32)
    val = rng.random(ci.shape[0]).astype(np.float32)
    ref = oracle.spmm_csr(rp, ci, val, X)
    st = plan_structure(rp, ci, n_cols, dev)
    n0 = 123
    y = spmm_2src_raw(st, T(val, dev), T(X[:n0], dev), T(X[n0:], dev)).cpu().numpy()
    assert np.array_equal(y, ref)


@pytest.mark.parametrize("F", [128, 16, 40, 64, 8, 256])
def test_spmm_peer_form_single_gpu(dev, F):
    """The fused-gather kernel (cogdl_b200_spmm_csr_f32_peers) with the 'peers' being three separate
    buffers on this GPU: checks the (owner << shift | row) column decoding and the per-owner base
    pointers without needing NVLink (the multi-GPU run is tools/dist_gpu_check.py)."""
    import ctypes

    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import _scratch
    from cogdl_b200.structure import _ptr, _stream

    rp, ci, n_cols = case("two_hubs")
    n = rp.shape[0] - 1
    rng = np.random.default_rng(14)
    X = rng.standard_normal((n_cols, F)).astype(np.float32)
    val = rng.random(ci.shape[0]).astype(np.float32)
    ref = oracle.spmm_csr(rp, ci, val, X)
    # shards: [0,400) local, [400,700) owner 1, [700,1000) owner 2 ; owner 0 = local buffer itself
    bounds = [0, 400, 700, n_cols]
    shift = 9
    enc = ci.copy()
    for o in (1, 2):
        m = (ci >= bounds[o]) & (ci < bounds[o + 1])
        enc[m] = bounds[1] + (o << shift) + (ci[m] - bounds[o])
    shards = [T(X[bounds[o]:bounds[o + 1]], dev) for o in range(3)]
    st = plan_structure(rp, enc, n_cols, dev)
    ptrs = (ctypes.c_void_p * 3)(*[t.data_ptr() for t in shards])
    y = torch.empty((n, F), device=dev)
    plan, keep = st.plan_struct(_scratch("spmm", st, F))
    _cabi.call("cogdl_b200_spmm_csr_f32_peers", _ptr(st.rowptr), _ptr(st.colind), _ptr(T(val, dev)), _ptr(shards[0]),
               bounds[1], ctypes.cast(ptrs, ctypes.c_void_p), 3, shift, _ptr(y), n, F, plan, _stream(dev))
    torch.cuda.synchronize()
    got = y.cpu().numpy()
    unsplit = np.diff(rp) <= st.chunk_edges
    assert np.array_equal(got[unsplit], ref[unsplit]) and rel(got, ref) <= TOL


# ------------------------------------------------------------------------------------ SDDMM
@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "rect", "empty_graph"])
@pytest.mark.parametrize("F", [128, 16, 40, 7, 256, 1, 600])
def test_sddmm_matches_oracle(dev, name, F):
    from cogdl_b200.operators._raw import sddmm_raw

    rp, ci, n_cols = case(name)
    rng = np.random.default_rng(5)
    n = rp.shape[0] - 1
    D1 = rng.standard_normal((n, F)).astype(np.float32)
    D2 = rng.standard_normal((n_cols, F)).astype(np.float32)
    ref = oracle.sddmm_csr(rp, ci, D1, D2)
    out = sddmm_raw(plan_structure(rp, ci, n_cols, dev), T(D1, dev), T(D2, dev)).cpu().numpy()
    assert rel(out, ref) <= TOL


# ------------------------------------------------------------------------------------ csr2csc
@pytest.mark.parametrize("name", list(CASES))
def test_csr2csc_bit_exact(dev, name):
    rp, ci, n_cols = case(name)
    colptr, rowind, perm = oracle.csr2csc(rp, ci, n_cols)
    st_t, p = plan_structure(rp, ci, n_cols, dev).csc()
    assert np.array_equal(st_t.rowptr.cpu().numpy(), colptr)
    assert np.array_equal(st_t.colind.cpu().numpy(), rowind)
    assert np.array_equal(p.cpu().numpy(), perm)


def test_gather_rows(dev):
    from cogdl_b200.operators._raw import gather_rows_raw

    rng = np.random.default_rng(6)
    perm = rng.permutation(1000).astype(np.int32)
    x = rng.standard_normal((1000, 8)).astype(np.float32)
    out = gather_rows_raw(T(perm, dev), T(x, dev)).cpu().numpy()
    assert np.array_equal(out, oracle.gather_rows(perm, x))


# ------------------------------------------------------------------------------------ edge softmax
@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "two_hubs", "empty_graph"])
@pytest.mark.parametrize("H", [8, 1, 2, 4, 16, 32, 3, 6])
def test_edge_softmax_fwd_bwd(dev, name, H):
    from cogdl_b200.operators._raw import edge_softmax_fwd_raw, edge_softmax_bwd_raw

    rp, ci, n_cols = case(name)
    rng = np.random.default_rng(7)
    e = np.clip(rng.standard_normal((ci.shape[0], H)) * 3, -10, 10).astype(np.float32)
    g = rng.standard_normal((ci.shape[0], H)).astype(np.float32)
    yref = oracle.edge_softmax_fwd(rp, e)
    gref = oracle.edge_softmax_bwd(rp, yref, g)
    # chunk 256: tiles of 2048 floats or the warp kernel (H >= 16); 64 / 16: the 512- and 1024-float tiles,
    # many chunks per hub row (split-row statistics), cp.async.bulk staging when H % 4 == 0; 0: no plan
    for chunk in (256, 64, 16, 0):
        st = plan_structure(rp, ci, n_cols, dev, chunk=chunk)
        y = edge_softmax_fwd_raw(st, T(e, dev))
        gin = edge_softmax_bwd_raw(st, T(yref, dev), T(g, dev))
        assert rel(y.cpu().numpy(), yref) <= TOL, chunk
        assert rel(gin.cpu().numpy(), gref) <= TOL, chunk
        if ci.shape[0]:
            # rows sum to one per head
            seg = np.add.reduceat(y.cpu().numpy(), rp[:-1][np.diff(rp) > 0], axis=0)
            assert np.allclose(seg, 1.0, atol=1e-5)
        if chunk:
            assert int(st.plan.counters.abs().sum()) == 0   # arrival counters left clean by both passes
        # unaligned views (offset by one float): the bulk path must be refused, results unchanged
        if H % 4 == 0 and ci.shape[0]:
            buf = torch.empty(e.size + 1, device=dev)
            ev = buf[1:].view(e.shape)
            ev.copy_(T(e, dev))
            assert torch.equal(edge_softmax_fwd_raw(st, ev), y) or rel(edge_softmax_fwd_raw(st, ev).cpu().numpy(), yref) <= TOL


@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "two_hubs", "empty_graph"])
@pytest.mark.parametrize("H", [8, 1, 4, 16, 3])
def test_gat_attention_backward_and_colsum(dev, name, H):
    """cogdl_b200_gat_attn_bwd_f32 + cogdl_b200_edge_colsum_f32 against the oracle's written-out autograd."""
    from cogdl_b200.operators._raw import gat_attn_bwd_raw, edge_colsum_raw

    rp, ci, n_cols = case(name)
    if n_cols != rp.shape[0] - 1:
        pytest.skip("square graphs only (h_l / h_r share the node set)")
    n = rp.shape[0] - 1
    rng = np.random.default_rng(21)
    att = oracle.edge_softmax_fwd(rp, np.clip(rng.standard_normal((ci.shape[0], H)) * 2, -8, 8).astype(np.float32))
    d_att = rng.standard_normal((ci.shape[0], H)).astype(np.float32)
    hl, hr = rng.standard_normal((n, H)).astype(np.float32), rng.standard_normal((n, H)).astype(np.float32)
    de_ref, gr_ref, gc_ref = oracle.gat_attn_bwd(rp, ci, att, d_att, hl, hr, 0.2)
    for chunk in (256, 16, 0):
        st = plan_structure(rp, ci, n_cols, dev, chunk=chunk)
        de, gr = gat_attn_bwd_raw(st, T(att, dev), T(d_att, dev), T(hl, dev), T(hr, dev), 0.2)
        assert rel(de.cpu().numpy(), de_ref) <= TOL and rel(gr.cpu().numpy(), gr_ref) <= TOL, chunk
        st_t, perm = st.csc()
        gc = edge_colsum_raw(st_t, perm, de)
        assert rel(gc.cpu().numpy(), gc_ref) <= TOL, chunk
        gc2 = edge_colsum_raw(st_t, perm, de)
        assert torch.equal(gc, gc2)            # deterministic


# ------------------------------------------------------------------------------------ multi-head
@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "rect", "empty_graph"])
@pytest.mark.parametrize("H,F", [(8, 128), (8, 16), (8, 8), (2, 64), (4, 32), (1, 128), (3, 5), (8, 24), (2, 256)])
def test_mhspmm_and_mhsddmm(dev, name, H, F):
    from cogdl_b200.operators._raw import mhspmm_raw, mhsddmm_raw

    rp, ci, n_cols = case(name)
    n = rp.shape[0] - 1
    rng = np.random.default_rng(8)
    att = rng.random((ci.shape[0], H)).astype(np.float32)
    feat = rng.standard_normal((n_cols, H, F)).astype(np.float32)
    grad = rng.standard_normal((n, H, F)).astype(np.float32)
    ref = oracle.mhspmm(rp, ci, att, feat)
    ref_sd = oracle.mhsddmm(rp, ci, grad, feat)
    for chunk, seg_cost in ((0, None), (256, None), (256, 0)):   # seg_cost 0: row kernel with hub chunks
        st = plan_structure(rp, ci, n_cols, dev, chunk=chunk, seg_cost=seg_cost)
        out = mhspmm_raw(st, T(att, dev), T(feat, dev)).cpu().numpy()
        unsplit = np.diff(rp) <= chunk if chunk else np.ones(n, bool)
        assert np.array_equal(out[unsplit], ref[unsplit])
        assert rel(out, ref) <= TOL
        sd = mhsddmm_raw(st, T(grad, dev), T(feat, dev)).cpu().numpy()
        assert rel(sd, ref_sd) <= TOL


def test_mhspmm_transpose_with_fused_perm(dev):
    """grad_feat of the GAT aggregation: CSC pass with att[perm] fused into the kernel."""
    from cogdl_b200.operators._raw import mhspmm_raw

    rp, ci, n_cols = case("hub")
    rng = np.random.default_rng(9)
    H, F = 8, 16
    att = rng.random((ci.shape[0], H)).astype(np.float32)
    grad = rng.standard_normal((rp.shape[0] - 1, H, F)).astype(np.float32)
    colptr, rowind, perm = oracle.csr2csc(rp, ci, n_cols)
    ref = oracle.mhspmm(colptr, rowind, att, grad, perm=perm)
    st = plan_structure(rp, ci, n_cols, dev)
    st_t, p = st.csc()
    out = mhspmm_raw(st_t, T(att, dev), T(grad, dev), perm=p).cpu().numpy()
    assert rel(out, ref) <= TOL


# ------------------------------------------------------------------------------------ scatter_max
@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "two_hubs", "rect", "empty_graph"])
@pytest.mark.parametrize("F", [256, 128, 16, 7, 40, 1, 3, 9, 17, 33])
def test_scatter_max_fwd_bwd(dev, name, F):
    from cogdl_b200.operators._raw import scatter_max_fwd_raw, scatter_max_bwd_raw

    rp, ci, n_cols = case(name)
    n = rp.shape[0] - 1
    rng = np.random.default_rng(10)
    # mixed sign + deliberate ties (quantised values) to exercise "first max wins"
    X = np.round(rng.standard_normal((n_cols, F)) * 4).astype(np.float32) / 4
    ref, ref_id = oracle.scatter_max_fwd(rp, ci, X)
    for chunk, seg_cost in ((0, None), (256, None), (256, 0)):   # seg_cost 0: row kernel with hub chunks
        out, arg = scatter_max_fwd_raw(plan_structure(rp, ci, n_cols, dev, chunk=chunk, seg_cost=seg_cost), T(X, dev))
        assert np.array_equal(out.cpu().numpy(), ref)         # max is exact
        assert np.array_equal(arg.cpu().numpy(), ref_id)      # integer output: bit exact, ties included
    g = rng.standard_normal((n, F)).astype(np.float32)
    gref = oracle.scatter_max_bwd(g, ref_id, n_src=n_cols)
    gx = scatter_max_bwd_raw(T(g, dev), T(ref_id, dev), n_cols).cpu().numpy()
    assert rel(gx, gref) <= TOL   # atomics: order differs, values within tolerance


def test_scatter_max_reference_semantics_agree_on_positive_features(dev):
    from cogdl_b200.operators._raw import scatter_max_fwd_raw

    rp, ci, n_cols = case("ragged")
    X = (np.random.default_rng(11).random((n_cols, 64)) + 0.01).astype(np.float32)
    ref, ref_id = oracle.scatter_max_fwd(rp, ci, X, reference_semantics=True)
    out, arg = scatter_max_fwd_raw(plan_structure(rp, ci, n_cols, dev), T(X, dev))
    has = np.diff(rp) > 0
    assert np.array_equal(out.cpu().numpy()[has], ref[has]) and np.array_equal(arg.cpu().numpy()[has], ref_id[has])


def test_scatter_max_and_mhspmm_name_their_kernel(dev):
    """cogdl_b200_last_kernel() names what scatter_max (both forms) and the row form of the multi-head SpMM
    launched, not the kernel of an earlier call."""
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import mhspmm_raw, scatter_max_fwd_raw, spmm_raw

    rp, ci, n_cols = case("hub")
    st = plan_structure(rp, ci, n_cols, dev)
    rng = np.random.default_rng(15)
    spmm_raw(st, None, T(rng.standard_normal((n_cols, 128)).astype(np.float32), dev))
    assert "stream_kernel<" in _cabi.last_kernel()
    scatter_max_fwd_raw(st, T(rng.standard_normal((n_cols, 16)).astype(np.float32), dev))
    assert _cabi.last_kernel() == "cogdl_b200::scatter_max_fwd_kernel<float4,GROUP=4,NV=1>", _cabi.last_kernel()
    spmm_raw(st, None, T(rng.standard_normal((n_cols, 128)).astype(np.float32), dev))
    att = T(rng.random((ci.shape[0], 8)).astype(np.float32), dev)
    mhspmm_raw(st, att, T(rng.standard_normal((n_cols, 8, 8)).astype(np.float32), dev))
    assert _cabi.last_kernel() == "cogdl_b200::mhspmm_kernel<float4,GROUP=16,no_perm>", _cabi.last_kernel()
    scatter_max_fwd_raw(st, T(rng.standard_normal((n_cols, 256)).astype(np.float32), dev))
    assert _cabi.last_kernel() == "cogdl_b200::scatter_max_stream_kernel<NV=2,U=2>", _cabi.last_kernel()


# ------------------------------------------------------------------------------------ fused GAT
@pytest.mark.parametrize("name", ["tiny", "ragged", "hub", "empty_graph"])
@pytest.mark.parametrize("H,F", [(8, 128), (8, 16), (8, 8), (1, 64), (4, 32), (3, 5), (2, 192)])
def test_fused_gat_forward(dev, name, H, F):
    from cogdl_b200.operators._raw import gat_fwd_raw

    rp, ci, n_cols = case(name)
    if n_cols != rp.shape[0] - 1:
        pytest.skip("square only")
    n = n_cols
    rng = np.random.default_rng(12)
    h_l = rng.standard_normal((n, H)).astype(np.float32)
    h_r = rng.standard_normal((n, H)).astype(np.float32)
    feat = rng.standard_normal((n, H, F)).astype(np.float32)
    ref, ref_att = oracle.gat_fwd(rp, ci, h_l, h_r, feat, 0.2, return_att=True)
    out, att = gat_fwd_raw(plan_structure(rp, ci, n_cols, dev), T(h_l, dev), T(h_r, dev), T(feat, dev), 0.2, True)
    assert rel(out.cpu().numpy(), ref) <= TOL
    assert rel(att.cpu().numpy(), ref_att) <= TOL


# ------------------------------------------------------------------------------------ hub plan invariants
@pytest.mark.parametrize("name", ["ragged", "hub", "two_hubs", "tiny", "empty_graph"])
@pytest.mark.parametrize("chunk,seg", [(64, 128), (256, 32), (8, 16)])
def test_hub_plan_invariants(dev, name, chunk, seg):
    """The plan is what every kernel's work decomposition rests on: hub chunks must tile exactly the
    hub rows, segments must partition exactly the non-hub rows (in contiguous, hub-free runs), edge_row
    must be the COO row array, the hub list must be sorted by descending degree."""
    from cogdl_b200.structure import CSRStructure

    rp, ci, n_cols = case(name)
    n = rp.shape[0] - 1
    deg = np.diff(rp)
    st = CSRStructure(T(rp, dev), T(ci, dev), n_cols=n_cols, chunk_edges=chunk, seg_cost=seg)
    pl = st.plan
    hubs = np.nonzero(deg > chunk)[0]
    assert pl.n_hub_rows == len(hubs) and pl.n_empty_rows == int((deg == 0).sum())
    assert pl.n_chunks == int(np.ceil(deg[hubs] / chunk).sum())
    hub_rows = pl.hub_rows[: pl.n_hub_rows].cpu().numpy()
    assert sorted(hub_rows.tolist()) == hubs.tolist()
    assert np.all(np.diff(deg[hub_rows]) <= 0)                       # descending degree
    if pl.n_hub_rows:
        assert np.array_equal(pl._hub_deg_np, deg[hub_rows].astype(np.int32))
    chunks = pl.chunks[: 2 * pl.n_chunks].cpu().numpy().reshape(-1, 2)
    for r in hubs:                                                   # a row's chunks: contiguous slots, one first_slot
        mine = np.nonzero(chunks[:, 0] == r)[0]
        assert len(mine) == -(-deg[r] // chunk)
        assert np.array_equal(mine, np.arange(mine[0], mine[0] + len(mine))) and np.all(chunks[mine, 1] == mine[0])
    if ci.shape[0] == 0:
        return
    assert pl.n_segs > 0
    segs = pl.segs.cpu().numpy().reshape(-1, 2)
    covered = np.zeros(n, np.int32)
    for a, b in segs:
        assert 0 <= a < b <= n
        assert np.all(deg[a:b] <= chunk)                             # hub-free
        covered[a:b] += 1
        cost = int(rp[b] - rp[a]) + (b - a)
        assert cost <= seg + chunk + 1                               # bounded work per warp
    assert np.array_equal(covered, (deg <= chunk).astype(np.int32))  # every non-hub row exactly once
    assert np.array_equal(pl.edge_row.cpu().numpy(), np.repeat(np.arange(n), deg).astype(np.int32))
    assert int(pl.counters.abs().sum()) == 0


# ------------------------------------------------------------------------------------ structure tools
def test_coo2csr_index_device_bit_exact(dev):
    from cogdl_b200.data import coo2csr_index

    rng = np.random.default_rng(13)
    n, e = 5000, 60000
    row = rng.integers(0, n, e).astype(np.int64)
    rp_ref, re_ref = oracle.coo2csr_index(row, n)
    rp, re = coo2csr_index(torch.from_numpy(row).to(dev), n)
    assert np.array_equal(rp.cpu().numpy(), rp_ref) and np.array_equal(re.cpu().numpy(), re_ref)


def test_errors_are_raised_not_swallowed(dev):
    import cogdl_b200
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n_cols = case("tiny")
    st = plan_structure(rp, ci, n_cols, dev)
    with pytest.raises(ValueError):
        spmm_raw(st, torch.ones(3, device=dev), torch.ones(n_cols, 4, device=dev))  # wrong nnz
    with pytest.raises(RuntimeError):
        spmm_raw(st, None, torch.ones(n_cols, 4))  # CPU tensor: no fallback
    lib = cogdl_b200._cabi.load()
    assert lib.cogdl_b200_spmm_csr_f32(None, None, None, None, None, 5, 4, None, None) == cogdl_b200._cabi.EINVAL
    assert "null pointer" in cogdl_b200._cabi.last_error()


# ------------------------------------------------------------------------------------ row-stream launches
@pytest.mark.parametrize("F", [128, 40, 256])
def test_stream_spmm_on_hub_chunks_matches_the_oracle(dev, F):
    """The row-stream SpMM with 64-edge hub chunks: the oracle's bits on unsplit rows, the arrival counters left
    at zero."""
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n_cols = case("two_hubs")
    rng = np.random.default_rng(21)
    X = rng.standard_normal((n_cols, F)).astype(np.float32)
    val = rng.random(ci.shape[0]).astype(np.float32)
    st = plan_structure(rp, ci, n_cols, dev, chunk=64)
    y = spmm_raw(st, T(val, dev), T(X, dev)).cpu().numpy()
    ref = oracle.spmm_csr(rp, ci, val, X)
    unsplit = np.diff(rp) <= 64
    assert np.array_equal(y[unsplit], ref[unsplit]) and rel(y, ref) <= TOL
    assert int(st.plan.counters.abs().sum()) == 0


@pytest.mark.parametrize("name", ["two_hubs", "ragged", "empty_graph"])
@pytest.mark.parametrize("H,F", [(1, 128), (1, 256), (8, 128), (2, 256)])
def test_sddmm_stream_and_row_forms_match_the_oracle(dev, name, H, F):
    """Rows of 128 / 256 floats per head take the row-stream SDDMM when the plan has segments and the row form
    otherwise.  Both agree with the oracle, with and without hub chunks."""
    from cogdl_b200.operators._raw import mhsddmm_raw, sddmm_raw

    rp, ci, n_cols = case(name)
    n = rp.shape[0] - 1
    rng = np.random.default_rng(23)
    grad = rng.standard_normal((n, H, F)).astype(np.float32)
    feat = rng.standard_normal((n_cols, H, F)).astype(np.float32)
    if H == 1:
        ref = oracle.sddmm_csr(rp, ci, grad[:, 0], feat[:, 0])
        run = lambda st: sddmm_raw(st, T(grad[:, 0], dev), T(feat[:, 0], dev))
    else:
        ref = oracle.mhsddmm(rp, ci, grad, feat)
        run = lambda st: mhsddmm_raw(st, T(grad, dev), T(feat, dev))
    # stream form (default plan), row form with hub chunks (plan without segments), row form without a plan
    for chunk, seg_cost in ((64, None), (64, 0), (0, None)):
        st = plan_structure(rp, ci, n_cols, dev, chunk=chunk, seg_cost=seg_cost)
        out = run(st).cpu().numpy()
        assert rel(out, ref) <= TOL, f"chunk={chunk} seg_cost={seg_cost}"
        if chunk:
            assert int(st.plan.counters.abs().sum()) == 0

"""Parity at BENCHMARK size (BASELINE.json configs C3 / C4 / C5 shapes), not only on toy graphs.

Every op that bench.py times on a full-size graph is compared here, at that size, with the CPU oracle:
  * C3  arxiv-shaped graph (169 343 nodes, 1 335 586 nnz incl. self loops, max degree ~22 600), H = 8,
        F = 128: edge-softmax fwd / bwd, multi-head SpMM (CSR and perm-fused CSC), multi-head SDDMM,
        GAT forward -- the WHOLE graph goes through the oracle;
  * C4  products-shaped graph (2 449 029 nodes, 61 859 140 edges): scatter_max F = 256 and unweighted
        SpMM F = 128 on a contiguous >= 10 M-edge row slice PLUS the 64 top-degree hub rows (where the
        32-bit item math, chunk scratch and in-order hub combination are actually exercised);
  * C5  one papers100M/8 shard (13 882 494 rows, 201 960 734 edges), SpMM F = 128: same slicing.

Tolerances are ELEMENT-WISE: |a - b| <= 1e-5 * max(|b|, scale of the element's reduction group) (the
row for SpMM / scatter_max, the (row, head) group for edge-aligned tensors); integer outputs and SpMM
rows that the hub plan does not split must be bit-exact.  Hub rows of SpMM are also held to an fp64
sum: the fp32 sequential oracle is itself ~eps*sqrt(deg) off on 10^5..10^6-edge rows.
"""
import numpy as np
import pytest
import torch

import oracle
from tests.gpu_util import dev

pytestmark = pytest.mark.gpu

TOL = 1e-5


def rowwise_err(got, ref):
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    flat = ref.reshape(ref.shape[0], -1)
    scale = np.maximum(np.abs(flat), np.abs(flat).max(axis=1, keepdims=True))
    return float((np.abs(got.reshape(flat.shape) - flat) / np.maximum(scale, 1e-30)).max())


def edgewise_err(got, ref, rowptr, mag=None):
    """Edge-aligned [nnz, H] tensors: scale = max(|ref|, max |ref| over the (destination row, head)
    group, 0.05 * mag).  `mag` (optional) is the magnitude of the terms the element is a signed sum of
    (sum_f |a_f b_f| for a dot product): where a result cancels to ~0 its own size is not a yardstick."""
    got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
    starts = rowptr[:-1].astype(np.int64)
    nonempty = rowptr[1:] > rowptr[:-1]
    gmax = np.zeros((rowptr.shape[0] - 1, ref.shape[1]))
    gmax[nonempty] = np.maximum.reduceat(np.abs(ref), starts[nonempty], axis=0)
    scale = np.maximum(np.abs(ref), np.repeat(gmax, np.diff(rowptr), axis=0))
    if mag is not None:
        scale = np.maximum(scale, 0.05 * np.asarray(mag, np.float64))
    return float((np.abs(got - ref) / np.maximum(scale, 1e-30)).max())


def sub_csr(rp, ci, rows):
    """(rebased rowptr, colind) of the listed rows, host numpy int32."""
    lens = (rp[rows + 1] - rp[rows]).astype(np.int64)
    out_rp = np.zeros(rows.shape[0] + 1, np.int64)
    np.cumsum(lens, out=out_rp[1:])
    pos = np.repeat(rp[rows].astype(np.int64) - out_rp[:-1], lens) + np.arange(out_rp[-1])
    return out_rp.astype(np.int32), ci[pos]


def slice_and_hubs(rp, min_edges=10_000_000, n_hubs=64):
    """Row ids of a contiguous slice holding >= min_edges edges (from the middle of the graph) plus the
    n_hubs highest-degree rows."""
    n = rp.shape[0] - 1
    deg = np.diff(rp)
    start = n // 3
    end = int(np.searchsorted(rp, rp[start] + min_edges))
    end = min(max(end, start + 1), n)
    hubs = np.argsort(-deg, kind="stable")[:n_hubs]
    return np.unique(np.concatenate([np.arange(start, end), hubs]))


# ------------------------------------------------------------------------------------------- C3
@pytest.fixture(scope="module")
def arxiv(dev):
    import cogdl_b200
    from cogdl_b200 import synth

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0)
    g = cogdl_b200.Graph(row_ptr=rp, col=col, num_nodes=n).to(dev)
    st = g.structure()
    return st, rp.numpy().astype(np.int32), col.numpy().astype(np.int32), n


def test_c3_edge_softmax_fwd_bwd_full_arxiv_h8(dev, arxiv):
    from cogdl_b200.operators._raw import edge_softmax_fwd_raw, edge_softmax_bwd_raw

    st, rp, ci, n = arxiv
    assert int(np.diff(rp).max()) > 20000        # the 22 K-edge hub is in this graph
    gen = torch.Generator(device=dev).manual_seed(3)
    logits = (torch.randn(st.nnz, 8, device=dev, generator=gen) * 3).clamp_(-10, 10)
    y = edge_softmax_fwd_raw(st, logits)
    ref = oracle.edge_softmax_fwd(rp, logits.cpu().numpy())
    assert edgewise_err(y.cpu().numpy(), ref, rp) <= TOL
    sums = np.add.reduceat(y.double().cpu().numpy(), rp[:-1].astype(np.int64), axis=0)
    assert np.abs(sums - 1.0).max() <= 1e-5      # every (row, head) group sums to one
    gy = torch.randn(st.nnz, 8, device=dev, generator=gen)
    gin = edge_softmax_bwd_raw(st, y, gy)
    yh, gh = y.cpu().numpy(), gy.cpu().numpy()
    gref = oracle.edge_softmax_bwd(rp, yh, gh)
    # gin = y*g - y*sum(y*g): magnitude of the two terms (deg-2 groups with g1 ~ g2 cancel to ~0)
    s_abs = np.add.reduceat((yh * np.abs(gh)).astype(np.float64), rp[:-1].astype(np.int64), axis=0)
    mag = yh * (np.abs(gh) + np.repeat(s_abs, np.diff(rp), axis=0))
    assert edgewise_err(gin.cpu().numpy(), gref, rp, mag=mag) <= TOL


def test_c3_mhspmm_mhsddmm_gat_full_arxiv_h8_f128(dev, arxiv):
    from cogdl_b200.operators._raw import edge_softmax_fwd_raw, mhspmm_raw, mhsddmm_raw, gat_fwd_raw

    st, rp, ci, n = arxiv
    H, F = 8, 128
    gen = torch.Generator(device=dev).manual_seed(4)
    att = edge_softmax_fwd_raw(st, (torch.randn(st.nnz, H, device=dev, generator=gen) * 3).clamp_(-10, 10))
    h = torch.randn(n, H, F, device=dev, generator=gen)
    att_h, h_h = att.cpu().numpy(), h.cpu().numpy()
    # forward mh-SpMM: unsplit rows bit-exact (CSR order, fp32 mul then add), all rows element-wise
    out = mhspmm_raw(st, att, h).cpu().numpy()
    ref = oracle.mhspmm(rp, ci, att_h, h_h)
    unsplit = np.diff(rp) <= st.chunk_edges
    assert np.array_equal(out[unsplit], ref[unsplit])
    assert rowwise_err(out.reshape(n, H, F).reshape(n * H, F), ref.reshape(n * H, F)) <= TOL
    # backward pieces: perm-fused CSC mh-SpMM (= grad wrt feat) and mh-SDDMM (= grad wrt attention)
    st_t, perm = st.csc()
    gout = torch.randn(n, H, F, device=dev, generator=gen)
    gfeat = mhspmm_raw(st_t, att, gout, perm=perm).cpu().numpy()
    colptr, rowind, perm_ref = oracle.csr2csc(rp, ci, n)
    assert np.array_equal(perm.cpu().numpy(), perm_ref)
    gfeat_ref = oracle.mhspmm(colptr, rowind, att_h, gout.cpu().numpy(), perm=perm_ref)
    assert rowwise_err(gfeat.reshape(n * H, F), gfeat_ref.reshape(n * H, F)) <= TOL
    gatt = mhsddmm_raw(st, gout, h).cpu().numpy()
    gatt_ref = oracle.mhsddmm(rp, ci, gout.cpu().numpy(), h_h)
    # a dot product of 128 N(0,1) pairs cancels to ~0 for some edges: yardstick includes sum_f |g_f h_f|
    mag = oracle.mhsddmm(rp, ci, np.abs(gout.cpu().numpy()), np.abs(h_h))
    assert edgewise_err(gatt, gatt_ref, rp, mag=mag) <= TOL
    # GAT forward (attention kernel + mh-SpMM) against the fp64 oracle
    hl, hr = torch.randn(n, H, device=dev, generator=gen), torch.randn(n, H, device=dev, generator=gen)
    o, a = gat_fwd_raw(st, hl, hr, h, 0.2, True)
    o_ref, a_ref = oracle.gat_fwd(rp, ci, hl.cpu().numpy(), hr.cpu().numpy(), h_h, 0.2, return_att=True)
    assert edgewise_err(a.cpu().numpy(), a_ref, rp) <= TOL
    assert rowwise_err(o.cpu().numpy().reshape(n * H, F), o_ref.reshape(n * H, F)) <= TOL


# ------------------------------------------------------------------------------------------- C4
@pytest.fixture(scope="module")
def products(dev):
    import cogdl_b200
    from cogdl_b200 import synth

    n, e = synth.SHAPES["products"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, device=dev, self_loops=False)
    st = cogdl_b200.CSRStructure.from_int64(rp, col, n_cols=n)
    del rp, col
    rp_h, ci_h = st.rowptr.cpu().numpy(), st.colind.cpu().numpy()
    rows = slice_and_hubs(rp_h)
    srp, sci = sub_csr(rp_h, ci_h, rows)
    assert srp[-1] >= 10_000_000
    return st, rp_h, rows, srp, sci, n


def test_c4_scatter_max_f256_products_slice_and_hubs(dev, products):
    from cogdl_b200.operators._raw import scatter_max_fwd_raw

    st, rp_h, rows, srp, sci, n = products
    gen = torch.Generator(device=dev).manual_seed(5)
    x = torch.rand(n, 256, device=dev, generator=gen) + 0.01     # strictly positive: reference == fixed semantics
    out, arg = scatter_max_fwd_raw(st, x)
    ridx = torch.from_numpy(rows).to(dev)
    got_o, got_a = out[ridx].cpu().numpy(), arg[ridx].cpu().numpy()
    ref_o, ref_a = oracle.scatter_max_fwd(srp, sci, x.cpu().numpy())
    assert np.array_equal(got_a, ref_a), "argmax must be bit-exact (first max in CSR order), hubs included"
    assert np.array_equal(got_o, ref_o), "max is a selection: exact"
    ref_o2, ref_a2 = oracle.scatter_max_fwd(srp, sci, x.cpu().numpy(), reference_semantics=True)
    assert np.array_equal(ref_o2, ref_o) and np.array_equal(ref_a2, ref_a)


def test_c4_spmm_f128_products_slice_and_hubs(dev, products):
    from cogdl_b200.operators._raw import spmm_raw

    st, rp_h, rows, srp, sci, n = products
    gen = torch.Generator(device=dev).manual_seed(6)
    x = torch.randn(n, 128, device=dev, generator=gen)
    y = spmm_raw(st, None, x)
    got = y[torch.from_numpy(rows).to(dev)].cpu().numpy()
    xh = x.cpu().numpy()
    ref = oracle.spmm_csr(srp, sci, None, xh)
    deg = np.diff(srp)
    unsplit = deg <= st.chunk_edges
    assert unsplit.sum() > 100000 and (~unsplit).sum() >= 64
    assert np.array_equal(got[unsplit], ref[unsplit]), "unsplit rows: bit-identical to the reference CPU order"
    # rows up to 4096 edges: the fp32 sequential oracle is still a valid yardstick (its own error ~ eps*sqrt(deg)/5)
    mid = deg <= 4096
    assert rowwise_err(got[mid], ref[mid]) <= TOL
    # heavier hubs (up to ~6e5 edges here): the sequential fp32 sum is itself > 1e-5 off -> fp64 yardstick
    big = np.nonzero(~mid)[0]
    assert big.size >= 32
    ref64 = np.stack([xh[sci[srp[j]:srp[j + 1]]].astype(np.float64).sum(0) for j in big])
    assert rowwise_err(got[big], ref64) <= TOL
    some = np.nonzero(~unsplit & mid)[0][:512]
    ref64s = np.stack([xh[sci[srp[j]:srp[j + 1]]].astype(np.float64).sum(0) for j in some])
    assert rowwise_err(got[some], ref64s) <= TOL


# ------------------------------------------------------------------------------------------- C5
def test_c5_papers_shard_spmm_f128_slice_and_hubs(dev):
    import cogdl_b200
    from cogdl_b200 import synth
    from cogdl_b200.operators._raw import spmm_raw

    rows_n, edges = synth.shard_sizes(8, "weak")
    rp, col = synth.shard_csr(0, 1, rows_n, edges, 0.0, seed=0, device=dev)
    st = cogdl_b200.CSRStructure.from_int64(rp, col, n_cols=rows_n)
    del rp, col
    gen = torch.Generator(device=dev).manual_seed(7)
    x = torch.randn(rows_n, 128, device=dev, generator=gen)
    y = spmm_raw(st, None, x)
    rp_h, ci_h = st.rowptr.cpu().numpy(), st.colind.cpu().numpy()
    assert int(np.diff(rp_h).max()) > 500000          # the ~1.5 M-edge hub of this shard
    rows = slice_and_hubs(rp_h, n_hubs=16)
    srp, sci = sub_csr(rp_h, ci_h, rows)
    got = y[torch.from_numpy(rows).to(dev)].cpu().numpy()
    xh = x.cpu().numpy()
    ref = oracle.spmm_csr(srp, sci, None, xh)
    unsplit = np.diff(srp) <= st.chunk_edges
    assert np.array_equal(got[unsplit], ref[unsplit])
    assert rowwise_err(got[unsplit], ref[unsplit]) == 0.0
    hub_ids = np.nonzero(~unsplit)[0]
    big = hub_ids[np.argsort(-np.diff(srp)[hub_ids])[:16]]
    ref64 = np.stack([xh[sci[srp[j]:srp[j + 1]]].astype(np.float64).sum(0) for j in big])
    assert rowwise_err(got[big], ref64) <= TOL, "hub rows (up to ~1.5 M edges) within 1e-5 of the fp64 sum"
    rest = np.setdiff1d(hub_ids, big)[:2000]
    ref64r = np.stack([xh[sci[srp[j]:srp[j + 1]]].astype(np.float64).sum(0) for j in rest])
    assert rowwise_err(got[rest], ref64r) <= TOL

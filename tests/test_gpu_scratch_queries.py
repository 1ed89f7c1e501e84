"""Every entry point with a hub-plan scratch need, on a graph with hub chunks in its rows and its columns: the wrapper
asks for exactly its family's cogdl_b200_<family>_scratch_bytes, the entry runs with partials_bytes at that value, and
with 4 bytes less it returns COGDL_B200_ESCRATCH before any launch."""
import ctypes
from types import SimpleNamespace

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.gpu_util import dev

pytestmark = pytest.mark.gpu

# H a power of two with H * chunk_edges <= 2048: the edge-softmax kernels take their split-row path, which uses the
# partials; F = K * d with d a power of two for the routing
N, H, F, K, B, T, D = 1500, 4, 32, 4, 2, 3, 4


@pytest.fixture(scope="module")
def g(dev):
    """A symmetric power-law graph (hub rows and hub columns) and every operand the cases read."""
    from cogdl_b200 import synth
    from cogdl_b200.operators import _raw
    from cogdl_b200.operators.fused_gcn import fused_gcn_raw
    from cogdl_b200.operators.fused_sage import fused_sage_raw
    from cogdl_b200.operators.label_prop import label_prop_raw
    from cogdl_b200.structure import CSRStructure

    rp, col = synth.powerlaw_csr(N, 8 * N, seed=5)
    m = sp.csr_matrix((np.ones(col.numel()), col.numpy(), rp.numpy()), shape=(N, N))
    m = (m + m.T).tocsr()
    m.sort_indices()
    st = CSRStructure(torch.from_numpy(m.indptr.astype(np.int32)).to(dev),
                      torch.from_numpy(m.indices.astype(np.int32)).to(dev))
    st_t, perm = st.csc()
    nnz = st.nnz
    gen = torch.Generator().manual_seed(0)

    def r(*shape):
        return torch.randn(*shape, generator=gen).to(dev)

    def idx(hi, n):
        return torch.randint(0, hi, (n,), generator=gen, dtype=torch.int32).to(dev)

    g = SimpleNamespace(st=st, st_t=st_t, perm=perm, val=r(nnz).abs(), x=r(N, F), z=r(N, F), rs=r(N).abs(),
                        b_dev=r(1), h_l=r(N, H), h_r=r(N, H), feat=r(N, H, F), e=r(nnz, H), etype=idx(T, nnz),
                        h_e=r(T, H), x128=r(N, 128), w_gcn=r(16, 128) / 11.3, w_sage=r(16, 256) / 16,
                        beta=torch.ones(1, device=dev), attr=r(nnz, D), w_enc=r(F, D), q=r(N, F), c=r(N, F),
                        idx2=idx(5, nnz), b=r(5, F), coef=r(T, B), raw=_raw, fused_gcn_raw=fused_gcn_raw,
                        fused_sage_raw=fused_sage_raw, label_prop_raw=label_prop_raw)
    g.att = _raw.edge_softmax_fwd_raw(st, g.e)
    g.sa = _raw.softmax_aggr_fwd_raw(st, g.x, g.beta, 1e-7, want_lse=True)
    g.ge = _raw.genconv_edge_fwd_raw(st, g.x, g.attr, g.w_enc, g.beta, 1e-7, want_lse=True)
    g.dr = _raw.disen_route_fwd_raw(st, g.q, g.c, K, 1.0, want_saved=True)
    assert st.plan.n_chunks > 0 and st_t.plan.n_chunks > 0 and st.plan.n_segs > 0
    return g


def _peers(g):
    from cogdl_b200.operators._raw import _launch, _scratch
    from cogdl_b200.structure import _ptr

    y = torch.empty_like(g.x)
    ptrs = (ctypes.c_void_p * 1)(g.x.data_ptr())      # every column is local: the peer form's gather with one shard
    _launch("cogdl_b200_spmm_csr_f32_peers", g.st, _scratch("spmm", g.st, F), _ptr(g.st.rowptr), _ptr(g.st.colind),
            _ptr(g.val), _ptr(g.x), N, ctypes.cast(ptrs, ctypes.c_void_p), 1, 12, _ptr(y), N, F)


# (id, family, shape after n_chunks, plan of the transpose, call)
CASES = [
    ("spmm_f32", "spmm", (F,), False, lambda g: g.raw.spmm_raw(g.st, g.val, g.x)),
    ("spmm_f16", "spmm", (F,), False, lambda g: g.raw.spmm_raw(g.st, g.val, g.x.half())),
    ("spmm_2src", "spmm", (F,), False, lambda g: g.raw.spmm_2src_raw(g.st, g.val, g.x[:700], g.x[700:])),
    ("spmm_peers", "spmm", (F,), False, _peers),
    ("spmm_residual", "spmm", (F,), False, lambda g: g.raw.spmm_residual_raw(g.st, g.val, g.x, g.z, 0.5, 0.5, g.rs)),
    ("label_prop", "spmm", (F,), False, lambda g: g.label_prop_raw(g.st, g.val, g.x, g.z, 0.5, 0.5, clamp=(-1, 1))),
    ("spmm_residual_dcoef", "spmm", (F,), False,
     lambda g: g.raw.spmm_residual_dcoef_raw(g.st, g.val, g.x, g.z, 1.0, g.b_dev)),
    ("spmm_accum", "spmm", (F,), False, lambda g: g.raw.spmm_accum_raw(g.st, g.val, g.x, g.z.clone(), row_scale=g.rs)),
    ("mhspmm", "mhspmm", (H, F), False, lambda g: g.raw.mhspmm_raw(g.st, g.att, g.feat)),
    ("mhspmm_dropout", "mhspmm", (H, F), False, lambda g: g.raw.mhspmm_raw(g.st, g.att, g.feat, drop_scale=2.0)),
    ("gat_fwd", "gat_fwd", (H, F), False, lambda g: g.raw.gat_fwd_raw(g.st, g.h_l, g.h_r, g.feat, 0.2, True)),
    ("gat_fwd_dropout", "gat_fwd", (H, F), False,
     lambda g: g.raw.gat_fwd_raw(g.st, g.h_l, g.h_r, g.feat, 0.2, True, drop=(7, 2 ** 62, 4 / 3))),
    ("edge_softmax_fwd", "edge_softmax", (H,), False, lambda g: g.raw.edge_softmax_fwd_raw(g.st, g.e)),
    ("edge_softmax_bwd", "edge_softmax", (H,), False, lambda g: g.raw.edge_softmax_bwd_raw(g.st, g.att, g.e)),
    ("gat_attn_bwd", "edge_softmax", (H,), False,
     lambda g: g.raw.gat_attn_bwd_raw(g.st, g.att, g.e, g.h_l, g.h_r, 0.2)),
    ("gat_attn_bwd_dropout", "edge_softmax", (H,), False,
     lambda g: g.raw.gat_attn_bwd_raw(g.st, g.att, g.e, g.h_l, g.h_r, 0.2, drop_scale=2.0)),
    ("hgn_attn", "edge_softmax", (H,), False,
     lambda g: g.raw.hgn_attn_raw(g.st, g.etype, g.h_l, g.h_r, g.h_e, 0.2, True, res_attn=g.att, alpha=0.1)),
    ("hgn_attn_bwd", "edge_softmax", (H,), False,
     lambda g: g.raw.hgn_attn_bwd_raw(g.st, g.etype, g.att, g.e, g.h_l, g.h_r, g.h_e, 0.2, 0.9)),
    ("scatter_max", "scatter_max", (F,), False, lambda g: g.raw.scatter_max_fwd_raw(g.st, g.x)),
    ("edge_colsum", "edge_colsum", (H,), True, lambda g: g.raw.edge_colsum_raw(g.st_t, g.perm, g.e)),
    ("gcn_fused", "gcn_fused", (128,), False, lambda g: g.fused_gcn_raw(g.st, g.val, g.x128, g.w_gcn)),
    ("sage_fused_sum", "sage_fused", (128, 0), False,
     lambda g: g.fused_sage_raw(g.st, g.val, g.rs, g.x128, g.w_sage, aggr="sum")),
    ("sage_fused_max", "sage_fused", (128, 1), False,
     lambda g: g.fused_sage_raw(g.st, None, None, g.x128, g.w_sage, aggr="max")),
    ("softmax_aggr_fwd", "softmax_aggr", (F,), False,
     lambda g: g.raw.softmax_aggr_fwd_raw(g.st, g.x, g.beta, 1e-7, want_lse=True)),
    ("softmax_aggr_fwd_q", "softmax_aggr", (F,), False,
     lambda g: g.raw.softmax_aggr_fwd_raw(g.st, g.x, g.beta, 1e-7, want_lse=True, want_q=True)),
    ("softmax_aggr_bwd", "softmax_aggr_bwd", (F,), True,
     lambda g: g.raw.softmax_aggr_bwd_raw(g.st, g.x, g.beta, 1e-7, g.z, g.sa[0], g.sa[1])),
    ("genconv_edge_fwd", "softmax_aggr", (F,), False,
     lambda g: g.raw.genconv_edge_fwd_raw(g.st, g.x, g.attr, g.w_enc, g.beta, 1e-7, want_q=True)),
    ("genconv_edge_bwd", "genconv_edge_bwd", (F, 1), True,
     lambda g: g.raw.genconv_edge_bwd_raw(g.st, g.x, g.attr, g.w_enc, g.beta, 1e-7, g.z, g.ge[0], g.ge[1])),
    ("disen_route_fwd", "disen_route", (F, K), False, lambda g: g.raw.disen_route_fwd_raw(g.st, g.q, g.c, K, 1.0)),
    ("disen_route_bwd_rows", "disen_route", (F, K), False,
     lambda g: g.raw.disen_route_bwd_raw(g.st, g.q, g.c, K, 1.0, g.z, *g.dr)),
    ("disen_route_bwd_cols", "disen_route", (F, K), True,
     lambda g: g.raw.disen_route_bwd_raw(g.st, g.q, g.c, K, 1.0, g.z, *g.dr)),
    ("comp_aggr", "comp_aggr", (F,), False, lambda g: g.raw.comp_aggr_raw(g.st, g.idx2, g.val, g.x, g.b, "mult")),
    ("rgcn_aggr", "rgcn_aggr", (B, F), False, lambda g: g.raw.rgcn_aggr_raw(g.st, g.etype, g.val, g.coef, g.x)),
]


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_entry_checks_the_scratch_its_query_gives(dev, g, case, monkeypatch):
    from cogdl_b200 import _cabi
    from cogdl_b200.structure import CSRStructure

    _, family, shape, transpose, run = case
    st = g.st_t if transpose else g.st
    lib = _cabi.load()
    need = int(getattr(lib, f"cogdl_b200_{family}_scratch_bytes")(st.plan.n_chunks, *shape))
    assert need > 0
    run(g)                                   # builds what the call caches
    torch.cuda.synchronize(dev)

    plan_struct, asked, short = CSRStructure.plan_struct, [], [0]

    def exact_plan(self, partial_bytes=0):
        plan, keep = plan_struct(self, partial_bytes)
        if self is st:
            asked.append(partial_bytes)
            keep[0].partials_bytes = partial_bytes - short[0]
        return plan, keep

    monkeypatch.setattr(CSRStructure, "plan_struct", exact_plan)
    run(g)
    torch.cuda.synchronize(dev)
    assert asked == [need]
    short[0] = 4
    n0 = lib.cogdl_b200_launch_count()
    with pytest.raises(_cabi.CogdlB200Error) as e:
        run(g)
    assert e.value.code == _cabi.ESCRATCH, str(e.value)
    assert lib.cogdl_b200_launch_count() == n0

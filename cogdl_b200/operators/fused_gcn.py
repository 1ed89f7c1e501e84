"""Fused GCN layer: act((A.X).W^T + (A.1) b^T) in one kernel with a wgmma GEMM epilogue (SURVEY 8f-3).

Mathematically the reference layer `act(spmm(graph, linear(x)))` (cogdl/layers/gcn_layer.py:51-64; the bias
is added BEFORE the aggregation there, hence the (A.1) b^T term), re-associated -- so it is opt-in
(`GCNLayer(..., fused=True)` in cogdl_b200.layers, or call `fused_gcn_layer` directly) and is held to 1e-5
against an fp64 evaluation instead of being bit-matched.  Kernel: cogdl_b200/csrc/fused_gcn.cu.
"""
import torch

from .. import _cabi
from ..structure import CSRStructure, _ptr, graph_operands, require_cuda
from ._raw import _launch, _scratch, spmm_adjoint_raw, spmm_raw


def supported(K, Fout):
    return bool(_cabi.load().cogdl_b200_gcn_fused_supported(int(K), int(Fout)))


_ROWSUM = {}     # (structure id, weights storage, version) -> A.1, for fixed edge weights (GCN: sym-norm, never trained)


def cached_rowsum(st, val):
    """A.1 = per-row sum of the edge values, computed once per (structure, weight tensor) with the SpMM kernel."""
    if val is None:
        return None
    key = (id(st), val.data_ptr(), val._version, val.numel())
    ent = _ROWSUM.get(key)
    if ent is None:
        if len(_ROWSUM) >= 8:
            _ROWSUM.pop(next(iter(_ROWSUM)))
        ones = torch.ones((st.n_cols, 4), dtype=torch.float32, device=val.device)
        ent = _ROWSUM[key] = (spmm_raw(st, val, ones)[:, 0].contiguous(), st, val)   # keep st / val alive under the key
    return ent[0]


def fused_gcn_raw(st: CSRStructure, val, x, weight, bias=None, relu=False, cache_rowsum=True):
    """x [n_src,128] fp32, weight [Fout,128] (nn.Linear layout), bias [Fout] | None -> [n_rows, Fout]."""
    dev = require_cuda(x, weight, val, bias)
    if x.dtype != torch.float32 or weight.dtype != torch.float32:
        raise TypeError("fused_gcn_raw: float32 only")
    x, weight = x.contiguous(), weight.contiguous()
    K, Fout = x.shape[1], weight.shape[0]
    if weight.shape[1] != K or not supported(K, Fout):
        raise ValueError(f"fused GCN layer needs in_features == 128 and out_features <= 128, got {K} -> {Fout}")
    val = None if val is None else val.detach().contiguous().view(-1).float() if val.dtype != torch.float32 or not val.is_contiguous() else val.detach().view(-1)
    bias = None if bias is None else bias.contiguous().float()
    if st.nnz == 0:        # no edge anywhere: A = 0, so (A.X).W^T + (A.1) b^T = 0 and act(0) = 0 for ReLU / identity
        return torch.zeros((st.n_rows, Fout), dtype=torch.float32, device=dev)
    out = torch.empty((st.n_rows, Fout), dtype=torch.float32, device=dev)
    hub = torch.empty((st.n_rows, K), dtype=torch.float32, device=dev) if st.plan.n_chunks > 0 else None
    rowsum = cached_rowsum(st, val) if (cache_rowsum and val is not None and bias is not None) else None
    _launch("cogdl_b200_gcn_fused_f32", st, _scratch("gcn_fused", st, K), _ptr(st.rowptr), _ptr(st.colind), _ptr(val),
            _ptr(x), _ptr(weight), _ptr(bias), _ptr(rowsum), _ptr(out), _ptr(hub), st.n_rows, K, Fout, int(bool(relu)))
    return out


class FusedGCNFunction(torch.autograd.Function):
    """Forward: the fused kernel.  Backward (training): with G' = dOUT * relu'(OUT),
       dW = G'^T (A.X)   db = G'^T (A.1)   dX = A^T (G' W)        -- A.X is recomputed by one SpMM (it was never
       written in the forward), the dense products are plain library GEMMs (cuBLAS via torch.matmul)."""

    @staticmethod
    def forward(ctx, st, val, x, weight, bias, relu, sym):
        out = fused_gcn_raw(st, val, x, weight, bias, relu)
        ctx.st, ctx.relu, ctx.sym = st, bool(relu), bool(sym)
        ctx.save_for_backward(val, x, weight, bias, out if relu else None)
        return out

    @staticmethod
    def backward(ctx, g):
        val, x, weight, bias, out = ctx.saved_tensors
        st = ctx.st
        g = g.contiguous()
        if ctx.relu:
            g = g * (out > 0)
        gx = gw = gb = None
        if ctx.needs_input_grad[3] or (bias is not None and ctx.needs_input_grad[4]):
            ax = spmm_raw(st, val, x)
            if ctx.needs_input_grad[3]:
                gw = g.t() @ ax
            if bias is not None and ctx.needs_input_grad[4]:
                ones = torch.ones((x.shape[0], 4), device=x.device)
                gb = g.t() @ spmm_raw(st, val, ones)[:, 0]
        if ctx.needs_input_grad[2]:
            gx = spmm_adjoint_raw(st, val, (g @ weight).contiguous(), ctx.sym)
        return None, None, gx, gw, gb, None, None


def fused_gcn_layer(graph, x, weight, bias=None, relu=False):
    """graph: cogdl_b200.Graph or a real cogdl.data.Graph (same attribute surface as spmm())."""
    st, val, out_norm, in_norm, sym = graph_operands(graph)
    if out_norm is not None or in_norm is not None:
        raise NotImplementedError("fused GCN layer: graphs with separate in/out norms take the unfused path")
    return FusedGCNFunction.apply(st, val, x, weight, bias, relu, sym)

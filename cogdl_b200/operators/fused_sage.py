"""Fused GraphSAGE layer: act(x.W_self^T + b + agg(x).W_neigh^T) with the neighbour half in the fused kernel's
wgmma epilogue.

The reference layer is `fc(cat[x, agg(x)])` (cogdl/layers/sage_layer.py:69-87) with fc.weight = [W_self | W_neigh].
Here S = x.W_self^T + b is one library GEMM (as the unfused `fc` uses), and the aggregation never goes to global
memory: it is formed tile by tile in shared memory and multiplied by W_neigh there (cogdl_b200/csrc/fused_gcn.cu,
EPI_SELF instantiations).  Nothing is re-associated: the aggregated tile is bit-identical to the unfused
aggregation, only the GEMM rounds differently (bf16x3 split, ~1e-7 of the row scale vs fp64).  Opt-in through
`SAGELayer(..., fused=True)` in cogdl_b200.layers, or call `fused_sage_layer` directly.
"""
import torch
import torch.nn.functional as F

from ..structure import CSRStructure, _ptr, graph_operands, require_cuda
from ._raw import _launch, _scratch, scatter_max_bwd_raw, scatter_max_fwd_raw, spmm_adjoint_raw, spmm_raw
from .fused_gcn import supported

AGGR = {"sum": 0, "max": 1}     # COGDL_B200_AGGR_SUM / _MAX; mean is "sum" with row-normalised weights or row_scale


def _flat_f32(t):
    return None if t is None else t.detach().reshape(-1).float().contiguous()


def fused_sage_raw(st: CSRStructure, val, row_scale, x, weight, bias=None, aggr="sum", relu=False):
    """x [n_src,128] fp32, weight [Fout,256] (fc.weight: self half | neighbour half), bias [Fout] | None.
    aggr "sum": agg = row_scale * (A.x), A = (st, val); "max": agg = neighbour max (val, row_scale must be None).
    Returns act(x[:n_rows].W_self^T + b + agg.W_neigh^T), [n_rows, Fout]."""
    dev = require_cuda(x, weight, val, row_scale, bias)
    if x.dtype != torch.float32 or weight.dtype != torch.float32:
        raise TypeError("fused_sage_raw: float32 only")
    if aggr not in AGGR:
        raise ValueError(f"fused_sage_raw: aggr must be 'sum' or 'max', got {aggr!r}")
    if aggr == "max" and (val is not None or row_scale is not None):
        raise ValueError("fused_sage_raw: max aggregation takes no edge values or row scale")
    x = x.contiguous()
    K, Fout = x.shape[1], weight.shape[0]
    if weight.shape[1] != 2 * K or not supported(K, Fout):
        raise ValueError(f"fused SAGE layer needs in_feats == 128 and out_feats <= 128 (fc.weight [Fout, 256]), "
                         f"got fc.weight {tuple(weight.shape)} for x {tuple(x.shape)}")
    n = st.n_rows
    if x.shape[0] < n:
        raise ValueError(f"fused_sage_raw: x has {x.shape[0]} rows, the graph {n}")
    val, row_scale = _flat_f32(val), _flat_f32(row_scale)
    if row_scale is not None and row_scale.numel() != n:
        raise ValueError(f"row_scale has {row_scale.numel()} entries, the graph {n} rows")
    S = F.linear(x[:n], weight[:, :K], bias).contiguous()           # self half + bias: the unfused fc's GEMM
    if st.nnz == 0:          # no edge anywhere: agg = 0 for sum and max
        return torch.relu(S) if relu else S
    w_neigh = weight[:, K:].contiguous()
    out = torch.empty((n, Fout), dtype=torch.float32, device=dev)
    hub = torch.empty((n, K), dtype=torch.float32, device=dev) if st.plan.n_chunks > 0 else None
    _launch("cogdl_b200_sage_fused_f32", st, _scratch("sage_fused", st, K, AGGR[aggr]), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(val), _ptr(row_scale), _ptr(x), _ptr(w_neigh), _ptr(S), _ptr(out), _ptr(hub), n, K, Fout, AGGR[aggr],
            int(bool(relu)))
    return out


class FusedSAGEFunction(torch.autograd.Function):
    """Forward: the fused kernel.  Backward, with G' = dOUT * relu'(OUT) and the aggregation recomputed (it was
    never written in the forward):
       dW = [G'^T x | G'^T agg]   db = sum_rows G'   dx = G' W_self + (neighbour term of d = G' W_neigh)
    neighbour term: sum / mean  A^T (row_scale * d)  (the CSR itself when the graph is flagged symmetric, else the
    cached transpose with permuted weights, as FusedGCNFunction); max  scatter_max backward of d through the
    recomputed argmax.  Dense products are library GEMMs."""

    @staticmethod
    def forward(ctx, st, val, row_scale, x, weight, bias, aggr, relu, sym):
        out = fused_sage_raw(st, val, row_scale, x, weight, bias, aggr, relu)
        ctx.st, ctx.aggr, ctx.relu, ctx.sym = st, aggr, bool(relu), bool(sym)
        ctx.save_for_backward(val, row_scale, x, weight, bias, out if relu else None)
        return out

    @staticmethod
    def backward(ctx, g):
        val, row_scale, x, weight, bias, out = ctx.saved_tensors
        st, K = ctx.st, x.shape[1]
        n = st.n_rows
        g = g.contiguous()
        if ctx.relu:
            g = g * (out > 0)
        rs = None if row_scale is None else row_scale.detach().reshape(-1, 1).float()
        need_w, need_x = ctx.needs_input_grad[4], ctx.needs_input_grad[3]
        gx = gw = gb = None
        agg = arg = None
        if ctx.aggr == "max" and (need_w or need_x):
            agg, arg = scatter_max_fwd_raw(st, x)
        elif need_w:
            agg = spmm_raw(st, val, x)
            if rs is not None:
                agg = rs * agg
        if need_w:
            gw = torch.cat([g.t() @ x[:n], g.t() @ agg], dim=1)
        if bias is not None and ctx.needs_input_grad[5]:
            gb = g.sum(0)
        if need_x:
            d = (g @ weight[:, K:]).contiguous()
            if ctx.aggr == "max":
                gx = scatter_max_bwd_raw(d, arg, x.shape[0])
            else:
                if rs is not None:
                    d = rs * d
                gx = spmm_adjoint_raw(st, val, d, ctx.sym)
            gx[:n] += g @ weight[:, :K]
        return None, None, None, gx, gw, gb, None, None, None


def fused_sage_layer(graph, x, weight, bias=None, aggr="mean", relu=False):
    """graph: cogdl_b200.Graph or a real cogdl.data.Graph.  aggr "mean" row-normalises the graph first (as the
    reference MeanAggregator); "sum" and "mean" use the edge weights and graph.in_norm as spmm() does."""
    if aggr == "mean":
        graph.row_norm()
    st, val, out_norm, row_scale, sym = graph_operands(graph)
    if out_norm is not None:
        raise NotImplementedError("fused SAGE layer: graphs with an out_norm take the unfused path")
    if aggr == "max":
        val = row_scale = None
    elif val.requires_grad:
        raise NotImplementedError("fused SAGE layer: trainable edge weights take the unfused path")
    return FusedSAGEFunction.apply(st, val, row_scale, x, weight, bias, "max" if aggr == "max" else "sum", relu, sym)

"""R-GCN relational aggregation under a basis decomposition (cogdl/layers/rgcn_layer.py:118-150) without a
per-relation tensor.

With W_t = sum_b coef[t, b] V_b, the relational sum sum_t A_t x W_t (A_t: the graph restricted to the type-t edges)
needs no [T, N, F_out] tensor:

    agg[i, b] = sum_{q in row i} w_q coef[t_q, b] x[col_q]        one gather of x per edge, B accumulators
    out       = agg.view(N, B * F_in) @ V.view(B * F_in, F_out)   one GEMM

The aggregation is one launch of cogdl_b200_rgcn_aggr_f32 (cogdl_b200/csrc/rgcn.cu).  agg[:, b] is bit-identical to
this package's SpMM with per-slot values fl(w * coef[type, b]).  The backward is the same kernel family plus GEMMs: the
feature gradient runs the fan-out over the cached transpose (on d out for the layer, per basis on d agg for the
aggregation alone), and d coef is a per-edge dot (cogdl_b200_rgcn_edge_dot_f32) reduced per type by the SpMM over the
type-grouped slot index.  Everything is reproducible run to run, and nothing but the first call on a graph synchronises
with the host.
"""
import torch

from ..structure import graph_operands, rgcn_structure_for, unsupported_operands
from ._raw import rgcn_aggr_raw, rgcn_edge_dot_raw, spmm_raw


def _dcoef(rs, val, dagg, x, T):
    """d coef [T, B]: sum over the type-t slots q of w_q <dagg[row_q, b], x[col_q]>, reduced in slot order."""
    p = rgcn_edge_dot_raw(rs.st, val, dagg, x)
    return spmm_raw(rs.by_type(T), None, p)


def _transposed(rs, val):
    st_t, type_t, perm = rs.transpose()
    return st_t, type_t, val.detach()[perm]


class RgcnAggregateFunction(torch.autograd.Function):
    """agg [N, B, F] = the fan-out aggregation of x with coefficients coef, over the typed structure rs and the
    per-slot weights val (structural: they get no gradient)."""

    @staticmethod
    def forward(ctx, rs, val, x, coef):
        ctx.rs = rs
        ctx.save_for_backward(val, x, coef)
        return rgcn_aggr_raw(rs.st, rs.type, val, coef, x)

    @staticmethod
    def backward(ctx, g):
        val, x, coef = ctx.saved_tensors
        rs = ctx.rs
        g = g.contiguous()
        dx = dcoef = None
        if ctx.needs_input_grad[2]:
            # dx[j] = sum_b sum_{q: col_q = j} w_q coef[t_q, b] g[row_q, b]: the per-basis fan-out over the transpose
            st_t, type_t, w_t = _transposed(rs, val)
            dx = rgcn_aggr_raw(st_t, type_t, w_t, coef, g, per_basis=True).sum(dim=1)
        if ctx.needs_input_grad[3]:
            dcoef = _dcoef(rs, val, g, x, coef.shape[0])
        return None, None, dx, dcoef


class RgcnConvFunction(torch.autograd.Function):
    """out [N, F_out] = agg.view(N, B * F_in) @ V.view(B * F_in, F_out): the relational sum sum_t A_t x W_t with
    W_t = sum_b coef[t, b] V_b.  Backward: d V = agg^T d out; d x = D.view(N, B * F_out) @ [V_b^T] with D the fan-out of
    d out over the transpose; d coef from d agg = d out V^T by the edge dot."""

    @staticmethod
    def forward(ctx, rs, val, x, coef, V):
        N, F_in = x.shape
        B, F_out = V.shape[0], V.shape[2]
        agg = rgcn_aggr_raw(rs.st, rs.type, val, coef, x)
        out = agg.view(N, B * F_in) @ V.reshape(B * F_in, F_out)
        ctx.rs = rs
        ctx.save_for_backward(val, x if ctx.needs_input_grad[3] else None, coef, V,
                              agg if ctx.needs_input_grad[4] else None)
        return out

    @staticmethod
    def backward(ctx, g):
        val, x, coef, V, agg = ctx.saved_tensors
        rs = ctx.rs
        g = g.contiguous()
        B, F_in, F_out = V.shape
        N = g.shape[0]
        dx = dcoef = dV = None
        if ctx.needs_input_grad[4]:
            dV = (agg.view(N, B * F_in).t() @ g).view(B, F_in, F_out)
        if ctx.needs_input_grad[2]:
            st_t, type_t, w_t = _transposed(rs, val)
            D = rgcn_aggr_raw(st_t, type_t, w_t, coef, g)                      # [N, B, F_out]
            dx = D.view(-1, B * F_out) @ V.transpose(1, 2).reshape(B * F_out, F_in)
        if ctx.needs_input_grad[3]:
            dagg = (g @ V.reshape(B * F_in, F_out).t()).view(N, B, F_in)
            dcoef = _dcoef(rs, val, dagg, x, coef.shape[0])
        return None, None, dx, dcoef, dV


def _operands(graph, x, coef, entry):
    """(rs, val, x with out_norm applied, in_norm or None) of a graph with edge types in graph.edge_attr, checked."""
    err = unsupported_operands(graph, x, coef, entry=entry, what="features and coefficients")
    if err is not None:
        raise err
    st, val, out_norm, in_norm, _ = graph_operands(graph)
    etype = graph.edge_attr          # read once the CSR exists: the types are in the order of its slots
    if etype is None:
        raise ValueError(f"{entry}: the graph carries no edge types (graph.edge_attr is None)")
    if val.requires_grad:
        raise ValueError(f"{entry}: edge weights that require grad are not supported (they would get no gradient)")
    if x.dim() != 2 or x.shape[0] != st.n_cols:
        raise ValueError(f"{entry}: x must be [{st.n_cols}, F], got {tuple(x.shape)}")
    if coef.dim() != 2:
        raise ValueError(f"{entry}: coef must be [T, B], got {tuple(coef.shape)}")
    rs = rgcn_structure_for(st, etype)
    if rs.max_type >= coef.shape[0]:
        raise ValueError(f"{entry}: edge type {rs.max_type} is out of range for {coef.shape[0]} relations")
    val = val.to(x.device, torch.float32)
    if out_norm is not None:
        x = out_norm.to(x.device) * x
    return rs, val, x, None if in_norm is None else in_norm.to(x.device)


def rgcn_aggregate(graph, x, coef):
    """The basis aggregation of R-GCN: agg[i, b] = sum_t coef[t, b] (A_t x)[i] for fp32 CUDA x [N, F] and coef
    [T, B], with A_t the graph restricted to its type-t edges, weighted and normalised as spmm(graph, .) weights it
    (the raw edge weights in CSR order, out_norm on x, in_norm on the rows).  The types come from graph.edge_attr ([E]
    integers in [0, T), read after the CSR exists so each stays with its edge).  Returns [N, B, F], with autograd to x
    and coef; edge weights get none (a weight tensor that requires grad raises).  Raises ValueError for a type outside
    [0, T) before any launch, and, as spmm does, on CPU or non-fp32 tensors and dense grb_adj graphs."""
    rs, val, x, in_norm = _operands(graph, x, coef, "rgcn_aggregate")
    agg = RgcnAggregateFunction.apply(rs, val, x, coef)
    return agg if in_norm is None else in_norm.view(-1, 1, 1) * agg


def rgcn_conv(graph, x, coef, weight):
    """R-GCN's relational sum sum_t spmm(A_t, x W_t) with W_t = sum_b coef[t, b] weight[b]: coef [T, B], weight
    [B, F_in, F_out], x [N, F_in], all fp32 CUDA; the graph as rgcn_aggregate takes it.  One fan-out aggregation and
    one GEMM, with autograd to x, coef and weight.  Returns [N, F_out]."""
    rs, val, x, in_norm = _operands(graph, x, coef, "rgcn_conv")
    if weight.dim() != 3 or weight.shape[0] != coef.shape[1] or weight.shape[1] != x.shape[1]:
        raise ValueError(f"rgcn_conv: weight must be [{coef.shape[1]}, {x.shape[1]}, F_out], got {tuple(weight.shape)}")
    out = RgcnConvFunction.apply(rs, val, x, coef, weight)
    return out if in_norm is None else in_norm.view(-1, 1) * out

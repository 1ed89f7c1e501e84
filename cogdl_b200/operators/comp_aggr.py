"""CompGCN composition aggregation (cogdl/models/nn/compgcn.py:94-151) without per-edge feature tensors.

The reference CompGCNLayer gathers x[col] and rel_embed[type] into [E/2, F_in] tensors per edge half, composes them,
multiplies the per-edge result by W ([E/2, F_out]), scales it by the edge norm, builds an int64 [E/2, F_out] index
and scatter_adds with float atomics.  The message is linear in W:

    sum_e w_e phi(x[col_e], R'[t_e]) W  ==  (sum_e w_e phi(x[col_e], R'[t_e])) W

so the layer is one sparse composition aggregation into [2, N, F_in] (cogdl_b200/csrc/comp_aggr.cu) followed by
N-row GEMMs.  Its backward is the same kernel family on the cached transpose (dx) and on the type-grouped CSR (dR').
Nothing edge-sized and feature-wide is allocated, and forward and backward are bitwise reproducible.
"""
import torch

from ..structure import CompStructure, comp_structure_for
from ._raw import comp_aggr_raw

COMPGCN_OPS = ("sub", "mult")


class CompAggrFunction(torch.autograd.Function):
    """[2, N, F] aggregation of both edge halves, agg[h, i] = sum_{e in h, row_e = i} w_e phi(x[col_e], rel[t_e]),
    with gradients for x and rel (the weights are structural)."""

    @staticmethod
    def forward(ctx, cs, x, rel, opn):
        N, F = x.shape
        out = comp_aggr_raw(cs.csr, cs.type, cs.w, x, rel, opn).view(2, N, F)
        ctx.cs, ctx.opn = cs, opn
        ctx.save_for_backward(x, rel)
        return out

    @staticmethod
    def backward(ctx, g):
        x, rel = ctx.saved_tensors
        cs, opn = ctx.cs, ctx.opn
        g = g.contiguous().view(2 * cs.n_nodes, -1)
        dx = drel = None
        if ctx.needs_input_grad[1]:
            # dx[j] = sum_{e: col_e = j} w_e g[stacked row_e] (* rel[t_e] for mult)
            t, ttype, tw = cs.transpose()
            dx = comp_aggr_raw(t, ttype, tw, g, rel, "mult" if opn == "mult" else "copy")
        if ctx.needs_input_grad[2]:
            # drel[t] = sum_{e: t_e = t} w_e g[stacked row_e] * x[col_e]   (mult)
            #         = -sum_{e: t_e = t} w_e g[stacked row_e]              (sub)
            st, tcol, tw = cs.by_type(rel.shape[0])
            if opn == "mult":
                drel = comp_aggr_raw(st, tcol, tw, g, x, "mult")
            else:
                drel = comp_aggr_raw(st, None, tw, g, None, "copy").neg_()
        return None, dx, drel, None


def compgcn_aggregate(edge_index, edge_type, x, rel, opn, chunk_edges=None):
    """The two per-half aggregations of CogDL's CompGCNLayer before their weights: returns (agg_in, agg_out), each
    [N, F_in] with N = x.shape[0], where for half h (edges [0, E // 2) and [E // 2, E) of edge_index, in the order
    given) agg_h[i] = sum_{e in h, row_e = i} phi(x[col_e], rel[t_e]) / deg_h(i), phi = x - r ("sub") or x * r
    ("mult").  edge_index: (row, col) or [2, E] int64 on x's device; edge_type: [E] integers, on the host or the
    device.  The edge tensors are not modified, and the structure built from them is cached on their storage and
    version.  Raises ValueError for an index outside [0, N) or a type outside [0, rel.shape[0])."""
    if not x.is_cuda:
        raise RuntimeError("compgcn_aggregate: CUDA tensors only (no CPU fallback)")
    if x.dtype != torch.float32 or rel.dtype != torch.float32:
        raise TypeError(f"compgcn_aggregate: x and rel must be float32, got {x.dtype} and {rel.dtype}")
    if x.dim() != 2 or rel.dim() != 2 or rel.shape[1] != x.shape[1]:
        raise ValueError(f"compgcn_aggregate: x [N, F] and rel [T, F] expected, got {tuple(x.shape)} and "
                         f"{tuple(rel.shape)}")
    if opn not in COMPGCN_OPS:
        raise ValueError(f"compgcn_aggregate: opn must be one of {COMPGCN_OPS}, got {opn!r}")
    if isinstance(edge_type, CompStructure):
        cs = edge_type
    else:
        row, col = edge_index
        kw = {} if chunk_edges is None else {"chunk_edges": chunk_edges}
        cs = comp_structure_for(row, col, edge_type, x.shape[0], **kw)
    if cs.n_nodes != x.shape[0]:
        raise ValueError(f"compgcn_aggregate: structure for {cs.n_nodes} nodes, x has {x.shape[0]} rows")
    if cs.max_type >= rel.shape[0]:
        raise ValueError(f"compgcn_aggregate: edge type {cs.max_type} is out of range for {rel.shape[0]} relation rows")
    out = CompAggrFunction.apply(cs, x, rel, opn)
    return out[0], out[1]

"""Simple-HGN attention (myGATConv of CogDL's examples/simple_hgn/conv.py) on the fused GAT kernels.

The example's layer forms, per edge p = (i, j) of type t and head h,

    a   = edge_softmax(leakyrelu(h_l[i] + h_r[j] + h_e[t]))
    m   = (1 - alpha) * dropout(a) + alpha * res_attn          (the blend only when res_attn is given)
    out = mh_spmm(graph, m, h)

with an [E, H] tensor per step, two of which (and the dropout's mask) autograd keeps for the backward.  Here the
attention stage is one launch of cogdl_b200_hgn_attn_f32
(cogdl_b200/csrc/simple_hgn.cu): the logits are formed while loading, the dropout mask is drawn in the kernel (the rule
and seed of the fused GAT's attention dropout) and only two [E, H] tensors are written -- the returned attention m and,
when a gradient is needed, the softmax with the mask in its sign bit.  The backward keeps the signed softmax, and m only
when res_attn is given.  The aggregation is the multi-head SpMM over m.

Backward: d h is the CSC multi-head SpMM over m (perm fused; without res_attn over the signed softmax, read as the
dropout SpMM reads it, so m is not kept), d m the multi-head SDDMM, (d logit, d h_l) one pass of
cogdl_b200_hgn_attn_bwd_f32, d h_r the column sums over the cached transpose, d h_e [T, H] the SpMM over the slots
grouped by type (RgcnStructure.by_type) and d res_attn = alpha * d m.  No float atomics: every gradient is reproducible
run to run.
"""
import torch

from ..structure import graph_operands, rgcn_structure_for, unsupported_operands
from ._raw import (attn_dropout_args, edge_colsum_raw, hgn_attn_bwd_raw, hgn_attn_raw, hgn_max_table, mhsddmm_raw,
                   mhspmm_raw, spmm_raw)
from .fused_gat import draw_seed


class HgnAttentionFunction(torch.autograd.Function):
    """(out [n_rows, H, F], attention [nnz, H]) of the Simple-HGN attention over the typed structure rs.  drop =
    (seed, drop_below, scale) or None; the attention output carries no gradient (the layer returns it detached)."""

    @staticmethod
    def forward(ctx, rs, h, h_l, h_r, h_e, res_attn, slope, drop, alpha):
        st = rs.st
        want_att = any(t.requires_grad for t in (h_l, h_r, h_e))
        mix, att = hgn_attn_raw(st, rs.type, h_l, h_r, h_e, slope, want_att, drop=drop, res_attn=res_attn,
                                alpha=alpha)
        out = mhspmm_raw(st, mix, h)
        ctx.rs, ctx.slope = rs, float(slope)
        ctx.alpha = float(alpha) if res_attn is not None else 0.0
        ctx.keep_scale = 1.0 if drop is None else drop[2]
        ctx.dropped = drop is not None
        # without res_attn, mix is att read as the dropout SpMM reads it (dropped ? 0 : a * scale, the same rounding):
        # the backward aggregates over att and only one [E, H] tensor is kept
        ctx.save_for_backward(h, h_l, h_r, h_e, att, mix if res_attn is not None or att is None else None)
        ctx.mark_non_differentiable(mix)
        return out, mix

    @staticmethod
    def backward(ctx, grad_out, _grad_att):
        h, h_l, h_r, h_e, att, mix = ctx.saved_tensors
        rs = ctx.rs
        st = rs.st
        grad_out = grad_out.contiguous()
        need_h, need_l, need_r, need_e, need_res = ctx.needs_input_grad[1:6]
        st_t, perm = st.csc()
        dh = None
        if need_h:
            if mix is not None:
                dh = mhspmm_raw(st_t, mix, grad_out, perm=perm)
            else:
                dh = mhspmm_raw(st_t, att, grad_out, perm=perm, drop_scale=ctx.keep_scale if ctx.dropped else None)
        dl = dr = de = dres = None
        if need_l or need_r or need_e or need_res:
            dm = mhsddmm_raw(st, grad_out, h)                                   # [E, H]
            if need_res:
                dres = dm * ctx.alpha
            if need_l or need_r or need_e:
                d_edge, g_row = hgn_attn_bwd_raw(st, rs.type, att, dm, h_l, h_r, h_e, ctx.slope,
                                                 (1.0 - ctx.alpha) * ctx.keep_scale)
                dl = g_row if need_l else None
                dr = edge_colsum_raw(st_t, perm, d_edge) if need_r else None
                de = spmm_raw(rs.by_type(h_e.shape[0]), None, d_edge) if need_e else None
        return None, dh, dl, dr, de, dres, None, None, None


def hgn_attention(graph, h, h_l, h_r, h_e, edge_type, negative_slope, attn_drop=0.0, res_attn=None, alpha=0.0,
                  seed=None):
    """Simple-HGN's attention and aggregation on the graph's CSR: h [N, H, F], h_l [n_rows, H], h_r [N, H], the type
    table h_e [T, H], all fp32 CUDA; edge_type [E] integers in [0, T) and res_attn [E, H], both in the graph's CSR edge
    order (read them after the graph's CSR exists).  Per edge p = (i, j) and head h,

        a = softmax over row i of leakyrelu(h_l[i] + h_r[j] + h_e[edge_type[p]])
        m = (1 - alpha) * dropout(a) + alpha * res_attn     (m = dropout(a) without res_attn)
        out[i] = sum over row i of m[p] * h[j]

    The dropout keeps (CSR edge p, head h) iff the draw of (seed, p, h) is >= attn_drop * 2^64, as the fused GAT's
    attention dropout does, and scales a kept attention by 1 / (1 - attn_drop); seed None draws one from torch's CPU
    generator.  Returns (out [n_rows, H, F], m [E, H]); gradients flow through out to h, h_l, h_r, h_e and res_attn, m
    carries none.  Raises ValueError for a type outside [0, T) or a table with T * H above the kernels' limit, and, as
    spmm does, on CPU or non-fp32 tensors and dense grb_adj graphs -- all before any launch."""
    entry = "hgn_attention"
    err = unsupported_operands(graph, h, h_l, h_r, h_e, res_attn, entry=entry, what="features and attention terms")
    if err is not None:
        raise err
    st = graph_operands(graph).st
    if h.dim() != 3 or h.shape[0] != st.n_cols:
        raise ValueError(f"{entry}: h must be [{st.n_cols}, H, F], got {tuple(h.shape)}")
    H = h.shape[1]
    if h_l.shape != (st.n_rows, H) or h_r.shape != (st.n_cols, H):
        raise ValueError(f"{entry}: h_l must be [{st.n_rows}, {H}] and h_r [{st.n_cols}, {H}], got {tuple(h_l.shape)} "
                         f"and {tuple(h_r.shape)}")
    if h_e.dim() != 2 or h_e.shape[1] != H:
        raise ValueError(f"{entry}: h_e must be [T, {H}], got {tuple(h_e.shape)}")
    T = h_e.shape[0]
    if T < 1 or T * H > hgn_max_table():
        raise ValueError(f"{entry}: the type table is [T={T}, H={H}]; the fused attention takes T * H from 1 to "
                         f"{hgn_max_table()}")
    if res_attn is not None and res_attn.shape != (st.nnz, H):
        raise ValueError(f"{entry}: res_attn must be [{st.nnz}, {H}], got {tuple(res_attn.shape)}")
    rs = rgcn_structure_for(st, edge_type)
    if rs.max_type >= T:
        raise ValueError(f"{entry}: edge type {rs.max_type} is out of range for {T} types")
    drop = None
    if attn_drop:
        drop_below, scale = attn_dropout_args(attn_drop)
        drop = (draw_seed() if seed is None else int(seed) & (2 ** 64 - 1), drop_below, scale)
    return HgnAttentionFunction.apply(rs, h, h_l, h_r, h_e, res_attn, float(negative_slope), drop, float(alpha))

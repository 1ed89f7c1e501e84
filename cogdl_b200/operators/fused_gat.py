"""fused_gat_func -- the fused GAT operator behind cogdl.utils.fused_gat_op.

Reference: cogdl/operators/fused_gat.py:3-41 binds dgNN's fused_gatconv, but the binding is stale at
this pin (6 args / 3 outputs vs dgNN's 7 / 4; SURVEY 3.3), so it is dead code there.  We keep the
call signature `fused_gat_func(attn_row, attn_col, row_ptr, col_ind, col_ptr, row_ind,
negative_slope, in_feat)` and implement the op natively.  col_ptr/row_ind are accepted for
signature compatibility; the transpose comes from the cached structure.

Attention dropout (`attn_drop`, the nn.Dropout of gat_layer.py:76) runs inside the kernels: (CSR edge p, head h) is
kept iff draw(seed, p, h) >= floor(attn_drop * 2^64) (the counter-based generator of the sampler,
cogdl_b200_sample_draw) and a kept attention is scaled by 1 / (1 - attn_drop).  The saved attention carries the mask
in its sign bit, so the backward needs neither the seed nor a mask tensor.
"""
import torch

from ..structure import structure_for, CSRStructure
from ._raw import attn_dropout_args, gat_fwd_raw, mhspmm_raw, mhsddmm_raw, gat_attn_bwd_raw, edge_colsum_raw


def draw_seed():
    """A 64-bit seed from torch's CPU default generator: follows torch.manual_seed, needs no device synchronisation
    and gives every call a fresh mask."""
    lo, hi = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64).tolist()
    return (hi << 32) | lo


class FusedGATFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, attn_row, attn_col, row_ptr, col_ind, col_ptr, row_ind, negative_slope, in_feat, attn_drop=0.0,
                seed=None):
        st = row_ptr if isinstance(row_ptr, CSRStructure) else structure_for(row_ptr, col_ind, in_feat.shape[0])
        need_grad = any(t.requires_grad for t in (attn_row, attn_col, in_feat))
        drop = None
        if attn_drop:
            drop_below, scale = attn_dropout_args(attn_drop)
            drop = (draw_seed() if seed is None else int(seed) & (2 ** 64 - 1), drop_below, scale)
        out, att = gat_fwd_raw(st, attn_row, attn_col, in_feat, negative_slope, want_att=need_grad, drop=drop)
        ctx.st, ctx.slope = st, float(negative_slope)
        ctx.drop_scale = None if drop is None else drop[2]
        if need_grad:
            ctx.save_for_backward(attn_row, attn_col, in_feat, att)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        """Native backward (precedent dgNN fused_gatconv_kernel.cu:636-790), five library calls, no eager
        index arithmetic:  d feat = CSC mh-SpMM (perm fused) . d att = mh-SDDMM . (d edge, g_row) = softmax
        backward * LeakyReLU' + row sums in one pass (cogdl_b200_gat_attn_bwd_f32) . g_col = column sums of
        d edge through the cached transpose (cogdl_b200_edge_colsum_f32)."""
        attn_row, attn_col, feat, att = ctx.saved_tensors
        st = ctx.st
        grad_out = grad_out.contiguous()
        st_t, perm = st.csc()
        ds = ctx.drop_scale      # dropout: att is signed, the same three calls read the mask from it
        grad_feat = mhspmm_raw(st_t, att, grad_out, perm=perm, drop_scale=ds) if ctx.needs_input_grad[7] else None
        g_row = g_col = None
        if ctx.needs_input_grad[0] or ctx.needs_input_grad[1]:
            grad_att = mhsddmm_raw(st, grad_out, feat)                        # [E,H]
            d_edge, g_row = gat_attn_bwd_raw(st, att, grad_att, attn_row, attn_col, ctx.slope, drop_scale=ds)
            g_col = edge_colsum_raw(st_t, perm, d_edge) if ctx.needs_input_grad[1] else None
            if not ctx.needs_input_grad[0]:
                g_row = None
        return g_row, g_col, None, None, None, None, None, grad_feat, None, None


def fused_gat_func(attn_row, attn_col, row_ptr, col_ind, col_ptr, row_ind, negative_slope, in_feat):
    return FusedGATFunction.apply(attn_row, attn_col, row_ptr, col_ind, col_ptr, row_ind, negative_slope, in_feat)

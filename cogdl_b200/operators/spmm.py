"""csrspmm -- drop-in for cogdl.operators.spmm.csrspmm (cogdl/operators/spmm.py:24-80)."""
import torch

from ..structure import structure_for, CSRStructure
from ._raw import spmm_raw, sddmm_raw, gather_rows_raw


def _as_structure(rowptr, colind, n_cols):
    if isinstance(rowptr, CSRStructure):
        return rowptr
    return structure_for(rowptr, colind, n_cols)


class SPMMFunction(torch.autograd.Function):
    """out = A @ feat.  Backward as in the reference (spmm.py:57-80): grad_feat = A^T @ grad (the CSR
    itself when `sym`, else the cached transpose instead of a cuSPARSE csr2csc per call) and
    grad_edge_weight = SDDMM(grad, feat) when the weights require grad."""

    @staticmethod
    def forward(ctx, rowptr, colind, feat, edge_weight_csr=None, sym=False):
        st = _as_structure(rowptr, colind, feat.shape[0])
        out = spmm_raw(st, edge_weight_csr, feat)
        ctx.st, ctx.sym = st, bool(sym)
        need_w = edge_weight_csr is not None and edge_weight_csr.requires_grad
        ctx.has_w = edge_weight_csr is not None
        ctx.save_for_backward(edge_weight_csr if ctx.has_w else None, feat if need_w else None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        w, feat = ctx.saved_tensors
        st = ctx.st
        grad_out = grad_out.contiguous()
        grad_feat = grad_w = None
        if ctx.needs_input_grad[2]:
            if ctx.sym:
                grad_feat = spmm_raw(st, w, grad_out)
            else:
                st_t, perm = st.csc()
                w_t = None if w is None else gather_rows_raw(perm, w.detach().float())
                if w_t is not None and grad_out.dtype == torch.float16:
                    w_t = w_t.half()
                grad_feat = spmm_raw(st_t, w_t, grad_out)
        if ctx.has_w and ctx.needs_input_grad[3]:
            grad_w = sddmm_raw(st, grad_out.float(), feat.float()).to(w.dtype)
        return None, None, grad_feat, grad_w, None


class ActSPMMFunction(torch.autograd.Function):
    """SPMMFunction with an activation-compressed feature (the reference's ActSPMMFunction, spmm.py:89-133): when the
    edge weights require grad, feat is saved quantized (cogdl_b200.actnn.ops.quantize_activation, no scheme) and
    dequantized for the SDDMM weight gradient; otherwise nothing of feat is saved and it is SPMMFunction."""

    @staticmethod
    def forward(ctx, rowptr, colind, feat, edge_weight_csr=None, sym=False):
        from ..actnn.ops import quantize_activation

        st = _as_structure(rowptr, colind, feat.shape[0])
        out = spmm_raw(st, edge_weight_csr, feat)
        ctx.st, ctx.sym = st, bool(sym)
        ctx.has_w = edge_weight_csr is not None
        ctx.quantized = None
        if ctx.has_w and edge_weight_csr.requires_grad:
            ctx.quantized, ctx.feat_shape = quantize_activation(feat, None), feat.shape
        ctx.save_for_backward(edge_weight_csr if ctx.has_w else None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        from ..actnn.ops import dequantize_activation

        (w,) = ctx.saved_tensors
        feat = None
        if ctx.quantized is not None:
            feat = dequantize_activation(ctx.quantized, ctx.feat_shape)
            ctx.quantized = None
        st = ctx.st
        grad_out = grad_out.contiguous()
        grad_feat = grad_w = None
        if ctx.needs_input_grad[2]:
            if ctx.sym:
                grad_feat = spmm_raw(st, w, grad_out)
            else:
                st_t, perm = st.csc()
                w_t = None if w is None else gather_rows_raw(perm, w.detach().float())
                grad_feat = spmm_raw(st_t, w_t, grad_out)
        if feat is not None and ctx.needs_input_grad[3]:
            grad_w = sddmm_raw(st, grad_out.float(), feat.float()).to(w.dtype)
        return None, None, grad_feat, grad_w, None


def csrspmm(rowptr, colind, x, csr_data, sym=False, actnn=False):
    """Same signature as the reference.  actnn=True saves the features activation-compressed for the edge-weight
    gradient (ActSPMMFunction); the output is the same as with actnn=False."""
    if actnn:
        return ActSPMMFunction.apply(rowptr, colind, x, csr_data, sym)
    return SPMMFunction.apply(rowptr, colind, x, csr_data, sym)

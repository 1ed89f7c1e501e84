"""csrspmm -- drop-in for cogdl.operators.spmm.csrspmm (cogdl/operators/spmm.py:24-80)."""
import torch

from ..structure import structure_for, CSRStructure
from ._raw import sddmm_raw, spmm_adjoint_raw, spmm_raw


def _as_structure(rowptr, colind, n_cols):
    if isinstance(rowptr, CSRStructure):
        return rowptr
    return structure_for(rowptr, colind, n_cols)


class SPMMFunction(torch.autograd.Function):
    """out = A @ feat.  Backward as in the reference (spmm.py:57-80): grad_feat = A^T @ grad (the CSR
    itself when `sym`, else the cached transpose instead of a cuSPARSE csr2csc per call) and
    grad_edge_weight = SDDMM(grad, feat) when the weights require grad.  actnn=True is the reference's
    ActSPMMFunction (spmm.py:89-133): feat is then saved quantized (cogdl_b200.actnn.ops.quantize_activation, no
    scheme) and dequantized for the SDDMM; the output and grad_feat do not change."""

    @staticmethod
    def forward(ctx, rowptr, colind, feat, edge_weight_csr=None, sym=False, actnn=False):
        st = _as_structure(rowptr, colind, feat.shape[0])
        out = spmm_raw(st, edge_weight_csr, feat)
        ctx.st, ctx.sym = st, bool(sym)
        ctx.has_w = edge_weight_csr is not None
        need_w = ctx.has_w and edge_weight_csr.requires_grad
        ctx.quantized = None
        if need_w and actnn:
            from ..actnn.ops import quantize_activation

            ctx.quantized, ctx.feat_shape = quantize_activation(feat, None), feat.shape
        ctx.save_for_backward(edge_weight_csr, feat if need_w and not actnn else None)
        return out

    @staticmethod
    def backward(ctx, grad_out):
        w, feat = ctx.saved_tensors
        if ctx.quantized is not None:
            from ..actnn.ops import dequantize_activation

            feat = dequantize_activation(ctx.quantized, ctx.feat_shape)
            ctx.quantized = None
        grad_out = grad_out.contiguous()
        grad_feat = grad_w = None
        if ctx.needs_input_grad[2]:
            grad_feat = spmm_adjoint_raw(ctx.st, w, grad_out, ctx.sym)
        if ctx.has_w and ctx.needs_input_grad[3]:
            grad_w = sddmm_raw(ctx.st, grad_out.float(), feat.float()).to(w.dtype)
        return None, None, grad_feat, grad_w, None, None


def csrspmm(rowptr, colind, x, csr_data, sym=False, actnn=False):
    """Same signature as the reference.  actnn=True saves the features activation-compressed for the edge-weight
    gradient; the output is the same as with actnn=False."""
    return SPMMFunction.apply(rowptr, colind, x, csr_data, sym, actnn)

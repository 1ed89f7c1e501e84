"""GENConv aggregation (DeeperGCN / RevGCN; cogdl/layers/deepergcn_layer.py:64-93) without per-edge feature tensors.

The reference gathers x[col] into an [nnz, F] tensor, adds the edge encoder's output, applies relu + eps, runs the
edge softmax with F "heads" on beta times that, multiplies, and scatter_adds with float atomics -- several [nnz, F]
tensors per call in the forward and as many in the backward.  Here the softmax aggregations (softmax_sg, softmax,
mean = beta 0, sum = deg * mean) are one pass of cogdl_b200/csrc/softmax_aggr.cu over the CSR, with an online softmax
per channel in registers, and the backward is one pass over the cached transpose.  No [nnz, F] tensor exists unless
the caller passes an edge term (then its gradient is the only one written).  With a linear edge encoder (CogDL's
EdgeEncoder: edge term = edge_attr @ W.T), passing edge_attr and the encoder's weight instead forms the edge term inside
the kernels (cogdl_b200/csrc/genconv_edge.cu), so no [nnz, F] tensor exists in either direction.  max and powermean
without an edge term go through the existing scatter_max and SpMM kernels.
"""
import torch

from ..structure import CSRStructure, graph_operands
from ._raw import (GENCONV_EDGE_MAX_D, genconv_edge_bwd_raw, genconv_edge_fwd_raw, softmax_aggr_bwd_raw,
                   softmax_aggr_fwd_raw)
from .scatter_max import ScatterMaxFunction
from .spmm import SPMMFunction

AGGRS = ("softmax_sg", "softmax", "mean", "sum", "max", "powermean")


class SoftmaxAggrFunction(torch.autograd.Function):
    """out = sum_e softmax_e(beta m_e) m_e, m_e = relu(x[col_e] + edge_term[e]) + eps, with gradients for x, the
    edge term and beta (softmax_sg does not stop the gradient through the weights, as in CogDL).  beta is a
    one-element CUDA tensor; the kernels read it on the device, so a trainable beta costs no host sync."""

    @staticmethod
    def forward(ctx, st, x, edge_term, beta, eps):
        need_x, need_a, need_b = ctx.needs_input_grad[1:4]
        out, lse2, q = softmax_aggr_fwd_raw(st, x, beta, eps, edge_term, want_lse=need_x or need_a, want_q=need_b)
        ctx.st, ctx.eps = st, float(eps)
        ctx.save_for_backward(x, edge_term, beta, out, lse2, q)
        return out

    @staticmethod
    def backward(ctx, g):
        x, edge_term, beta, out, lse2, q = ctx.saved_tensors
        need_x, need_a, need_b = ctx.needs_input_grad[1:4]
        g = g.contiguous()
        dx = da = db = None
        if need_x or need_a:
            dx, da = softmax_aggr_bwd_raw(ctx.st, x, beta, ctx.eps, g, out, lse2, edge_term, want_edge_grad=need_a)
        if need_b:
            db = (g * (q - out * out)).sum().reshape(beta.shape)
        return None, dx if need_x else None, da, db, None


class GenconvEdgeFunction(torch.autograd.Function):
    """SoftmaxAggrFunction with edge_term = attr @ w.T formed in the kernels: gradients for x, w (the encoder's
    [F, D] weight) and beta, each only when asked for (a frozen w costs no dW pass, an x without grad no dx).  attr
    takes no gradient."""

    @staticmethod
    def forward(ctx, st, x, w, beta, attr, eps):
        need_x, need_w, need_b = ctx.needs_input_grad[1:4]
        out, lse2, q = genconv_edge_fwd_raw(st, x, attr, w, beta, eps, want_lse=need_x or need_w, want_q=need_b)
        ctx.st, ctx.eps = st, float(eps)
        ctx.save_for_backward(x, w, beta, attr, out, lse2, q)
        return out

    @staticmethod
    def backward(ctx, g):
        x, w, beta, attr, out, lse2, q = ctx.saved_tensors
        need_x, need_w, need_b = ctx.needs_input_grad[1:4]
        g = g.contiguous()
        dx = dw = db = None
        if need_x or need_w:
            dx, dw = genconv_edge_bwd_raw(ctx.st, x, attr, w, beta, ctx.eps, g, out, lse2, want_dx=need_x,
                                          want_dw=need_w)
        if need_b:
            db = (g * (q - out * out)).sum().reshape(beta.shape)
        return None, dx, dw, db, None, None


def _degrees(st):
    return (st.rowptr[1:] - st.rowptr[:-1]).to(torch.float32).unsqueeze(1)


def _check_edge_encoder(x, edge_term, edge_attr, edge_weight):
    """True when the call passes a linear edge encoder (edge_attr and edge_weight); rejects the combinations the
    fused kernels do not take.  Sizes against the graph are checked by the raw wrappers."""
    if edge_attr is None and edge_weight is None:
        return False
    if edge_attr is None or edge_weight is None:
        raise ValueError("genconv_aggregate: edge_attr and edge_weight go together")
    if edge_term is not None:
        raise ValueError("genconv_aggregate: pass edge_term or edge_attr with edge_weight, not both")
    if edge_attr.dim() != 2 or edge_weight.dim() != 2:
        raise ValueError(f"genconv_aggregate: edge_attr must be [nnz, D] and edge_weight [F, D], got "
                         f"{tuple(edge_attr.shape)} and {tuple(edge_weight.shape)}")
    if edge_attr.shape[1] > GENCONV_EDGE_MAX_D:
        raise ValueError(f"genconv_aggregate: edge_attr has D = {edge_attr.shape[1]} features; at most "
                         f"{GENCONV_EDGE_MAX_D} (pass edge_term = the encoder's output instead)")
    if edge_weight.shape != (x.shape[1], edge_attr.shape[1]):
        raise ValueError(f"genconv_aggregate: edge_weight must be [F={x.shape[1]}, D={edge_attr.shape[1]}], got "
                         f"{tuple(edge_weight.shape)}")
    if edge_attr.requires_grad:
        raise ValueError("genconv_aggregate: edge_attr that requires grad is not supported (its gradient is not "
                         "computed); pass edge_term = the encoder's output instead")
    return True


def genconv_aggregate(graph, x, aggr, beta=None, eps=1e-7, edge_term=None, p=1.0, *, edge_attr=None, edge_weight=None):
    """The aggregated h of CogDL's GENConv.forward before message_norm / residual / MLP.

    graph: cogdl_b200.Graph, a real cogdl.data.Graph or a CSRStructure; x [n_cols, F] fp32 CUDA; edge_term: the
    edge encoder's output [nnz, F] in CSR order (graph.edge_attr after the graph is in CSR form) or None.
    edge_attr [nnz, D] (CSR order, 1 <= D <= 16, no gradient) with edge_weight [F, D], the weight of a bias-free
    linear edge encoder, instead of edge_term: the same result as edge_term = edge_attr @ edge_weight.T, with the
    product formed inside the kernels (no [nnz, F] tensor in the forward or the backward; edge_weight gets its
    gradient).  The softmax aggregations only.
      softmax_sg  softmax with the layer's beta (tensor or float; required)
      softmax     beta = 1
      mean        beta = 0: weights 1/deg
      sum         deg * mean
      max         neighbour max of relu(x) + eps (scatter_max kernel); no edge term
      powermean   (mean of clamp(relu(x) + eps, 1e-7, 1)^p)^(1/p) (SpMM kernel); no edge term
    Degree-0 rows give 0 (max, powermean included)."""
    if aggr not in AGGRS:
        raise ValueError(f"genconv_aggregate: aggr must be one of {AGGRS}, got {aggr!r}")
    if not x.is_cuda:
        raise RuntimeError("genconv_aggregate: CUDA tensors only (no CPU fallback)")
    if x.dtype != torch.float32:
        raise TypeError(f"genconv_aggregate: x must be float32, got {x.dtype}")
    if x.dim() != 2:
        raise ValueError(f"genconv_aggregate: x must be [N, F], got {tuple(x.shape)}")
    fused_edge = _check_edge_encoder(x, edge_term, edge_attr, edge_weight)
    st = graph if isinstance(graph, CSRStructure) else graph_operands(graph).st
    if aggr in ("max", "powermean"):
        if fused_edge:
            raise NotImplementedError(f"genconv_aggregate: aggr={aggr!r} with edge_attr has no kernel")
        if edge_term is not None:
            raise NotImplementedError(f"genconv_aggregate: aggr={aggr!r} with an edge term has no kernel")
        msg = torch.relu(x) + eps
        if aggr == "max":
            return ScatterMaxFunction.apply(st, None, msg)
        deg = _degrees(st)
        inv = torch.where(deg > 0, 1.0 / deg, torch.zeros_like(deg))
        h = SPMMFunction.apply(st, None, torch.clamp(msg, 1e-7, 1.0).pow(p).contiguous(), None, False) * inv
        return h.pow(1.0 / p)
    if aggr == "softmax_sg":
        if beta is None:
            raise ValueError("genconv_aggregate: softmax_sg needs beta")
        if not torch.is_tensor(beta):
            beta = torch.full((1,), float(beta), dtype=torch.float32, device=x.device)
    else:
        beta = torch.full((1,), 1.0 if aggr == "softmax" else 0.0, dtype=torch.float32, device=x.device)
    if fused_edge:
        h = GenconvEdgeFunction.apply(st, x, edge_weight, beta, edge_attr, eps)
    else:
        h = SoftmaxAggrFunction.apply(st, x, edge_term, beta, eps)
    if aggr == "sum":
        h = h * _degrees(st)
    return h

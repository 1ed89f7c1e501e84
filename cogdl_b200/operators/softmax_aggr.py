"""GENConv aggregation (DeeperGCN / RevGCN; cogdl/layers/deepergcn_layer.py:64-93) without per-edge feature tensors.

The reference gathers x[col] into an [nnz, F] tensor, adds the edge encoder's output, applies relu + eps, runs the
edge softmax with F "heads" on beta times that, multiplies, and scatter_adds with float atomics -- several [nnz, F]
tensors per call in the forward and as many in the backward.  Here the softmax aggregations (softmax_sg, softmax,
mean = beta 0, sum = deg * mean) are one pass of cogdl_b200/csrc/softmax_aggr.cu over the CSR, with an online softmax
per channel in registers, and the backward is one pass over the cached transpose.  No [nnz, F] tensor exists unless
the caller passes an edge term (then its gradient is the only one written).  max and powermean without an edge term
go through the existing scatter_max and SpMM kernels.
"""
import torch

from ..structure import CSRStructure, graph_operands
from ._raw import softmax_aggr_bwd_raw, softmax_aggr_fwd_raw
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


def _degrees(st):
    return (st.rowptr[1:] - st.rowptr[:-1]).to(torch.float32).unsqueeze(1)


def genconv_aggregate(graph, x, aggr, beta=None, eps=1e-7, edge_term=None, p=1.0):
    """The aggregated h of CogDL's GENConv.forward before message_norm / residual / MLP.

    graph: cogdl_b200.Graph, a real cogdl.data.Graph or a CSRStructure; x [n_cols, F] fp32 CUDA; edge_term: the
    edge encoder's output [nnz, F] in CSR order (graph.edge_attr after the graph is in CSR form) or None.
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
    st = graph if isinstance(graph, CSRStructure) else graph_operands(graph).st
    if aggr in ("max", "powermean"):
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
    h = SoftmaxAggrFunction.apply(st, x, edge_term, beta, eps)
    if aggr == "sum":
        h = h * _degrees(st)
    return h

"""DisenGCN neighbourhood routing (cogdl/layers/disengcn_layer.py:40-91) without per-edge feature tensors.

The reference layer runs `iterations` routing steps, each of which builds five [E, K, d] fp32 tensors (the gathered
h_dst[row] and h_src[col], their product, the index_select and the weighted messages) plus an int64 [K, E, d] index,
and scatter_adds with float atomics; autograd keeps most of them.  Here one step is one pass of
cogdl_b200/csrc/disen_routing.cu over the CSR (online softmax per channel in registers), and its backward is a row
pass over the CSR plus a column pass over the cached transpose.  Nothing edge-sized is allocated, and forward and
backward are bitwise reproducible.
"""
import torch

from ..structure import CSRStructure, graph_operands
from ._raw import disen_route_bwd_raw, disen_route_fwd_raw

SUPPORTED_D = (1, 2, 4, 8, 16, 32)


class DisenRouteFunction(torch.autograd.Function):
    """One routing step out = normalize(sum_e softmax_e(q_i . c_j / tau) c_j + c_i) per channel, with gradients for
    q and c.  Chained by autograd over the iterations; c's gradient accumulates from every step."""

    @staticmethod
    def forward(ctx, st, q, c, K, tau):
        train = ctx.needs_input_grad[1] or ctx.needs_input_grad[2]
        out, lse2, r = disen_route_fwd_raw(st, q, c, K, tau, want_saved=train)
        ctx.st, ctx.K, ctx.tau = st, int(K), float(tau)
        ctx.save_for_backward(q, c, out, lse2, r)
        return out

    @staticmethod
    def backward(ctx, g):
        q, c, out, lse2, r = ctx.saved_tensors
        dq, dc = disen_route_bwd_raw(ctx.st, q, c, ctx.K, ctx.tau, g.contiguous(), out, lse2, r)
        return None, dq if ctx.needs_input_grad[1] else None, dc if ctx.needs_input_grad[2] else None, None, None


def disen_routing(graph, h, K, iterations, tau=1.0):
    """The output of CogDL's DisenGCNLayer.forward given h = act(x W + b): h [N, F] is cut into K channels of
    d = F / K columns, each normalised to unit length (c), and `iterations` routing steps run from q = c.  Returns
    [N, F] in h's column layout.  graph: cogdl_b200.Graph, a real cogdl.data.Graph or a CSRStructure, square.
    d must be a power of two from 1 to 32 and tau > 0.  A zero channel of h, or of a step's u, gives NaN as in the
    reference (no epsilon)."""
    if not h.is_cuda:
        raise RuntimeError("disen_routing: CUDA tensors only (no CPU fallback)")
    if h.dtype != torch.float32:
        raise TypeError(f"disen_routing: h must be float32, got {h.dtype}")
    if h.dim() != 2:
        raise ValueError(f"disen_routing: h must be [N, F], got {tuple(h.shape)}")
    N, F = h.shape
    if K < 1 or F % K:
        raise ValueError(f"disen_routing: F={F} is not a multiple of K={K}")
    st = graph if isinstance(graph, CSRStructure) else graph_operands(graph).st
    hk = h.reshape(N, K, F // K)
    c = (hk / hk.pow(2).sum(-1, keepdim=True).sqrt()).reshape(N, F)
    q = c
    for _ in range(iterations):
        q = DisenRouteFunction.apply(st, q, c, K, tau)
    return q

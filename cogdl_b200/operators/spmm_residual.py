"""spmm_residual -- `a * spmm(graph, x) + b * z` in one SpMM launch (the propagation step of GCNII and APPNP).

The reference computes it as `(1 - alpha) * spmm(graph, x) + alpha * init_x` (cogdl/layers/gcnii_layer.py:24-30,
cogdl/models/nn/ppnp.py:77-83): the SpMM, then the graph's in_norm, then three elementwise passes over [N, F].  Here
the scaling, the in_norm and the addition run in the SpMM's store (cogdl_b200_spmm_residual_f32), with the same fp32
roundings in the same order, so the forward is bit-identical to that sequence run with this package's spmm."""
import torch

from ..structure import graph_operands, unsupported_operands
from ._raw import sddmm_raw, spmm_adjoint_raw, spmm_residual_raw


class SpmmResidualFunction(torch.autograd.Function):
    """out = a * (r * (A @ x)) + b * z.  Backward: d x = a * (A^T @ (r * g)) through the same kernel (A itself when
    `sym`, as SPMMFunction does, else the cached transpose), d z = b * g, and d val = SDDMM(a * r * g, x) when the edge
    weights require grad."""

    @staticmethod
    def forward(ctx, st, x, z, val, a, b, row_scale, sym):
        out = spmm_residual_raw(st, val, x, z, a, b, row_scale)
        ctx.st, ctx.a, ctx.b, ctx.sym = st, a, b, bool(sym)
        need_w = val is not None and val.requires_grad
        ctx.save_for_backward(val, x if need_w else None, row_scale)
        return out

    @staticmethod
    def backward(ctx, g):
        val, x, r = ctx.saved_tensors
        st = ctx.st
        g = g.contiguous()
        gr = g if r is None else r.view(-1, 1) * g
        dx = dz = dval = None
        if ctx.needs_input_grad[1]:
            dx = spmm_adjoint_raw(st, val, gr, ctx.sym, ctx.a)
        if ctx.needs_input_grad[2]:
            dz = ctx.b * g
        if val is not None and ctx.needs_input_grad[3]:
            dval = sddmm_raw(st, ctx.a * gr, x)
        return None, dx, dz, dval, None, None, None, None


def spmm_residual(graph, x, z, a, b):
    """a * spmm(graph, x) + b * z (z may be None) for fp32 CUDA tensors, in one SpMM launch.  The graph is taken as
    cogdl_b200.spmm takes it: the cached int32 CSR and hub plan, out_norm applied to x first, in_norm applied to the
    SpMM's rows (here inside the kernel), and the backward over A when graph.is_symmetric(), else over the cached
    transpose.  The result is bit-identical to `a * spmm(graph, x) + b * z` computed by this package."""
    err = unsupported_operands(graph, x, z, entry="spmm_residual")
    if err is not None:
        raise err
    st, val, out_norm, r, sym = graph_operands(graph)
    if out_norm is not None:
        x = out_norm.to(x.device) * x
    if r is not None:
        if r.requires_grad:
            raise ValueError("spmm_residual: an in_norm that requires grad is not supported")
        r = r.to(x.device).reshape(-1)
    return SpmmResidualFunction.apply(st, x, z, val, float(a), float(b), r, sym)

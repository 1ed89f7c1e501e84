"""spmm_residual -- `a * spmm(graph, x) + b * z` in one SpMM launch (the propagation step of GCNII and APPNP).

The reference computes it as `(1 - alpha) * spmm(graph, x) + alpha * init_x` (cogdl/layers/gcnii_layer.py:24-30,
cogdl/models/nn/ppnp.py:77-83): the SpMM, then the graph's in_norm, then three elementwise passes over [N, F].  Here
the scaling, the in_norm and the addition run in the SpMM's store (cogdl_b200_spmm_residual_f32), with the same fp32
roundings in the same order, so the forward is bit-identical to that sequence run with this package's spmm."""
import torch

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
    from ..utils.spmm_utils import _structure

    if getattr(graph, "grb_adj", None) is not None:
        raise ValueError("spmm_residual: graphs carrying a dense grb_adj are not supported; use spmm")
    if not x.is_cuda:
        raise RuntimeError("cogdl_b200.spmm_residual: CPU tensors are not supported (no CPU fallback); move the graph "
                           "and features to an H100 device")
    if x.dtype != torch.float32 or (z is not None and z.dtype != torch.float32):
        raise TypeError(f"spmm_residual takes float32 features, got {x.dtype}"
                        f"{'' if z is None else ' and ' + str(z.dtype)}")
    # the structure first: building the CSR of a graph held as COO puts its edge weights in CSR order
    st = _structure(graph)
    if graph.out_norm is not None:
        x = graph.out_norm.to(x.device) * x
    r = graph.in_norm
    if r is not None:
        if r.requires_grad:
            raise ValueError("spmm_residual: an in_norm that requires grad is not supported")
        r = r.to(x.device).reshape(-1)
    val = graph.raw_edge_weight
    return SpmmResidualFunction.apply(st, x, z, val, float(a), float(b), r, graph.is_symmetric())

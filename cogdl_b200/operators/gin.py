"""gin_aggregate -- GIN's `(1 + eps) * x + spmm(graph, x)` in one SpMM launch, forward and backward.

The reference (cogdl/layers/gin_layer.py:35, gine_layer.py:33-34) computes one SpMM and three eager passes over [N, F]
in the forward, and about as many in the backward.  Here the scaling by 1 + eps and the addition run in the SpMM's store
(cogdl_b200_spmm_residual_dcoef_f32), which reads 1 + eps on the device, so a trainable eps costs no host
synchronisation.  With a = 1 the epilogue rounds as the reference expression does (fp32 addition commutes), so the
forward and the feature gradient are bit-identical to autograd through that expression on this package's spmm."""
import torch

from ..structure import graph_operands, unsupported_operands
from ._raw import gather_rows_raw, sddmm_raw, spmm_adjoint_raw, spmm_residual_dcoef_raw


def _adjoint_dcoef(st, val, gr, g, b_dev, sym):
    """A^T @ gr + b * g in one launch, over A itself when sym, else over the cached transpose."""
    if not sym:
        st, perm = st.csc()
        val = None if val is None else gather_rows_raw(perm, val.detach().float())
    return spmm_residual_dcoef_raw(st, val, gr, g, 1.0, b_dev)


class GinAggregateFunction(torch.autograd.Function):
    """out = r * (A @ xg) + b * z, with b = one_plus_eps[0] read on the device and z = xg unless given (the graph's
    out_norm makes xg = out_norm * x while z stays x).  Backward: with z = xg, d xg = A^T (r g) + b g in one launch of
    the same entry over the adjoint; with a separate z, d xg = A^T (r g) and d z = b * g.  d b = (g * z).sum(), as
    torch's mul backward computes it; d val = SDDMM(r g, xg) when the edge weights require grad."""

    @staticmethod
    def forward(ctx, st, xg, z, one_plus_eps, val, row_scale, sym):
        out = spmm_residual_dcoef_raw(st, val, xg, xg if z is None else z, 1.0, one_plus_eps, row_scale)
        ctx.st, ctx.sym, ctx.fused = st, bool(sym), z is None
        need_w = val is not None and val.requires_grad
        need_b = one_plus_eps.requires_grad
        ctx.save_for_backward(val, xg if (need_w or (need_b and z is None)) else None,
                              z if need_b else None, one_plus_eps, row_scale)
        return out

    @staticmethod
    def backward(ctx, g):
        val, xg, z, b, r = ctx.saved_tensors
        st = ctx.st
        g = g.contiguous()
        gr = g if r is None else r.view(-1, 1) * g
        dxg = dz = db = dval = None
        if ctx.needs_input_grad[1]:
            if ctx.fused:
                dxg = _adjoint_dcoef(st, val, gr, g, b, ctx.sym)
            else:
                dxg = spmm_adjoint_raw(st, val, gr, ctx.sym)
        if ctx.needs_input_grad[2]:
            dz = b * g
        if ctx.needs_input_grad[3]:
            db = (g * (xg if ctx.fused else z)).sum().reshape(b.shape)
        if val is not None and ctx.needs_input_grad[4]:
            dval = sddmm_raw(st, gr, xg)
        return None, dxg, dz, db, dval, None, None


def gin_aggregate(graph, x, eps):
    """(1 + eps) * x + spmm(graph, x) for fp32 CUDA x [N, F] on a square graph, in one SpMM launch.  eps is a
    one-element fp32 tensor on x's device (GIN's parameter or buffer; 1 + eps is formed by torch, so a trainable eps
    gets its gradient through autograd) or a Python number.  The graph is taken as cogdl_b200.spmm takes it: the cached
    int32 CSR and hub plan, out_norm applied to the gathered x, in_norm to the SpMM's rows (here inside the kernel),
    and the backward over A when graph.is_symmetric(), else over the cached transpose.  The result and d x are
    bit-identical to `(1 + eps) * x + cogdl_b200.spmm(graph, x)` and its autograd; no host synchronisation."""
    eps_t = eps if torch.is_tensor(eps) else None
    err = unsupported_operands(graph, x, eps_t, entry="gin_aggregate")
    if err is not None:
        raise err
    if eps_t is not None and eps_t.numel() != 1:
        raise ValueError(f"gin_aggregate: eps must hold one value, got {eps_t.numel()}")
    st, val, out_norm, r, sym = graph_operands(graph)
    if x.dim() != 2 or x.shape[0] != st.n_rows or st.n_cols != st.n_rows:
        raise ValueError(f"x must be [{st.n_rows}, F] on a square graph, got {tuple(x.shape)}")
    if eps_t is not None:
        one_plus = (1 + eps_t).reshape(1)
    else:   # `(1 + eps) * x` with a Python eps multiplies by 1 + eps rounded to fp32
        one_plus = torch.full((1,), 1 + eps, dtype=torch.float32, device=x.device)
    z = None
    if out_norm is not None:
        z, x = x, out_norm.to(x.device) * x
    if r is not None:
        if r.requires_grad:
            raise ValueError("gin_aggregate: an in_norm that requires grad is not supported")
        r = r.to(x.device).reshape(-1)
    return GinAggregateFunction.apply(st, x, z, one_plus, val, r, sym)

"""random_propagate -- GRAND's propagation after DropNode, one SpMM launch per hop.

The reference (cogdl/models/nn/grand.py:98-104, Grand.rand_prop) runs, after drop_node,

    y = x
    for i in range(order):
        x = spmm(graph, x).detach_()
        y.add_(x)
    return y.div_(order + 1.0).detach_()

one SpMM, one read-modify-write pass of y per hop and a last pass for the division: 2 * order + 1 launches.  Here each
hop is one cogdl_b200_spmm_accum_f32 launch, which adds the hop's rows to the running sum in the SpMM's store and, on
the last hop, scales it as `div_` does on CUDA (a multiply by the fp32 reciprocal of the host scalar), so the result is
bit-identical to that loop run with this package's spmm.  The hops ping-pong between two buffers, with no host
synchronisation between them.

The fused hop is used where it was measured to be faster: rows of at most FUSED_MAX_F floats, a multiple of 4, on a
16-byte aligned x, which the SpMM runs with one vector per lane (the lean row-stream loops, DESIGN 3.16).  Wider or
scalar rows take the SpMM's multi-vector loop, where the accumulating store made each hop up to 2x slower than the
SpMM plus `add_` on the Cora and PubMed shapes (H100, 700 W), so there random_propagate runs the reference loop itself
on this package's spmm: same kernels for the SpMM, same result bits."""
import numpy as np
import torch

from ..structure import graph_operands, unsupported_operands
from ._raw import spmm_accum_raw


def div_scale(order):
    """The fp32 factor `y.div_(order + 1.0)` multiplies a CUDA tensor by: 1 / (order + 1) rounded to fp32, as torch's
    division by a host scalar computes it."""
    return float(np.float32(1.0) / np.float32(order + 1.0))


FUSED_MAX_F = 128


def fused_hops(x):
    """True when the hops of x run as cogdl_b200_spmm_accum_f32 launches (see the module notes)."""
    F = x.shape[1]
    return F <= FUSED_MAX_F and F % 4 == 0 and x.data_ptr() % 16 == 0


def _reference_loop(graph, x, order):
    """The reference's loop on this package's spmm, with its first `add_` out of place so x is left as it is."""
    from ..utils.spmm_utils import spmm

    h = spmm(graph, x)
    y = torch.add(x, h)
    for _ in range(order - 1):
        h = spmm(graph, h)
        y.add_(h)
    return y.div_(order + 1.0)


def random_propagate(graph, x, order):
    """Grand.rand_prop after drop_node, for fp32 CUDA x [N, F] on a square graph: (x + A x + ... + A^order x) /
    (order + 1), with A applied as cogdl_b200.spmm applies the graph (its CSR, edge weights, out_norm and in_norm).
    One launch per hop for rows the fused hop serves (fused_hops), else the reference loop on this package's spmm.
    Forward only: the result is detached, as the reference's.  order = 0 returns x detached (a view of x, as the
    reference returns x itself, divided by 1.0 in place)."""
    err = unsupported_operands(graph, x, entry="random_propagate")
    if err is not None:
        raise err
    order = int(order)
    if order < 0:
        raise ValueError(f"order must be >= 0, got {order}")
    if order == 0:
        return x.detach()
    st, val, out_norm, r, _ = graph_operands(graph)
    if x.dim() != 2 or x.shape[0] != st.n_rows or st.n_cols != st.n_rows:
        raise ValueError(f"x must be [{st.n_rows}, F] on a square graph, got {tuple(x.shape)}")
    with torch.no_grad():
        x = x.detach().contiguous()
        if not fused_hops(x):
            return _reference_loop(graph, x, order)
        val = None if val is None else val.detach()
        out_norm = None if out_norm is None else out_norm.to(x.device)
        r = None if r is None else r.to(x.device).reshape(-1)
        acc = torch.empty_like(x)
        bufs = (torch.empty_like(x), torch.empty_like(x)) if order > 1 else (None, None)
        scale = div_scale(order)
        h = x
        for k in range(1, order + 1):
            if out_norm is not None:
                h = out_norm * h
            last = k == order
            h = spmm_accum_raw(st, val, h, acc, acc_in=x if k == 1 else None, row_scale=r, last=last, scale=scale,
                               xn=None if last else bufs[k & 1])
    return acc

"""Graph-level readouts: pool each graph's node rows of a batch of graphs into one row per graph, forward and backward,
on the membership CSR of the batch vector (structure.membership_for: row g is graph g, its columns are g's nodes).

    batch_sum_pooling(x, batch)     cogdl/utils/utils.py:192    the row-stream SpMM with unit weights
    batch_mean_pooling(x, batch)    cogdl/utils/utils.py:199    the same SpMM, times 1 / n_g in its store
    batch_max_pooling(x, batch)     cogdl/utils/utils.py:206    scatter_max over the membership CSR
    graph_readout(xs, batch, mode)  GIN / InfoGraph: one of the three over a list of per-layer tensors
    set2set_attention(x, q, batch)  the attention read of Set2Set (cogdl/layers/set2set.py:56-60)
    sort_pool(h, batch, k)          the padding, sorting and cutting of SortPool (cogdl/models/nn/sortpool.py:108-126)

Every reduction is the plan-balanced kernel of its family with the chunk-order merge of hub rows, so the results are
bit-identical run to run (the reference's scatter_add_ has CUDA atomics), and none reads the host once the batch's
membership is cached (the reference reads max(batch), torch.unique or a CSR on the host per call).  Graph ids without
nodes are empty rows: 0 for every readout.  The backward of each runs over the membership's transpose, one edge per
node, so the sum's d x is dy[batch] bit for bit.

The mean applies 1 / n_g as a row scale in the SpMM's store, fl(fl(1 / n_g) * s), where the reference divides, fl(s /
n_g): relative to the exact quotient s / n_g the row scale's rounding error is at most 2^-23 + 2^-48, the division's
2^-24."""
import torch

from ..structure import membership_for, require_cuda
from ._raw import (edge_softmax_bwd_raw, edge_softmax_fwd_raw, scatter_max_bwd_raw, scatter_max_fwd_raw, sddmm_raw,
                   sort_pool_select_raw, spmm_adjoint_raw, spmm_raw, spmm_residual_raw)

READOUT_MODES = ("sum", "mean", "max")


def _check(x, batch, name="x"):
    require_cuda(x, batch)
    if x.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {x.dtype}")
    if x.dim() != 2 or x.shape[0] != batch.numel():
        raise ValueError(f"{name} must be [N = {batch.numel()}, F], got {tuple(x.shape)}")


class ReadoutFunction(torch.autograd.Function):
    """One readout of x [N, F] over a Membership mb: "sum" and "mean" are SpMMs over mb.st (the mean with the row scale
    mb.inv_count), "max" is scatter_max.  Backward: SpMMs over mb.st_t (the mean with the per-node weight
    mb.inv_count_node), and scatter_max's backward, whose argmax names each node at most once here."""

    @staticmethod
    def forward(ctx, x, mb, mode):
        ctx.mb, ctx.mode, ctx.n = mb, mode, x.shape[0]
        if mode == "sum":
            return spmm_raw(mb.st, None, x)
        if mode == "mean":
            return spmm_residual_raw(mb.st, None, x, None, 1.0, 0.0, row_scale=mb.inv_count)
        out, arg = scatter_max_fwd_raw(mb.st, x)
        ctx.save_for_backward(arg)
        return out

    @staticmethod
    def backward(ctx, g):
        mb, g = ctx.mb, g.contiguous()
        if ctx.mode == "sum":
            dx = spmm_adjoint_raw(mb.st, None, g, False)
        elif ctx.mode == "mean":
            dx = spmm_raw(mb.st_t, mb.inv_count_node, g)
        else:
            dx = scatter_max_bwd_raw(g, ctx.saved_tensors[0], ctx.n)
        return dx, None, None


def _pool(x, batch, mode, num_graphs):
    _check(x, batch)
    return ReadoutFunction.apply(x, membership_for(batch, num_graphs), mode)


def batch_sum_pooling(x, batch, num_graphs=None):
    """[B, F]: the sum of each graph's rows of x [N, F]; B = num_graphs, or max(batch) + 1."""
    return _pool(x, batch, "sum", num_graphs)


def batch_mean_pooling(x, batch, num_graphs=None):
    """[B, F]: the mean of each graph's rows of x (0 for a graph without nodes); see the module note on rounding."""
    return _pool(x, batch, "mean", num_graphs)


def batch_max_pooling(x, batch, num_graphs=None):
    """[B, F]: the column maxima of each graph's rows of x, with scatter_max's rules (DESIGN.md 3.5, 3.20): a strict `<`
    from -inf in node order, so ties go to the first node, a NaN is never selected and a column of NaN alone gives
    -inf; an empty graph gives 0.  The gradient goes to the selected node."""
    return _pool(x, batch, "max", num_graphs)


def graph_readout(xs, batch, mode="sum", num_graphs=None):
    """[B, sum of the widths]: the readout `mode` ("sum", "mean" or "max") of every tensor of xs, each [N, F_l], side by
    side in list order, over one membership.  The SpMM's store takes no row stride, so the pooled blocks are joined with
    torch.cat."""
    if mode not in READOUT_MODES:
        raise ValueError(f"unknown readout {mode!r} (one of {READOUT_MODES})")
    if len(xs) == 0:
        raise ValueError("graph_readout needs at least one tensor")
    for x in xs:
        _check(x, batch)
    mb = membership_for(batch, num_graphs)
    return torch.cat([ReadoutFunction.apply(x, mb, mode) for x in xs], dim=1)


class Set2SetAttentionFunction(torch.autograd.Function):
    """r = SpMM(a, x) with a = edge_softmax(e), e = SDDMM(q, x), over the membership CSR: r[g] = sum over g's nodes i of
    a_i x_i, a = softmax over g's nodes of <x_i, q_g>.  Saved: x, q and a ([N], one value per node).  Backward:
    d a = SDDMM(dr, x), d e = the edge-softmax backward, d q = SpMM(d e, x) and d x = A^T(a) dr + A^T(d e) q over the
    membership's transpose."""

    @staticmethod
    def forward(ctx, x, q, mb):
        st = mb.st
        e = sddmm_raw(st, q, x)
        a = edge_softmax_fwd_raw(st, e.view(-1, 1)).view(-1)
        ctx.mb = mb
        ctx.save_for_backward(x, q, a)
        return spmm_raw(st, a, x)

    @staticmethod
    def backward(ctx, dr):
        x, q, a = ctx.saved_tensors
        st, dr = ctx.mb.st, dr.contiguous()
        da = sddmm_raw(st, dr, x)
        de = edge_softmax_bwd_raw(st, a.view(-1, 1), da.view(-1, 1)).view(-1)
        dx = dq = None
        if ctx.needs_input_grad[1]:
            dq = spmm_raw(st, de, x)
        if ctx.needs_input_grad[0]:
            dx = spmm_adjoint_raw(st, a, dr, False)
            dx += spmm_adjoint_raw(st, de, q, False)
        return dx, dq, None


def set2set_attention(x, q, batch, num_graphs=None):
    """r [B, F] of one Set2Set step: r_g = sum over g's nodes of softmax_i(<x_i, q_g>) x_i, for x [N, F] and the LSTM's
    query q [B, F], B = num_graphs or max(batch) + 1.  An empty graph gives 0."""
    _check(x, batch)
    require_cuda(q)
    mb = membership_for(batch, num_graphs)
    if q.dtype != torch.float32 or q.shape != (mb.num_graphs, x.shape[1]):
        raise ValueError(f"q must be float32 [{mb.num_graphs}, {x.shape[1]}], got {q.dtype} {tuple(q.shape)}")
    return Set2SetAttentionFunction.apply(x, q, mb)


class SortPoolFunction(torch.autograd.Function):
    """cogdl_b200_sort_pool_select picks the rows by the last channel's bits; the pooled rows are the SpMM over its
    selection CSR with unit weights (one fp32 addition to 0 per element: -0 comes out as +0, and NaN as the canonical
    NaN).  Saved: the selected node of every output row ([B, k] int32, -1 for padding); the backward scatters dy
    through it with scatter_max's backward, whose targets are distinct here."""

    @staticmethod
    def forward(ctx, h, mb, k):
        h = h.contiguous()
        idx, sel = sort_pool_select_raw(mb.st, h[:, -1], k)
        ctx.n = h.shape[0]
        ctx.save_for_backward(idx)
        return spmm_raw(sel, None, h).view(mb.num_graphs, k, h.shape[1])

    @staticmethod
    def backward(ctx, g):
        (idx,) = ctx.saved_tensors
        B, k, F = g.shape
        arg = idx.view(B * k, 1).expand(B * k, F).contiguous()
        return scatter_max_bwd_raw(g.reshape(B * k, F), arg, ctx.n), None, None


def sort_pool(h, batch, k, num_graphs=None):
    """[B, k, F]: for each graph, its k rows of h [N, F] with the largest last channel, in descending order; ties go to
    the lower node index and NaN sorts above +inf (torch.sort(descending=True), stable); rows past the graph's node
    count are 0.  1 <= k <= sort_pool_max_k() (1024)."""
    _check(h, batch, "h")
    return SortPoolFunction.apply(h, membership_for(batch, num_graphs), k)

"""fp64 numpy restatements of the graph-level readouts (cogdl_b200.operators.readout) and their gradients.  `batch` is
an [N] integer array (node i in graph batch[i]), B the graph count; a graph's nodes are taken in ascending order."""
import numpy as np
import scipy.sparse as sp


def members(batch, B):
    """The node list of every graph, ascending (the membership CSR's rows)."""
    order = np.argsort(batch, kind="stable")
    bounds = np.searchsorted(batch[order], np.arange(B + 1))
    return [order[bounds[g]:bounds[g + 1]] for g in range(B)]


def sum_pool(x, batch, B):
    M = sp.csr_matrix((np.ones(len(batch)), (batch, np.arange(len(batch)))), shape=(B, len(batch)))
    return np.asarray(M @ x.astype(np.float64))


def sum_pool_grad(dy, batch):
    return dy.astype(np.float64)[batch]


def counts(batch, B):
    return np.bincount(batch, minlength=B).astype(np.float64)


def mean_pool(x, batch, B):
    n = counts(batch, B)
    return sum_pool(x, batch, B) / np.maximum(n, 1)[:, None]


def mean_pool_grad(dy, batch, B):
    return dy.astype(np.float64)[batch] / counts(batch, B)[batch][:, None]


def max_pool(x, batch, B):
    """(out [B, F], arg [B, F]) by scatter_max's rules: a strict `<` from -inf in node order (ties to the first node, NaN
    never selected; a column of NaN alone gives -inf, arg -1); an empty graph gives 0, arg -1."""
    F = x.shape[1]
    out, arg = np.zeros((B, F)), np.full((B, F), -1, np.int64)
    for g, nodes in enumerate(members(batch, B)):
        if len(nodes) == 0:
            continue
        out[g] = -np.inf
        for i in nodes:
            v = x[i].astype(np.float64)
            take = out[g] < v
            out[g, take], arg[g, take] = v[take], i
    return out, arg


def max_pool_grad(dy, arg, N):
    dx = np.zeros((N, dy.shape[1]))
    g, f = np.nonzero(arg >= 0)
    dx[arg[g, f], f] = dy[g, f]
    return dx


def set2set(x, q, batch, B):
    """(r [B, F], a [N]): a_i = softmax over graph g's nodes of <x_i, q_g>, r_g = sum_i a_i x_i."""
    x, q = x.astype(np.float64), q.astype(np.float64)
    e = (x * q[batch]).sum(1)
    a = np.zeros(len(batch))
    for nodes in members(batch, B):
        if len(nodes):
            w = np.exp(e[nodes] - e[nodes].max())
            a[nodes] = w / w.sum()
    return sum_pool(a[:, None] * x, batch, B), a


def set2set_grad(x, q, batch, B, dr):
    """(dx, dq) of set2set for the upstream gradient dr [B, F]."""
    x, q, dr = x.astype(np.float64), q.astype(np.float64), dr.astype(np.float64)
    _, a = set2set(x, q, batch, B)
    da = (dr[batch] * x).sum(1)
    s = np.zeros(B)
    np.add.at(s, batch, a * da)
    de = a * (da - s[batch])
    dq = sum_pool(de[:, None] * x, batch, B)
    dx = a[:, None] * dr[batch] + de[:, None] * q[batch]
    return dx, dq


def sort_pool(h, batch, B, k):
    """(out [B, k, F], idx [B, k]): per graph its k rows with the largest last channel, descending, ties to the lower
    node index, NaN above +inf (a stable torch.sort(descending=True)); padding rows 0 with idx -1."""
    F = h.shape[1]
    out, idx = np.zeros((B, k, F)), np.full((B, k), -1, np.int64)
    for g, nodes in enumerate(members(batch, B)):
        key = h[nodes, -1].astype(np.float64)
        nan = np.isnan(key)
        order = nodes[np.lexsort((nodes, -np.where(nan, 0.0, key), ~nan))][:k]
        idx[g, :len(order)] = order
        out[g, :len(order)] = h[order]
    return out, idx


def sort_pool_grad(dy, idx, N):
    dx = np.zeros((N, dy.shape[2]))
    g, r = np.nonzero(idx >= 0)
    dx[idx[g, r]] = dy[g, r]
    return dx

"""An fp64 restatement of R-GCN's basis layer (cogdl/layers/rgcn_layer.py) as the reference's loop was written to
compute it, and of what the reference computes instead.  Torch fp64 on the host, autograd-capable.

  relational sum:  sum_t A_t x W_t, W_t = sum_b alpha[t, b] V_b, A_t[i, j] = sum of w_hat over the type-t edges i -> j
  first present:   A x W_f with A over every edge and f the smallest type that has an edge (the reference's
                   `return h_list` inside its loop, with spmm over the whole graph)

w_hat is the row-normalised edge weight, w / (number of edges of the row), as graph.row_norm() gives it on a graph
held as COO."""
import torch


def row_norm_weights(row, n, w=None):
    """w / deg(row) in fp64 (w = 1 when None)."""
    row = torch.as_tensor(row, dtype=torch.int64)
    w = torch.ones(row.numel(), dtype=torch.float64) if w is None else torch.as_tensor(w, dtype=torch.float64)
    deg = torch.zeros(n, dtype=torch.float64).index_add_(0, row, torch.ones_like(w))
    return w / deg[row]


def type_weights(alpha, V, T):
    """W [T, F_in, F_out] = alpha @ V (alpha None: V itself, num_bases >= T)."""
    if alpha is None:
        return V
    B = V.shape[0]
    return (alpha @ V.reshape(B, -1)).reshape(T, V.shape[1], V.shape[2])


def relational_sum(row, col, etype, w_hat, x, W):
    """sum_t A_t x W_t in fp64: per edge, w_hat * (x[col] @ W[type]) summed into its row."""
    row, col, etype = (torch.as_tensor(t, dtype=torch.int64) for t in (row, col, etype))
    msg = torch.einsum("ef,efo->eo", x[col], W[etype]) * w_hat.view(-1, 1)
    return torch.zeros(x.shape[0], W.shape[2], dtype=msg.dtype).index_add_(0, row, msg)


def first_present(row, col, etype, w_hat, x, W):
    """What the reference layer aggregates for any T: every edge with the W of the smallest type present."""
    f = int(torch.as_tensor(etype).min())
    return relational_sum(row, col, torch.full_like(torch.as_tensor(etype, dtype=torch.int64), f), w_hat, x, W)


def layer_post(h, x, p, ln_eps=1e-5):
    """The reference layer's tail without dropout: layer_norm, bias, + x @ weight_self_loop."""
    if "layer_norm.weight" in p:
        h = torch.nn.functional.layer_norm(h, (h.shape[1],), p["layer_norm.weight"], p["layer_norm.bias"], ln_eps)
    if "bias" in p:
        h = h + p["bias"]
    return h + x @ p["weight_self_loop"]


def rgcn_layer_fp64(p, row, col, etype, w_hat, x, T):
    """One RGCNLayer (basis, self loop, no dropout) computing the relational sum; p maps parameter names to fp64."""
    W = type_weights(p.get("alpha"), p["weight"], T)
    return layer_post(relational_sum(row, col, etype, w_hat, x, W), x, p)

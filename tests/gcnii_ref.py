"""fp64 restatement of the reference GCNII (cogdl/models/nn/gcnii.py:111-125 with GCNIILayer,
cogdl/layers/gcnii_layer.py:24-30) and PPNP with "appnp" propagation (cogdl/models/nn/ppnp.py:56-87), in eval mode
(dropout off), as the reference graph normalises itself:

- CSR-built graph (no edge_index given): sym_norm() keeps the unit edge weights and sets in_norm = out_norm = deg^-1/2
  (data.py:240-252, deg = entries per CSR row, inf -> 0); spmm(graph, x) = in_norm * (A @ (out_norm * x)).
- edge_index-built graph: sym_norm() rescales the weights to w_e = deg[col]^-1/2 * deg[row]^-1/2 (graph_utils.py:82-89,
  deg = entries per row) and sets no row norms.
- APPNP assigns the (dropped-out) edge weights inside local_graph(), and set_weight clears in_norm / out_norm
  (data.py:150-154): its propagation uses the graph's current edge weights only -- the unit weights of a CSR-built
  graph, the normalised ones of an edge_index-built graph.

Parameters come as a {name: tensor} dict of the model's named_parameters(); the result is built from fp64 leaves
so that gradients of every parameter follow from one backward."""
import math

import numpy as np
import torch


def csr_rows(rp):
    rp = np.asarray(rp, np.int64)
    return np.repeat(np.arange(rp.shape[0] - 1), np.diff(rp))


def propagation(rp, col, built_from, model):
    """(A [n, n] fp64 sparse, in_norm [n, 1] or None, out_norm [n, 1] or None) of spmm(graph, .) in the model's
    forward, for a graph built from "csr" or "coo" (edge_index, given in CSR order)."""
    rows = csr_rows(rp)
    col = np.asarray(col, np.int64)
    n = np.asarray(rp).shape[0] - 1
    deg = np.bincount(rows, minlength=n).astype(np.float64)
    dinv = np.where(deg > 0, deg ** -0.5, 0.0)
    if built_from == "csr":
        w = np.ones(col.shape[0])
        norm = torch.from_numpy(dinv).view(-1, 1)
        in_norm, out_norm = (None, None) if model == "appnp" else (norm, norm)
    else:
        w = dinv[col] * dinv[rows]
        in_norm = out_norm = None
    A = torch.sparse_coo_tensor(torch.from_numpy(np.stack([rows, col])), torch.from_numpy(w), (n, n)).coalesce()
    return A, in_norm, out_norm


def spmm64(A, in_norm, out_norm, x):
    if out_norm is not None:
        x = out_norm * x
    y = torch.sparse.mm(A, x)
    return y if in_norm is None else in_norm * y


def leaves(params):
    return {k: torch.as_tensor(np.asarray(v)).double().requires_grad_(True) for k, v in params.items()}


def gcnii_fp64(p, A, in_norm, out_norm, x, n_layers, alpha, lmbda, residual):
    lin = lambda h, pre: h @ p[pre + ".weight"].t() + p[pre + ".bias"]  # noqa: E731
    h0 = torch.relu(lin(x, "fc_layers.0"))
    h = h0
    for i in range(n_layers):
        beta = math.log(lmbda / (i + 1) + 1)
        hid = spmm64(A, in_norm, out_norm, h)
        hid = (1 - alpha) * hid + alpha * h0
        out = beta * lin(hid, f"layers.{i}.linear") + (1 - beta) * hid
        if residual:
            out = out + h
        h = torch.relu(out)
    return lin(h, "fc_layers.1")


def appnp_fp64(p, A, x, n_mlp_layers, alpha, niter):
    h = x
    for i in range(n_mlp_layers):
        h = h @ p[f"nn.nn.mlp.{i}.weight"].t() + p[f"nn.nn.mlp.{i}.bias"]
        if i < n_mlp_layers - 1:
            h = torch.relu(h)
    local = h
    preds = local
    for _ in range(niter):
        preds = (1 - alpha) * torch.sparse.mm(A, preds) + alpha * local
    return preds

#!/usr/bin/env python
"""Generate tests/golden/disengcn.npz by running the REFERENCE's own DisenGCNLayer (cogdl/layers/disengcn_layer.py)
on CPU.  Run where the reference checkout exists, after oracle/build_ref.py:   python tests/golden/make_golden_disengcn.py

Cases (K, d, iterations, tau) below, on one square graph without self loops (DisenGCN.forward removes them) that has
degree-0 rows.  Every routing logit is a dot of two unit vectors over tau, so |logit| <= 1/tau; the reference's CPU
edge softmax halves logits above 10, and 1/tau stays below that (asserted).  Stored per case: W, b (a random bias,
so it is exercised) and the layer's output; the graph (CSR) and x once.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import import_reference  # noqa: E402

CASES = [(16, 4, 7, 1.0), (8, 8, 7, 1.0), (4, 16, 3, 0.5), (8, 2, 2, 2.0)]
IN_FEATS = 24


def case_key(K, d, T, tau):
    return f"K{K}_d{d}_T{T}_tau{tau:g}"


def main():
    Graph = import_reference()[0]
    from cogdl.layers import DisenGCNLayer

    n, e = 60, 420
    g = torch.Generator().manual_seed(11)
    row, col = torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g)
    keep = (row >= 3) & (row != col)     # rows 0-2 without edges: degree-0 rows; no self loops
    row, col = row[keep], col[keep]
    x = torch.randn(n, IN_FEATS, generator=g)
    out = {"x": x.numpy()}
    for K, d, T, tau in CASES:
        assert 1.0 / tau <= 10.0, "logits up to 1/tau must stay where the reference's CPU softmax is exact"
        graph = Graph(x=x, edge_index=(row, col))
        graph.row_indptr                 # CSR order before the forward reads edge_index
        torch.manual_seed(K * 100 + d)
        layer = DisenGCNLayer(IN_FEATS, K * d, K, T, tau=tau)
        with torch.no_grad():
            layer.bias.copy_(0.1 * torch.randn(K * d, generator=g))
            y = layer(graph, x)
        key = case_key(K, d, T, tau)
        out["W_" + key] = layer.weight.detach().numpy()
        out["b_" + key] = layer.bias.detach().numpy()
        out["out_" + key] = y.numpy()
        out.setdefault("rowptr", graph.row_indptr.numpy())
        out.setdefault("colind", graph.col_indices.numpy())
    np.savez_compressed(os.path.join(HERE, "disengcn.npz"), **out)
    print(f"wrote disengcn.npz: {sorted(k for k in out if k.startswith('out_'))}")


if __name__ == "__main__":
    main()

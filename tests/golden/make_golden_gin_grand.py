#!/usr/bin/env python
"""Generate tests/golden/gin_grand.npz by running the REFERENCE's own GINLayer, GINELayer and Grand.rand_prop
(cogdl/layers/gin_layer.py, gine_layer.py, cogdl/models/nn/grand.py) on CPU.
Run where the reference checkout exists, after oracle/build_ref.py:   python tests/golden/make_golden_gin_grand.py

Graph: a symmetric random graph with duplicate edges, a hub (node 0, linked to half the nodes) and an isolated node
(7), built from edge_index.  Stored: the arrays; for GINLayer (eps = 0.1 trainable, eps = -1 fixed) and GINELayer
(eps = -0.3 trainable), without apply_func, the output and, for the upstream gradient `g`, d x and d eps; and, on the
graph after sym_norm() (its CSR-order edges and weights stored as `srow`, `scol`, `sw`), Grand.rand_prop for order in
{0, 1, 2, 8} in train mode (torch.manual_seed(SEED) before the call; the DropNode mask that seed draws is stored as
`mask_<order>`) and in eval mode.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import import_reference  # noqa: E402

N, E, F = 300, 1500, 8
ISOLATED = 7
ORDERS = (0, 1, 2, 8)
DROPNODE = 0.5
SEED = 123
GIN_CASES = (("gin", 0.1, True), ("gin_fixed", -1.0, False), ("gine", -0.3, True))


def arrays():
    g = torch.Generator().manual_seed(53)
    row = torch.randint(0, N - 1, (E,), generator=g)
    col = torch.randint(0, N - 1, (E,), generator=g)
    hub_nbrs = torch.randperm(N - 1, generator=g)[: N // 2]
    row = torch.cat([row, torch.zeros_like(hub_nbrs), torch.tensor([N - 1])])   # the last node has an edge, so the
    col = torch.cat([col, hub_nbrs, torch.tensor([1])])                         # reference counts N nodes
    keep = (row != ISOLATED) & (col != ISOLATED)
    row, col = row[keep], col[keep]
    row, col = torch.cat([row, col]), torch.cat([col, row])
    return {"row": row.numpy(), "col": col.numpy(), "x": torch.randn(N, F, generator=g).numpy(),
            "g": torch.randn(N, F, generator=g).numpy()}


def make_graph(Graph, d):
    return Graph(x=torch.from_numpy(d["x"]).clone(),
                 edge_index=(torch.from_numpy(d["row"]).clone(), torch.from_numpy(d["col"]).clone()))


def main():
    Graph = import_reference()[0]
    from cogdl.layers import GINELayer, GINLayer
    from cogdl.models.nn.grand import Grand

    out = arrays()
    for key, eps, train in GIN_CASES:
        layer = (GINELayer if key == "gine" else GINLayer)(None, eps, train)
        x = torch.from_numpy(out["x"]).clone().requires_grad_(True)
        y = layer(make_graph(Graph, out), x)
        y.backward(torch.from_numpy(out["g"]))
        out[f"{key}_out"], out[f"{key}_dx"] = y.detach().numpy(), x.grad.numpy()
        if train:
            out[f"{key}_deps"] = layer.eps.grad.numpy()
    graph = make_graph(Graph, out)
    graph.sym_norm()
    graph.row_indptr
    out["srow"], out["scol"] = graph.edge_index[0].numpy(), graph.edge_index[1].numpy()
    out["sw"] = graph.edge_weight.numpy()
    for order in ORDERS:
        model = Grand(F, 16, 3, 0.0, 0.0, False, DROPNODE, order, 0.5)
        model.train()
        torch.manual_seed(SEED)
        out[f"mask_{order}"] = torch.bernoulli(1.0 - torch.ones(N) * DROPNODE).numpy()
        torch.manual_seed(SEED)
        with torch.no_grad():
            out[f"grand_train_{order}"] = model.rand_prop(graph, torch.from_numpy(out["x"]).clone()).numpy()
        model.eval()
        with torch.no_grad():
            out[f"grand_eval_{order}"] = model.rand_prop(graph, torch.from_numpy(out["x"]).clone()).numpy()
    np.savez_compressed(os.path.join(HERE, "gin_grand.npz"), **out)
    print(f"wrote gin_grand.npz: {sorted(k for k in out if k.startswith(('gin', 'grand')))}")


if __name__ == "__main__":
    main()

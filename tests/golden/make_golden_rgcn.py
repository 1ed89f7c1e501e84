#!/usr/bin/env python
"""Generate tests/golden/rgcn.npz by running the REFERENCE's own RGCNLayer (cogdl/layers/rgcn_layer.py) and spmm on
CPU.  Run where the reference checkout exists, after oracle/build_ref.py:   python tests/golden/make_golden_rgcn.py

Graph: a random shuffled COO on N nodes with edge types, built from edge_index.  Stored:
  * `row`, `col`, `x` and, for T = 1 (alpha None) and T = 4 with 2 bases (self-loop weight zeroed, no layer_norm, no
    bias, so the output is the aggregation alone), the layer's parameters and its output `out_t<T>`;
  * the graph after the layer call, in its CSR order: `srow`, `scol`, `stype_t<T>` and the row-normalised weights `sw`;
  * for T = 4, one piece per relation from the reference's own primitives: `piece_<t>` = spmm(g_t, x @ W_t), with g_t
    a Graph of the type-t edges carrying their row-normalised weights (the relational sum is their sum).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import import_reference  # noqa: E402

N, E, F_IN, F_OUT = 200, 1200, 12, 8
CASES = ((1, None), (4, 2))


def main():
    import_reference()
    from cogdl.data import Graph
    from cogdl.layers.rgcn_layer import RGCNLayer
    from cogdl.utils import spmm

    g = torch.Generator().manual_seed(61)
    row = torch.randint(0, N, (E,), generator=g)
    col = torch.randint(0, N, (E,), generator=g)
    row[0], col[0] = N - 1, 0                          # the last node has an edge, so the graph counts N nodes
    x = torch.randn(N, F_IN, generator=g)
    out = {"row": row.numpy(), "col": col.numpy(), "x": x.numpy()}
    for T, nb in CASES:
        etype = torch.randint(0, T, (E,), generator=g)
        if T > 1:
            etype[etype == 0] = 1                      # relation 0 absent: the first present relation is 1
        out[f"type_t{T}"] = etype.numpy()
        torch.manual_seed(62 + T)
        layer = RGCNLayer(F_IN, F_OUT, T, "basis", nb, layer_norm=T == 1, bias=True)
        with torch.no_grad():
            if layer.bias is not None:
                layer.bias.normal_()
            if T > 1:
                layer.weight_self_loop.zero_()
                layer.bias.zero_()
        graph = Graph(edge_index=(row.clone(), col.clone()), edge_attr=etype.clone(), x=x)
        with torch.no_grad():
            y = layer(graph, x)
        out[f"out_t{T}"] = y.numpy()
        for k, v in layer.state_dict().items():
            if v is not None:
                out[f"p_t{T}_{k}"] = v.numpy()
        srow, scol = graph.edge_index
        out["srow"], out["scol"], out["sw"] = srow.numpy(), scol.numpy(), graph.edge_weight.detach().numpy()
        out[f"stype_t{T}"] = graph.edge_attr.numpy()
        if T > 1:
            with torch.no_grad():
                W = (layer.alpha @ layer.weight.view(nb, -1)).view(T, F_IN, F_OUT)
                for t in range(T):
                    m = graph.edge_attr == t
                    gt = Graph(edge_index=(srow[m], scol[m]), edge_weight=graph.edge_weight[m], num_nodes=N)
                    out[f"piece_{t}"] = spmm(gt, x @ W[t]).numpy()
    path = os.path.join(HERE, "rgcn.npz")
    np.savez_compressed(path, **out)
    print("wrote", path, sorted(out))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Generate tests/golden/genconv.npz by running the REFERENCE's own GENConv (cogdl/layers/deepergcn_layer.py) on CPU.
Run where the reference checkout exists, after oracle/build_ref.py:   python tests/golden/make_golden_genconv.py

The aggregated h (what GENConv.forward hands to its MLP) is captured with a forward pre-hook on `conv.mlp`.
Cases: softmax_sg at beta 0.5 and 2, softmax, mean, sum and powermean (p = 2), each without and with an
EdgeEncoder.  max is left out: on CPU the reference's max pooling needs torch_scatter.  The logits beta * m stay
below 10, because the reference's CPU edge softmax halves larger ones.  Stored per case: h and, with an encoder,
the encoder's output in CSR order (the edge term); the graph (CSR) and x are stored once.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import import_reference  # noqa: E402

CASES = [("softmax_sg", 0.5), ("softmax_sg", 2.0), ("softmax", None), ("mean", None), ("sum", None), ("powermean", None)]


def case_key(aggr, beta, edge):
    return f"{aggr}{'' if beta is None else f'_b{beta:g}'}{'_edge' if edge else ''}"


def main():
    Graph = import_reference()[0]
    from cogdl.layers import GENConv

    torch.manual_seed(0)
    n, e, F, n_attr = 60, 400, 16, 4
    g = torch.Generator().manual_seed(7)
    row, col = torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g)
    keep = row >= 4                      # rows 0-3 without edges: degree-0 rows
    row, col = row[keep], col[keep]
    x = torch.randn(n, F, generator=g).clamp(-2.0, 2.0)
    edge_attr = torch.rand(row.numel(), n_attr, generator=g)
    out = {}
    for edge in (False, True):
        for aggr, beta in CASES:
            graph = Graph(x=x, edge_index=(row, col), edge_attr=edge_attr if edge else None)
            graph.row_indptr             # CSR order before the forward reads edge_index / edge_attr
            kw = {"beta": beta} if beta is not None else {}
            if aggr == "powermean":
                kw["p"] = 2.0
            conv = GENConv(F, F, aggr=aggr, edge_attr_size=[n_attr] if edge else None, **kw)
            captured = {}
            conv.mlp.register_forward_pre_hook(lambda mod, args: captured.setdefault("h", args[0].detach().clone()))
            with torch.no_grad():
                conv(graph, x)
                key = case_key(aggr, beta, edge)
                out["h_" + key] = captured["h"].numpy()
                if edge:
                    out["edge_" + key] = conv.edge_encoder(graph.edge_attr).numpy()
                    assert float((torch.relu(x[graph.col_indices] + conv.edge_encoder(graph.edge_attr)) * (beta or 1)).max()) <= 10
            out.setdefault("rowptr", graph.row_indptr.numpy())
            out.setdefault("colind", graph.col_indices.numpy())
    out["x"] = x.numpy()
    np.savez_compressed(os.path.join(HERE, "genconv.npz"), **out)
    print(f"wrote genconv.npz: {sorted(k for k in out if k.startswith('h_'))}")


if __name__ == "__main__":
    main()

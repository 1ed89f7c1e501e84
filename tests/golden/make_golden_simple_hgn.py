#!/usr/bin/env python
"""Generate tests/golden/simple_hgn.npz by running the REFERENCE's own Simple-HGN layer (myGATConv,
examples/simple_hgn/conv.py) on CPU.  Run where the reference checkout exists, after oracle/build_ref.py:
    python tests/golden/make_golden_simple_hgn.py

Graph: a shuffled COO on N nodes (some rows empty) with T = 5 edge types held in graph.edge_type, built from
edge_index.  The reference's CPU edge_softmax builds the CSR of a local copy of the graph and divides the COO-ordered
logits by the sums of the CSR-ordered rows, which pairs them with other rows' sums unless the edges are already in CSR
order.  So the CSR is built first (graph.row_indptr, a stable sort of the edges by row) and the types are put through
the same sort, which is what cogdl_b200.install_simple_hgn does on entry; `order` is that sort.  Three convs, attention
dropout 0:  c1 (H = 8) -> c2 (H = 8, res_attn = c1's attention, alpha = 0.05, residual Linear) -> c3 (H = 1, the output
layer), tanh after c1 and c2.  Loss = sum(out2 * g2) + sum(out3 * g3).  Stored: row, col, type, x, g2, g3, every
parameter (`c<k>_<name>`), the outputs `out<k>` and returned attentions `att<k>` (CSR order), and the gradients of x
and of every parameter (`grad_x`, `grad_c<k>_<name>`).  Every logit is asserted within [-10, 10]: the reference's CPU
edge_softmax halves larger logits.  The run uses the reference's scatter SpMM (its path when the C++ spmm_cpu op is
not loaded): through spmm_cpu the softmax's row sums get no gradient, so the layer's CPU backward would drop the
softmax's `- sum_row a * g` term.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import REF, import_reference  # noqa: E402

N, E, T, F_IN, HID, NCLS, EDGE_FEATS = 120, 900, 5, 16, 8, 3, 6
SLOPE, ALPHA = 0.2, 0.05


def main():
    import_reference()
    sys.path.insert(0, os.path.join(REF, "examples", "simple_hgn"))
    import cogdl.utils.spmm_utils as su
    from cogdl.data import Graph
    from conv import myGATConv

    su.CONFIGS["spmm_cpu_flag"], su.CONFIGS["fast_spmm_cpu"] = True, None

    g = torch.Generator().manual_seed(71)
    row = torch.randint(0, N - 10, (E,), generator=g)          # rows N-10 .. N-1 have no edges
    col = torch.randint(0, N, (E,), generator=g)
    row[0], col[0] = 3, N - 1                                  # the last node appears, so the graph counts N nodes
    etype = torch.randint(0, T, (E,), generator=g)
    x = torch.randn(N, F_IN, generator=g).requires_grad_(True)
    graph = Graph(edge_index=(row.clone(), col.clone()), num_nodes=N)
    graph.row_indptr                                           # builds the CSR: sorts the edges by row, stably
    order = torch.sort(row, stable=True).indices
    assert torch.equal(graph.edge_index[0], row[order]) and torch.equal(graph.edge_index[1], col[order])
    graph.edge_type = etype[order]
    torch.manual_seed(72)
    c1 = myGATConv(EDGE_FEATS, T, F_IN, HID, 8, attn_drop=0.0, negative_slope=SLOPE, activation="tanh")
    c2 = myGATConv(EDGE_FEATS, T, HID * 8, HID, 8, attn_drop=0.0, negative_slope=SLOPE, residual=True,
                   activation="tanh", alpha=ALPHA)
    c3 = myGATConv(EDGE_FEATS, T, HID * 8, NCLS, 1, attn_drop=0.0, negative_slope=SLOPE)
    convs = (c1, c2, c3)

    def logits(conv, inp):
        with torch.no_grad():
            h = (inp @ conv.W).view(-1, conv.nhead, conv.out_features)
            e = (conv.edge_emb @ conv.W_e).view(-1, conv.nhead, conv.edge_feats)
            z = (conv.a_l * h).sum(-1)[row] + (conv.a_r * h).sum(-1)[col] + (conv.a_e * e).sum(-1)[etype]   # any order
            return torch.nn.functional.leaky_relu(z, SLOPE)

    out1, att1 = c1(graph, x)
    out2, att2 = c2(graph, out1, res_attn=att1)
    out3, att3 = c3(graph, out2)
    for conv, inp in zip(convs, (x, out1, out2)):
        assert float(logits(conv, inp).abs().max()) <= 10.0, "a logit beyond 10: the CPU edge_softmax would halve it"
    ei = graph.edge_index
    assert torch.equal(ei[0], row[order]) and torch.equal(ei[1], col[order]), "the CPU path reordered the edges"
    g2 = torch.randn(out2.shape, generator=g)
    g3 = torch.randn(out3.shape, generator=g)
    ((out2 * g2).sum() + (out3 * g3).sum()).backward()
    out = {"row": row, "col": col, "type": etype, "order": order, "x": x, "g2": g2, "g3": g3, "grad_x": x.grad}
    for k, conv in enumerate(convs, 1):
        for name, prm in conv.named_parameters():
            out[f"c{k}_{name}"] = prm
            out[f"grad_c{k}_{name}"] = prm.grad
    for k, (o, a) in enumerate(((out1, att1), (out2, att2), (out3, att3)), 1):
        out[f"out{k}"], out[f"att{k}"] = o, a
    path = os.path.join(HERE, "simple_hgn.npz")
    np.savez_compressed(path, **{k: v.detach().numpy() for k, v in out.items()})
    print("wrote", path, sorted(out))


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Generate tests/golden/compgcn.npz by running the REFERENCE's own CompGCNLayer (cogdl/models/nn/compgcn.py) on CPU.
Run where the reference checkout exists, after oracle/build_ref.py:   python tests/golden/make_golden_compgcn.py

The KG: N entities, R relations, triples plus their reverses (type t + R), one extra edge so E is odd, the whole COO
shuffled (the halves [0, E // 2) and [E // 2, E) are not CSR prefixes).  Entities 0-2 appear in no triple, so they
are degree-0 rows of both halves.  Cases: opn in (sub, mult), without and with bases; dropout 0, BatchNorm in train
mode, tanh activation, a non-zero bias.  For the fixed upstream gradients G (node output) and GR (relation output)
the gradients of x, rel_embed (no bases) and every parameter are stored.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import import_reference  # noqa: E402

N, R, TRIPLES, F_IN, F_OUT = 50, 4, 90, 12, 10
CASES = [("sub", 0), ("mult", 0), ("sub", 3), ("mult", 3)]


def case_key(opn, bases):
    return f"{opn}_b{bases}"


def make_kg():
    g = torch.Generator().manual_seed(21)
    h = torch.randint(3, N, (TRIPLES,), generator=g)
    t = torch.randint(3, N, (TRIPLES,), generator=g)
    r = torch.randint(0, R, (TRIPLES,), generator=g)
    row = torch.cat([h, t, torch.tensor([5])])
    col = torch.cat([t, h, torch.tensor([7])])
    typ = torch.cat([r, r + R, torch.tensor([1])])
    perm = torch.randperm(row.numel(), generator=g)
    return row[perm], col[perm], typ[perm]


def main():
    import_reference()
    from cogdl.data import Graph
    from cogdl.models.nn.compgcn import CompGCNLayer

    row, col, typ = make_kg()
    assert row.numel() % 2 == 1
    g = torch.Generator().manual_seed(22)
    x0 = torch.randn(N, F_IN, generator=g)
    rel0 = torch.randn(2 * R, F_IN, generator=g)
    G = torch.randn(N, F_OUT, generator=g)
    GR = torch.randn(2 * R, F_OUT, generator=g)
    out = {"row": row.numpy(), "col": col.numpy(), "type": typ.numpy(), "x": x0.numpy(), "rel": rel0.numpy(),
           "G": G.numpy(), "GR": GR.numpy()}
    for opn, bases in CASES:
        key = case_key(opn, bases)
        torch.manual_seed(100 + bases + (opn == "mult"))
        layer = CompGCNLayer(F_IN, F_OUT, R, opn=opn, num_bases=bases, activation=torch.tanh, dropout=0.0).train()
        with torch.no_grad():
            layer.bias.copy_(0.2 * torch.randn(F_OUT, generator=g))
            layer.bn.weight.copy_(1.0 + 0.3 * torch.randn(F_OUT, generator=g))
            layer.bn.bias.copy_(0.1 * torch.randn(F_OUT, generator=g))
        graph = Graph(edge_index=(row.clone(), col.clone()), edge_attr=typ.clone())
        x, rel = x0.clone().requires_grad_(True), rel0.clone().requires_grad_(True)
        y, yr = layer(graph, x, rel)
        ((y * G).sum() + (yr * GR).sum()).backward()
        assert torch.equal(graph.edge_index[0], row), "the reference forward must not reorder the COO"
        out["y_" + key] = y.detach().numpy()
        out["yr_" + key] = yr.detach().numpy()
        out["dx_" + key] = x.grad.numpy()
        if not bases:
            out["drel_" + key] = rel.grad.numpy()
        for name, prm in layer.named_parameters():
            out[f"p_{key}_{name}"] = prm.detach().numpy()
            out[f"g_{key}_{name}"] = prm.grad.numpy()
    np.savez_compressed(os.path.join(HERE, "compgcn.npz"), **out)
    print(f"wrote compgcn.npz: {sorted(k for k in out if k.startswith('y_'))}")


if __name__ == "__main__":
    main()

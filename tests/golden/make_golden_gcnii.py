#!/usr/bin/env python
"""Generate tests/golden/gcnii_appnp.npz by running the REFERENCE's own GCNII (cogdl/models/nn/gcnii.py, 8 layers x 64,
residual off and on) and PPNP (cogdl/models/nn/ppnp.py, "appnp", K = 10) on CPU, in eval mode.
Run where the reference checkout exists, after oracle/build_ref.py:   python tests/golden/make_golden_gcnii.py

Graphs (tests/gcnii_refpkg_check.py builds the same two from the stored arrays): a symmetric random graph with
duplicate edges, built once from CSR (row_ptr, col: sym_norm sets in_norm / out_norm) and once from edge_index (sym_norm
rescales the edge weights).  Stored per (model, graph): the logits, taken under no_grad, where the reference's CPU spmm
applies in_norm / out_norm; and, for a fixed upstream gradient G, the gradient of every parameter.  The gradients of
GCNII on the CSR-built graph are not stored: with gradients on, the reference's CPU spmm takes spmm_scatter over
edge_index, which ignores in_norm / out_norm (spmm_utils.py:98-123), so its CPU autograd run computes a different
function from its own forward.  tests/gcnii_ref.py's fp64 gradients stand in for them there.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import import_reference  # noqa: E402

N, E, F_IN, HID, C = 300, 2400, 24, 64, 7
MODELS = ("gcnii_res0", "gcnii_res1", "appnp")
GRAPHS = ("csr", "coo")


def graph_arrays():
    """(rowptr, col, x, G) of the symmetric graph with duplicate edges, col in CSR order."""
    g = torch.Generator().manual_seed(41)
    row = torch.randint(0, N, (E,), generator=g)
    col = torch.randint(0, N, (E,), generator=g)
    row, col = torch.cat([row, col]), torch.cat([col, row])
    x = torch.randn(N, F_IN, generator=g)
    G = torch.randn(N, C, generator=g)
    order = torch.argsort(row * N + col)
    row, col = row[order], col[order]
    rp = torch.zeros(N + 1, dtype=torch.int64)
    rp[1:] = torch.cumsum(torch.bincount(row, minlength=N), 0)
    return rp, col, x, G


def make_graph(Graph, built_from, rp, col, x):
    """A fresh reference Graph of the arrays (every forward normalises the graph it is given)."""
    if built_from == "csr":
        return Graph(x=x.clone(), row_ptr=rp.clone(), col=col.clone())
    row = torch.repeat_interleave(torch.arange(N), rp[1:] - rp[:-1])
    return Graph(x=x.clone(), edge_index=(row, col.clone()))


def make_model(name):
    from cogdl.models.nn.gcnii import GCNII
    from cogdl.models.nn.ppnp import PPNP

    if name == "appnp":
        torch.manual_seed(12)
        return PPNP(F_IN, HID, C, 2, 0.5, "appnp", 0.1, 10)
    res = name == "gcnii_res1"
    torch.manual_seed(10 + res)
    return GCNII(F_IN, HID, C, 8, dropout=0.5, alpha=0.1, lmbda=0.5, residual=res)


def main():
    Graph = import_reference()[0]
    rp, col, x, G = graph_arrays()
    out = {"rowptr": rp.numpy(), "col": col.numpy(), "x": x.numpy(), "G": G.numpy()}
    for m in MODELS:
        model = make_model(m).eval()
        for k, p in model.named_parameters():
            out[f"p_{m}_{k}"] = p.detach().numpy()
        for gk in GRAPHS:
            with torch.no_grad():
                out[f"y_{m}_{gk}"] = model(make_graph(Graph, gk, rp, col, x)).numpy()
            if m != "appnp" and gk == "csr":
                continue
            model.zero_grad(set_to_none=True)
            y = model(make_graph(Graph, gk, rp, col, x))
            assert np.allclose(y.detach().numpy(), out[f"y_{m}_{gk}"], rtol=1e-5, atol=1e-6), (m, gk)
            (y * G).sum().backward()
            for k, p in model.named_parameters():
                out[f"g_{m}_{gk}_{k}"] = p.grad.numpy()
    np.savez_compressed(os.path.join(HERE, "gcnii_appnp.npz"), **out)
    print(f"wrote gcnii_appnp.npz: {sorted(k for k in out if k.startswith('y_'))}")


if __name__ == "__main__":
    main()

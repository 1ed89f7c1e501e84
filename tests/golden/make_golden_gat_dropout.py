#!/usr/bin/env python
"""Generate tests/golden/gat_dropout.npz by running the REFERENCE's own GATLayer (cogdl/layers/gat_layer.py) on CPU
with attention dropout.  Run where the reference checkout exists, after oracle/build_ref.py:
    python tests/golden/make_golden_gat_dropout.py

The layer's `self.dropout` is replaced by a module with p > 0 (so gat_layer.py:68 takes the unfused branch) that
multiplies the attention by a fixed mask and 1 / (1 - p).  The mask is the kernels' keep rule for a stored seed
(tests/gat_dropout_ref.keep_mask), so the GPU tests can run the fused layer with that seed against the same output.
The graph: N nodes, edges sorted by (row, col) so that the edge order is the CSR order, not symmetric, one hub row
(300 draws, about 220 distinct edges) and 60 degree-0 rows.  Cases: H = 8 (8 x 8) and H = 1 (1 x 16), p = 0.5, in_feats 24.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))

from make_golden import import_reference  # noqa: E402
from tests.gat_dropout_ref import keep_mask  # noqa: E402

N, E, F_IN, P, SLOPE = 400, 3000, 24, 0.5, 0.2
CASES = [("h8", 8, 8, 0x5EED0001), ("h1", 1, 16, 0x5EED0002)]


class FixedMaskDropout(torch.nn.Module):
    def __init__(self, p, mask):
        super().__init__()
        self.p = p
        self.register_buffer("mask", mask)

    def forward(self, x):
        return x * self.mask / (1.0 - self.p)


def make_graph():
    g = torch.Generator().manual_seed(41)
    row = torch.randint(60, N, (E,), generator=g)
    row[:300] = 77                                            # hub row
    col = torch.randint(0, N, (E,), generator=g)
    key = torch.unique(row * N + col)                          # sorted (row, col), no duplicates
    return key // N, key % N


def main():
    import_reference()
    from cogdl.data import Graph
    from cogdl.layers import GATLayer

    row, col = make_graph()
    n_e = row.numel()
    rowptr = np.zeros(N + 1, np.int64)
    rowptr[1:] = np.cumsum(np.bincount(row.numpy(), minlength=N))
    g = torch.Generator().manual_seed(42)
    x0 = torch.randn(N, F_IN, generator=g)
    out = {"row": row.numpy(), "col": col.numpy(), "rowptr": rowptr, "x": x0.numpy(), "p": np.float64(P),
           "slope": np.float64(SLOPE)}
    for key, H, F, seed in CASES:
        torch.manual_seed(7 + H)
        layer = GATLayer(F_IN, F, nhead=H, alpha=SLOPE, attn_drop=P).train()
        mask = torch.from_numpy(keep_mask(seed, n_e, H, P).astype(np.float32))
        layer.dropout = FixedMaskDropout(P, mask)
        graph = Graph(x=x0.clone(), edge_index=(row.clone(), col.clone()))
        assert set(zip(row.tolist(), col.tolist())) != set(zip(col.tolist(), row.tolist())), "must not be symmetric"
        assert torch.equal(graph.row_indptr, torch.from_numpy(rowptr)) and torch.equal(graph.col_indices, col)
        y = layer(graph, x0.clone())
        assert torch.equal(graph.edge_index[0], row) and torch.equal(graph.edge_index[1], col)
        out[f"seed_{key}"] = np.uint64(seed)
        out[f"mask_{key}"] = mask.numpy().astype(bool)
        out[f"y_{key}"] = y.detach().numpy()
        for name in ("W", "a_l", "a_r"):
            out[f"{name}_{key}"] = getattr(layer, name).detach().numpy()
    np.savez_compressed(os.path.join(HERE, "gat_dropout.npz"), **out)
    print(f"wrote gat_dropout.npz: E = {n_e}, cases {[c[0] for c in CASES]}")


if __name__ == "__main__":
    main()

#!/usr/bin/env python
"""Generate tests/golden/correct_smooth.npz by running the REFERENCE's own Correct & Smooth
(cogdl/models/nn/correct_smooth.py: CorrectSmooth.__call__ and diffusion) on CPU.
Run where the reference checkout exists, after oracle/build_ref.py:   python tests/golden/make_golden_correct_smooth.py

Graph: a symmetric random graph with duplicate edges, a hub (node 0, linked to half the nodes) and an isolated node
(7), built from edge_index.  Stored: the arrays, class logits, labels and split masks, and per case (autoscale on / off,
correct norm sym / row, smooth norm row / col; 20 correct and 20 smooth steps at the reference's default alphas) the
output of CorrectSmooth(...)(graph, softmax(logits)), which is what CorrectSmoothMLP.postprocess returns; and
diffusion(graph, x, nhtop=10) on a row-normalised copy.
"""
import itertools
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import import_reference  # noqa: E402

N, E, C, F_X, NPROP = 300, 1500, 5, 6, 20
ISOLATED = 7
CORRECT_ALPHA, SMOOTH_ALPHA = 1.0, 0.8
CASES = [(a, cn, sn) for a, cn, sn in itertools.product((False, True), ("sym", "row"), ("row", "col"))]


def case_key(autoscale, correct_norm, smooth_norm):
    return f"cs_{int(autoscale)}_{correct_norm}_{smooth_norm}"


def arrays():
    g = torch.Generator().manual_seed(47)
    row = torch.randint(0, N - 1, (E,), generator=g)
    col = torch.randint(0, N - 1, (E,), generator=g)
    hub_nbrs = torch.randperm(N - 1, generator=g)[: N // 2]
    row = torch.cat([row, torch.zeros_like(hub_nbrs)])
    col = torch.cat([col, hub_nbrs])
    row = torch.cat([row, torch.tensor([N - 1])])                    # the last node has an edge, so the reference's
    col = torch.cat([col, torch.tensor([1])])                        # Graph(edge_index=...) counts N nodes
    keep = (row != ISOLATED) & (col != ISOLATED)
    row, col = row[keep], col[keep]
    row, col = torch.cat([row, col]), torch.cat([col, row])
    split = torch.rand(N, generator=g)
    return {
        "row": row.numpy(), "col": col.numpy(),
        "logits": torch.randn(N, C, generator=g).numpy(),
        "y": torch.randint(0, C, (N,), generator=g).numpy(),
        "train_mask": (split < 0.4).numpy(), "val_mask": ((split >= 0.4) & (split < 0.6)).numpy(),
        "x": torch.rand(N, F_X, generator=g).numpy(),
    }


def make_graph(Graph, d):
    return Graph(x=torch.from_numpy(d["x"]).clone(), y=torch.from_numpy(d["y"]).clone(),
                 edge_index=(torch.from_numpy(d["row"]).clone(), torch.from_numpy(d["col"]).clone()),
                 train_mask=torch.from_numpy(d["train_mask"]).clone(), val_mask=torch.from_numpy(d["val_mask"]).clone(),
                 test_mask=torch.from_numpy(~(d["train_mask"] | d["val_mask"])).clone())


def main():
    Graph = import_reference()[0]
    from cogdl.models.nn.correct_smooth import CorrectSmooth, diffusion

    out = arrays()
    preds = torch.softmax(torch.from_numpy(out["logits"]), dim=-1)
    for autoscale, cn, sn in CASES:
        cs = CorrectSmooth(CORRECT_ALPHA, SMOOTH_ALPHA, NPROP, NPROP, autoscale, cn, sn, 1.0)
        with torch.no_grad():
            out[case_key(autoscale, cn, sn)] = cs(make_graph(Graph, out), preds.clone()).numpy()
    g = make_graph(Graph, out)
    g.row_norm()
    with torch.no_grad():
        out["diffusion"] = diffusion(g, torch.from_numpy(out["x"]).clone(), nhtop=10).numpy()
    np.savez_compressed(os.path.join(HERE, "correct_smooth.npz"), **out)
    print(f"wrote correct_smooth.npz: {sorted(k for k in out if k.startswith(('cs_', 'diff')))}")


if __name__ == "__main__":
    main()

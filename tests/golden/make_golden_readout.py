#!/usr/bin/env python
"""Generate tests/golden/readout.npz by running the REFERENCE's own readouts and graph-level models on CPU:
cogdl.utils.batch_sum_pooling / batch_mean_pooling, the GIN graph-classification model (cogdl/models/nn/gin.py), the
InfoGraph encoder (cogdl/models/nn/infograph.py, Encoder) and SortPool (cogdl/models/nn/sortpool.py).
Run where the reference checkout exists, after oracle/build_ref.py:   python tests/golden/make_golden_readout.py

Batch: N_GRAPHS random symmetric graphs of 5 to 40 nodes as one disjoint union, `batch` sorted (the reference's GIN
and SortPool read it so).  Stored: the arrays (row, col, x [N, 8], batch, x2 [N, 5]); sum / mean pooling of x2; the
GIN model (3 layers, hidden 16, dropout 0, built after torch.manual_seed(SEED_GIN)) in train mode: its logits, the
input of every linear_prediction (the pooled layer outputs, `gin_pooled_<i>`), the layer outputs (`gin_rep_<i>`) and,
for the upstream gradient `g_logits`, every parameter gradient (`gin_grad_<name>`); the InfoGraph encoder (3 layers,
hidden 16, sum pooling, built after torch.manual_seed(SEED_IG)): graph_rep and node_rep; SortPool (2 SAGE layers,
hidden 16, k = K, built after torch.manual_seed(SEED_SP)) in eval mode: its logits, the per-row sorted node features
it pools (`sp_h`) and the [B, k, F] tensor its conv1d reads (`sp_pooled`).
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import import_reference  # noqa: E402

N_GRAPHS, F_IN, F2 = 7, 8, 5
SEED_GIN, SEED_IG, SEED_SP = 21, 22, 23
K = 25


def arrays():
    rng = np.random.default_rng(61)
    rows, cols, batch, off = [], [], [], 0
    for b in range(N_GRAPHS):
        n = int(rng.integers(5, 41))
        e = int(rng.integers(n, 4 * n))
        r, c = rng.integers(0, n, e), rng.integers(0, n, e)
        rows += [r + off, c + off]
        cols += [c + off, r + off]
        batch.append(np.full(n, b))
        off += n
    return {"row": np.concatenate(rows), "col": np.concatenate(cols), "batch": np.concatenate(batch),
            "x": rng.standard_normal((off, F_IN)).astype(np.float32),
            "x2": rng.standard_normal((off, F2)).astype(np.float32),
            "g_logits": rng.standard_normal((N_GRAPHS, 4)).astype(np.float32)}


def make_graph(Graph, d, dev="cpu"):
    """The batch as the reference's graph-level models read it: a Graph with `batch`."""
    g = Graph(x=torch.from_numpy(d["x"]).clone(), edge_index=(torch.from_numpy(d["row"]).clone(),
                                                              torch.from_numpy(d["col"]).clone()))
    g.batch = torch.from_numpy(d["batch"]).clone()
    g = g.to(dev)
    g.row_indptr
    return g


def build_gin():
    from cogdl.models.nn.gin import GIN

    torch.manual_seed(SEED_GIN)
    return GIN(3, F_IN, 4, 16, 2, 0.0, "sum", True, 0.0)


def build_infograph_encoder():
    from cogdl.models.nn.infograph import Encoder

    torch.manual_seed(SEED_IG)
    return Encoder(F_IN, 16, 3, 2, "sum")


def build_sortpool():
    from cogdl.models.nn.sortpool import SortPool

    torch.manual_seed(SEED_SP)
    return SortPool(F_IN, 16, 4, 2, 8, 5, k=K, dropout=0.0)


def main():
    Graph = import_reference()[0]
    from cogdl.utils import batch_mean_pooling, batch_sum_pooling

    out = arrays()
    x2, batch = torch.from_numpy(out["x2"]), torch.from_numpy(out["batch"])
    out["sum_x2"] = batch_sum_pooling(x2, batch).numpy()
    out["mean_x2"] = batch_mean_pooling(x2, batch).numpy()

    gin = build_gin()
    pooled = {}
    for i, lin in enumerate(gin.linear_prediction):
        lin.register_forward_pre_hook(lambda m, a, i=i: pooled.__setitem__(i, a[0].detach().clone()))
    reps = {}
    for i, bn in enumerate(gin.batch_norm):
        bn.register_forward_hook(lambda m, a, o, i=i: reps.__setitem__(i + 1, torch.relu(o).detach().clone()))
    logits = gin(make_graph(Graph, out))
    logits.backward(torch.from_numpy(out["g_logits"]))
    out["gin_logits"] = logits.detach().numpy()
    for i, p in pooled.items():
        out[f"gin_pooled_{i}"] = p.numpy()
    for i, r in reps.items():
        out[f"gin_rep_{i}"] = r.numpy()
    for name, p in gin.named_parameters():
        if p.grad is not None:
            out[f"gin_grad_{name}"] = p.grad.numpy()

    enc = build_infograph_encoder()
    g = make_graph(Graph, out)
    graph_rep, node_rep = enc(g, g.x)
    out["ig_graph_rep"], out["ig_node_rep"] = graph_rep.detach().numpy(), node_rep.detach().numpy()

    sp = build_sortpool()
    sp.eval()
    sp.gnn_convs[-1].register_forward_hook(
        lambda m, a, o: out.__setitem__("sp_h", torch.relu(o).sort(dim=-1)[0].detach().numpy().copy()))
    sp.conv1d.register_forward_pre_hook(
        lambda m, a: out.__setitem__("sp_pooled", a[0].permute(0, 2, 1).detach().numpy().copy()))
    with torch.no_grad():
        out["sp_logits"] = sp(make_graph(Graph, out)).numpy()

    path = os.path.join(HERE, "readout.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {sorted(out)}")


if __name__ == "__main__":
    main()

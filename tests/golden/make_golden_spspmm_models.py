"""Golden run of the reference GTN and SRGCN on the CPU -> tests/golden/gtn_srgcn.npz.

The reference models import torch_sparse, which CogDL does not depend on; here a stand-in provides spspmm / spmm in
fp64 (tests/spspmm_models_ref.py: structural pattern, fp64 values and value gradients, returned in the input's dtype).
Both models run in eval mode (no dropout) from seeded parameters, and sum(G * logits) is backpropagated with a seeded G.
Stored: the inputs, the parameters, G, the logits and every parameter gradient.

    python -m tests.golden.make_golden_spspmm_models      (needs the reference package, oracle/_ref/pkg)
"""
import os
import sys
import types

import numpy as np
import torch

from tests import spspmm_models_ref as R

OUT = os.path.join(os.path.dirname(os.path.abspath(__file__)), "gtn_srgcn.npz")


def standin():
    mod = types.ModuleType("torch_sparse")
    mod.spspmm, mod.spmm = R.spspmm64, R.spmm64
    return mod


def run_gtn(GTN, Graph, dev="cpu", state=None):
    adj, x = R.gtn_inputs()
    torch.manual_seed(0)
    model = GTN(4, 2, R.F_GTN, R.HID_GTN, R.C_GTN, R.N_GTN, 2)
    if state is not None:
        model.load_state_dict(state)
    model = model.to(dev).eval()
    graph = Graph(x=x, edge_index=adj[0][0]).to(dev)
    graph.adj = [(i.to(dev), v.to(dev)) for i, v in adj]
    out = model(graph)
    G = torch.randn(out.shape, generator=torch.Generator().manual_seed(5))
    (out * G.to(dev)).sum().backward()
    return model, out.detach().cpu(), G


def run_srgcn(SRGCN, Graph, dev="cpu", state=None):
    ei, x = R.cora_inputs()
    torch.manual_seed(0)
    model = SRGCN(in_feats=R.F_CORA, hidden_size=8, out_feats=R.C_CORA, attention="node", activation="leaky_relu",
                  nhop=2, normalization="row_uniform", dropout=0.0, node_dropout=0.0, alpha=0.2, nhead=R.NHEAD,
                  subheads=1)
    if state is not None:
        model.load_state_dict(state)
    model = model.to(dev).eval()
    out = model(Graph(x=x, edge_index=ei).to(dev))
    G = torch.randn(out.shape, generator=torch.Generator().manual_seed(6))
    (out * G.to(dev)).sum().backward()
    return model, out.detach().cpu(), G


def main():
    from tests.refpkg import import_reference

    import_reference()
    sys.modules["torch_sparse"] = standin()
    from cogdl.data import Graph
    from cogdl.models.nn.gtn import GTN
    from cogdl.models.nn.srgcn import SRGCN

    d = {}
    adj, x = R.gtn_inputs()
    for r, (e, v) in enumerate(adj):
        d[f"gtn_index_{r}"], d[f"gtn_value_{r}"] = e.numpy().astype(np.int32), v.numpy()
    d["gtn_x"] = x.numpy()
    ei, xc = R.cora_inputs()
    d["srgcn_index"], d["srgcn_x"] = ei.numpy().astype(np.int32), xc.numpy()
    for tag, run, cls in (("gtn", run_gtn, GTN), ("srgcn", run_srgcn, SRGCN)):
        model, out, G = run(cls, Graph)
        d[f"{tag}_G"], d[f"{tag}_logits"] = G.numpy(), out.numpy()
        for k, p in model.named_parameters():
            d[f"{tag}_p_{k}"] = p.detach().numpy()
            if p.grad is not None:
                d[f"{tag}_g_{k}"] = p.grad.numpy()
    np.savez_compressed(OUT, **d)
    print(OUT, sum(v.nbytes for v in d.values()), "bytes")


if __name__ == "__main__":
    main()

"""Child process of tests/test_gpu_gat_dropout.py: the UNMODIFIED reference GAT (2 layers, 8 heads x 8, attn_drop 0.5,
feature dropout 0.6) trained for a few SGD steps on the GPU through cogdl_b200.install(gat=True).  Runs in its own
process because install() rebinds the reference's dispatch for the rest of the process.  Prints one JSON line.

Checked: install() alone leaves GATLayer.forward alone; the losses are finite and fall; the steps are bit-reproducible
under torch.manual_seed and another seed gives another mask; eval-mode logits match the reference's unfused path
(edge_softmax + mh_spmm, run after uninstall_gat()); CPU input, half input and a dropout of 1 run the original
forward; uninstall_gat() restores it.
"""
import copy
import json

import numpy as np
import torch
import torch.nn.functional as F

from tests.refpkg import import_reference
from tests.test_gpu_refpkg import rel

N, E, F_IN, CLASSES = 3000, 30000, 64, 7


def make_graph(Graph):
    g = torch.Generator().manual_seed(51)
    row = torch.randint(0, N, (E,), generator=g)
    col = torch.randint(0, N, (E,), generator=g)
    row[:2000] = 5                                      # a hub row
    x = torch.randn(N, F_IN, generator=g)
    y = torch.randint(0, CLASSES, (N,), generator=g)
    return Graph(x=x, edge_index=(row, col), y=y)


def main():
    import_reference()
    import cogdl.layers.gat_layer as gl
    from cogdl.data import Graph
    from cogdl.models.nn.gat import GAT

    import cogdl_b200

    res = {}
    dev = torch.device("cuda:0")
    original = gl.GATLayer.forward
    cogdl_b200.install()
    res["untouched_without_flag"] = gl.GATLayer.forward is original
    res["patched"] = cogdl_b200.install(gat=True)
    res["rebound"] = gl.GATLayer.forward is not original

    graph = make_graph(Graph).to(dev)
    torch.manual_seed(0)
    model0 = GAT(F_IN, 8, CLASSES, 2, 0.6, 0.5, 0.2, 8, False, 1).to(dev)

    def train(seed, steps=5):
        model = copy.deepcopy(model0).train()
        opt = torch.optim.SGD(model.parameters(), lr=0.5)
        torch.manual_seed(seed)
        losses = []
        for _ in range(steps):
            opt.zero_grad()
            out = model(graph)
            loss = F.cross_entropy(out, graph.y)
            loss.backward()
            opt.step()
            losses.append(loss.item())
        torch.cuda.synchronize()
        return losses, out.detach(), [p.detach().clone() for p in model.parameters()]

    l1, o1, p1 = train(1)
    l2, o2, p2 = train(1)
    _, o3, _ = train(2)
    res["losses"] = l1
    res["losses_finite"] = bool(np.isfinite(l1).all())
    res["loss_decreases"] = l1[-1] < l1[0]
    res["reproducible"] = l1 == l2 and torch.equal(o1, o2) and all(torch.equal(a, b) for a, b in zip(p1, p2))
    res["seed_changes_mask"] = not torch.equal(o1, o3)

    model0.eval()
    fused = model0(graph).detach()
    cogdl_b200.uninstall_gat()
    res["restored"] = gl.GATLayer.forward is original
    unfused = model0(graph).detach()
    res["eval_vs_unfused"] = rel(fused, unfused)

    # cases without a kernel run the original forward
    cogdl_b200.install(gat=True)
    calls, real = [], gl.GATLayer._cogdl_b200_original_forward
    layer = copy.deepcopy(model0.attentions[0])
    x = graph.x

    def probe(kind, lay, g, inp):
        gl.GATLayer._cogdl_b200_original_forward = lambda self, gr, xx: (calls.append(kind), real(self, gr, xx))[1]
        try:
            lay(g, inp)
        except Exception:  # noqa: BLE001  (only which forward ran is checked here)
            pass
        gl.GATLayer._cogdl_b200_original_forward = real

    probe("cpu", copy.deepcopy(layer).cpu().eval(), make_graph(Graph), make_graph(Graph).x)
    probe("half", copy.deepcopy(layer).half().eval(), graph, x.half())
    p1_layer = copy.deepcopy(layer).train()
    p1_layer.dropout.p = 1.0
    probe("p1", p1_layer, graph, x)
    res["uncovered_ran_original"] = calls
    cogdl_b200.uninstall_gat()
    res["restored"] = res["restored"] and gl.GATLayer.forward is original
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Child process of tests/test_gpu_actnn.py: the UNMODIFIED reference ActGCN, GCNII(actnn=True) and
GraphSAGE(actnn=True) on the GPU through cogdl_b200.install(actnn=True), against the same models without actnn and with
the same weights.  Runs in its own process because install() rebinds the reference's modules.  Prints one JSON line.

Checked: the models build (the reference exits at construction without actnn); with dropout 0 the training-mode
forward equals the uncompressed model's; at 8 bits, deterministic rounding, the parameter gradients are within 1e-2
relative (all parameter gradients as one vector); at 2 bits with stochastic rounding the gradient averaged over 64 seeds is at least 4x closer to the fp32
gradient than one seed's; at an arxiv-sized shape the memory the forward keeps for the backward (the allocator's
growth over the forward, output excluded) is at most 1/8 of the uncompressed GCNII's.
"""
import json

import torch
import torch.nn.functional as F

from tests.refpkg import import_reference

N, E, F_IN, HID, CLASSES = 3000, 30000, 96, 64, 7


def make_graph(Graph, n=N, e=E, f=F_IN, seed=7):
    g = torch.Generator().manual_seed(seed)
    row = torch.randint(0, n, (e,), generator=g)
    col = torch.randint(0, n, (e,), generator=g)
    x = torch.randn(n, f, generator=g)
    y = torch.randint(0, CLASSES, (n,), generator=g)
    return Graph(x=x, edge_index=(torch.cat([row, col]), torch.cat([col, row])), y=y)


def rel(a, b):
    return float((a - b).norm() / b.norm().clamp_min(1e-30))


def rel_all(ga, gb):
    """Relative error of all parameter gradients taken as one vector."""
    return rel(torch.cat([g.reshape(-1) for g in ga]), torch.cat([g.reshape(-1) for g in gb]))


def grads(model, graph):
    """Output and parameter gradients of one step.  `graph` is used once: the models normalise its edge weights in
    place (sym_norm / row_norm), so every call gets a fresh copy."""
    model.zero_grad()
    out = model(graph)
    F.cross_entropy(out, graph.y).backward()
    return out.detach(), [p.grad.detach().clone() for p in model.parameters()]


def main():
    import_reference()
    import cogdl_b200

    res = {"patched": cogdl_b200.install(actnn=True)}
    import actnn
    from actnn.conf import config
    from actnn.qscheme import QScheme

    from cogdl.data import Graph
    from cogdl.models.nn.actgcn import ActGCN
    from cogdl.models.nn.gcn import GCN
    from cogdl.models.nn.gcnii import GCNII
    from cogdl.models.nn.graphsage import SAGE

    res["stand_in"] = actnn.__name__ == "cogdl_b200.actnn"
    dev = torch.device("cuda:0")
    def fresh():
        return make_graph(Graph).to(dev)

    def pair(name):
        torch.manual_seed(0)
        if name == "gcn":
            a = ActGCN(F_IN, HID, CLASSES, 3, 0.0, "relu", False, None, 1)
            b = GCN(F_IN, HID, CLASSES, 3, 0.0, "relu", False, None)
        elif name == "gcnii":
            a = GCNII(F_IN, HID, CLASSES, 4, dropout=0.0, actnn=True)
            b = GCNII(F_IN, HID, CLASSES, 4, dropout=0.0)
        else:
            a = SAGE(F_IN, CLASSES, HID, 2, aggr="mean", dropout=0.0, activation="relu", actnn=True)
            b = SAGE(F_IN, CLASSES, HID, 2, aggr="mean", dropout=0.0, activation="relu")
        b.load_state_dict(a.state_dict())
        return a.to(dev).train(), b.to(dev).train()

    for name in ("gcn", "gcnii", "sage"):
        config.activation_compression_bits, config.stochastic = [8], False
        a, b = pair(name)
        oa, ga = grads(a, fresh())
        ob, gb = grads(b, fresh())
        res[f"{name}_forward_equal"] = torch.equal(oa, ob)
        res[f"{name}_forward_rel"] = rel(oa, ob)
        res[f"{name}_grad8_rel"] = rel_all(ga, gb)
        res[f"{name}_grad8_rel_worst_param"] = max(rel(x, y) for x, y in zip(ga, gb))

        config.activation_compression_bits, config.stochastic = [2], True
        a, b = pair(name)
        torch.manual_seed(100)
        grads(a, fresh())                      # sets the gradient scales that weigh the bit allocation
        QScheme.update_scale = False
        _, gb = grads(b, fresh())
        runs = []
        for s in range(64):
            torch.manual_seed(s)
            runs.append(grads(a, fresh())[1])
        QScheme.update_scale = True
        one = rel_all(runs[0], gb)
        avg = rel_all([torch.stack([r[i] for r in runs]).mean(0) for i in range(len(gb))], gb)
        res[f"{name}_grad2_one_rel"], res[f"{name}_grad2_avg_rel"] = one, avg

    # saved-activation memory at an arxiv-sized shape: GCNII 16 x 256
    config.activation_compression_bits, config.stochastic, config.perlayer = [2], True, False
    kept = {}
    for tag, act in (("actnn", True), ("fp32", False)):
        big = make_graph(Graph, n=169343, e=583121, f=128, seed=9).to(dev)
        torch.manual_seed(0)
        m = GCNII(128, 256, 40, 16, dropout=0.5, actnn=act).to(dev).train()
        F.cross_entropy(m(big), big.y % 40).backward()   # first step: graph normalisation, allocator warm-up
        torch.cuda.synchronize()
        before = torch.cuda.memory_allocated()
        out = m(big)
        torch.cuda.synchronize()
        kept[tag] = torch.cuda.memory_allocated() - before - out.numel() * out.element_size()
        del out, m, big
    res["saved_bytes"] = kept
    res["saved_ratio"] = kept["actnn"] / kept["fp32"]

    cogdl_b200.uninstall_actnn()
    import sys

    res["uninstalled"] = "actnn" not in sys.modules
    print(json.dumps(res))


if __name__ == "__main__":
    main()

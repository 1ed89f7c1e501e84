"""Child process of tests/test_gpu_simple_hgn.py: the UNMODIFIED Simple-HGN layer of the reference (myGATConv, staged
by oracle/stage_examples.py at oracle/_ref/examples/simple_hgn/conv.py) through cogdl_b200.install_simple_hgn, against its
own original forward on the same GPU graph after cogdl_b200.install().  Runs in its own process because install()
rebinds the reference's dispatch for the rest of the process.

The graph is built from a shuffled COO and its CSR is built before the types are set in CSR order: the original
forward gathers its logits in edge_index order and its GPU edge_softmax builds the CSR, so it pairs logits with edges
only on a graph already in CSR order.  Two stacked layers (the second with res_attn and a residual Linear) and a
one-head output layer: the outputs, returned attentions and the gradients of x and of every parameter agree within
1e-5 of the largest magnitude."""
import os
import sys

import torch

from tests.refpkg import import_reference

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def main():
    import_reference()
    import cogdl_b200

    cogdl_b200.install()
    sys.path.insert(0, os.path.join(ROOT, "oracle", "_ref", "examples", "simple_hgn"))
    from cogdl.data import Graph
    from conv import myGATConv

    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(3)
    n, e, T = 500, 6000, 5
    row, col = torch.randint(0, n, (e,), generator=g), torch.randint(0, n, (e,), generator=g)
    etype = torch.randint(0, T, (e,), generator=g)
    graph = Graph(edge_index=(row, col), num_nodes=n).to(dev)
    graph.row_indptr
    graph.edge_type = etype[torch.sort(row, stable=True).indices].to(dev)
    torch.manual_seed(4)
    convs = [myGATConv(8, T, 32, 8, 8, attn_drop=0.0, residual=False, activation="relu"),
             myGATConv(8, T, 64, 8, 8, attn_drop=0.0, residual=True, activation="relu", alpha=0.05),
             myGATConv(8, T, 64, 4, 1, attn_drop=0.0)]
    convs = [c.to(dev) for c in convs]
    x0 = torch.randn(n, 32, generator=g).to(dev)

    def step():
        for c in convs:
            c.zero_grad()
        x = x0.clone().requires_grad_(True)
        o1, a1 = convs[0](graph, x)
        o2, a2 = convs[1](graph, o1, res_attn=a1)
        o3, a3 = convs[2](graph, o2)
        (o3.square().sum() + o2.sum()).backward()
        grads = [x.grad] + [p.grad.clone() for c in convs for p in c.parameters()]
        return [o1, a1, o2, a2, o3, a3], grads

    ref_out, ref_grads = step()
    cogdl_b200.install_simple_hgn(myGATConv)
    got_out, got_grads = step()
    errs = [rel(a, b) for a, b in zip(got_out + got_grads, ref_out + ref_grads)]
    assert max(errs) <= 1e-5, errs
    cogdl_b200.uninstall_simple_hgn(myGATConv)
    print("simple_hgn refpkg ok", max(errs))


if __name__ == "__main__":
    main()

"""Child process of tests/test_gpu_genconv_edge.py: the UNMODIFIED reference DeeperGCN (softmax_sg, learnable beta,
edge_attr_size=[8]) and a lone GENConv with an EdgeEncoder through cogdl_b200.install(genconv=True), against the
reference's own CPU run made before install and an fp64 restatement (as tests/genconv_refpkg_check.py).  A spy on
EdgeEncoder.forward shows the encoder is folded into the kernels; a BondEncoder layer and edge features that require
grad show the edge-term kernels still take the cases the fused path does not.  Prints one JSON line."""
import copy
import json

import torch

from tests.genconv_ref import genconv_aggregate_fp64
from tests.refpkg import import_reference
from tests.test_gpu_refpkg import cora_shaped_graph, rel


def main():
    import_reference()
    from cogdl.data import Graph
    from cogdl.layers import GENConv
    from cogdl.layers.deepergcn_layer import EdgeEncoder
    from cogdl.models.nn.deepergcn import DeeperGCN

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    g_cpu = cora_shaped_graph(Graph, feats=64)
    g_cpu.row_indptr                                  # CSR order (edge_attr is permuted with it)
    n, nnz = g_cpu.num_nodes, g_cpu.col_indices.numel()
    g_cpu.edge_attr = torch.rand(nnz, 8, generator=torch.Generator().manual_seed(2))
    target = torch.randint(0, 7, (n,), generator=torch.Generator().manual_seed(1))
    rp, ci = g_cpu.row_indptr, g_cpu.col_indices

    def fp64_forward(self, graph, x):
        a = self.edge_encoder(graph.edge_attr)
        h = genconv_aggregate_fp64(rp, ci, x, self.aggr, beta=self.beta, eps=self.eps, edge_term=a)
        return self.mlp(h + x if self.residual else h)

    makers = {
        "deepergcn": lambda: DeeperGCN(64, 32, 7, 3, aggr="softmax_sg", beta=1.0, learn_beta=True, edge_attr_size=[8]),
        "genconv_edge": lambda: torch.nn.Sequential(GENConv(64, 7, aggr="softmax_sg", beta=0.7, learn_beta=True,
                                                            edge_attr_size=[8])),
    }

    def run(model, graph):
        model.zero_grad(set_to_none=True)
        out = model(graph) if not isinstance(model, torch.nn.Sequential) else model[0](graph, graph.x)
        torch.nn.functional.cross_entropy(out, target.to(out.device)).backward()
        return out.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}

    ref, exact, states = {}, {}, {}
    original = GENConv.forward
    for name, make in makers.items():
        torch.manual_seed(5)
        model = make().train()
        states[name] = copy.deepcopy(model.state_dict())
        ref[name] = run(model, copy.deepcopy(g_cpu))[0]
        m64 = make().double().train()
        m64.load_state_dict(states[name])
        g64 = copy.deepcopy(g_cpu)
        g64.x, g64.edge_attr = g64.x.double(), g64.edge_attr.double()
        GENConv.forward = fp64_forward
        try:
            exact[name] = run(m64, g64)
        finally:
            GENConv.forward = original

    import cogdl_b200
    from cogdl_b200 import _cabi

    cogdl_b200.install(genconv=True)
    calls = []
    encoder_forward = EdgeEncoder.forward

    def spy(self, edge_attr):
        calls.append(tuple(edge_attr.shape))
        return encoder_forward(self, edge_attr)

    EdgeEncoder.forward = spy
    dev = torch.device("cuda:0")
    result = {}
    for name, make in makers.items():
        torch.manual_seed(5)
        model = make()
        model.load_state_dict(states[name])
        model = model.to(dev).train()
        graph = copy.deepcopy(g_cpu).to(dev)
        calls.clear()
        out, grads = run(model, graph)
        gscale = max(float(g.abs().max()) for g in exact[name][1].values())
        result[name] = {
            "grad_errs_model_scale": {k: float((grads[k].double().cpu() - g).abs().max()) / gscale
                                      for k, g in exact[name][1].items()},
            "logits_vs_ref_cpu": rel(out, ref[name]),
            "logits_vs_fp64": rel(out, exact[name][0]),
            "grad_errs": {k: rel(grads[k], exact[name][1][k]) for k in exact[name][1]},
            "grads_present": sorted(grads) == sorted(exact[name][1]),
            "edge_encoder_calls": len(calls),
            "last_kernel": _cabi.last_kernel(),
        }

    # cases the fused path does not take: the layer's own encoder runs and the edge-term kernel aggregates
    graph = copy.deepcopy(g_cpu).to(dev)
    x = graph.x
    bond = GENConv(64, 7, aggr="softmax_sg", edge_attr_size=[4, 3]).to(dev)
    g_bond = copy.deepcopy(graph)
    g_bond.edge_attr = torch.stack([torch.arange(nnz) % 4, torch.arange(nnz) % 3], 1).to(dev)
    bond(g_bond, x)
    result["bond_encoder"] = {"last_kernel": _cabi.last_kernel()}
    trainable = GENConv(64, 7, aggr="softmax_sg", edge_attr_size=[8]).to(dev)
    g_tr = copy.deepcopy(graph)
    g_tr.edge_attr = g_tr.edge_attr.clone().requires_grad_(True)
    calls.clear()
    trainable(g_tr, x).sum().backward()
    fwd_kernel = _cabi.last_kernel()
    trainable(g_tr, x)
    result["attr_requires_grad"] = {"last_kernel": _cabi.last_kernel(), "encoder_calls": len(calls),
                                    "attr_grad": g_tr.edge_attr.grad is not None, "after_backward": fwd_kernel}
    for case in ("bond_encoder", "attr_requires_grad"):
        result[case]["edge_term_kernel"] = ",edge_term," in result[case]["last_kernel"]
    EdgeEncoder.forward = encoder_forward
    print(json.dumps(result))


if __name__ == "__main__":
    main()

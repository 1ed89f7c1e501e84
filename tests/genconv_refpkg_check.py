"""Child process of tests/test_gpu_genconv.py: the UNMODIFIED reference DeeperGCN (softmax_sg) and a GENConv with an
EdgeEncoder through cogdl_b200.install(genconv=True), against the reference's own CPU run made before install.
Runs in its own process because install() rebinds the reference's dispatch for the rest of the process (the CPU
phase of tests/test_gpu_refpkg.py must not see that).  Prints one JSON line of measured errors.

Parameter gradients are compared with an fp64 restatement (tests/genconv_ref.py in place of the aggregation, the
model's own layers around it): the reference's CPU edge-softmax backward is inexact (DESIGN.md section 3.8).
"""
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
    from cogdl.models.nn.deepergcn import DeeperGCN

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    g_cpu = cora_shaped_graph(Graph, feats=64)
    g_cpu.row_indptr                                  # CSR order (edge_attr is permuted with it)
    n, nnz = g_cpu.num_nodes, g_cpu.col_indices.numel()
    g_cpu.edge_attr = torch.rand(nnz, 5, generator=torch.Generator().manual_seed(2))
    target = torch.randint(0, 7, (n,), generator=torch.Generator().manual_seed(1))
    rp, ci = g_cpu.row_indptr, g_cpu.col_indices

    def fp64_forward(self, graph, x):
        a = self.edge_encoder(graph.edge_attr) if self.edge_encoder is not None and graph.edge_attr is not None else None
        h = genconv_aggregate_fp64(rp, ci, x, self.aggr, beta=self.beta, eps=self.eps, edge_term=a)
        return self.mlp(h + x if self.residual else h)

    makers = {
        "deepergcn": lambda: DeeperGCN(64, 32, 7, 3, aggr="softmax_sg", beta=1.0, learn_beta=True),
        "genconv_edge": lambda: torch.nn.Sequential(GENConv(64, 7, aggr="softmax_sg", beta=0.7, learn_beta=True,
                                                            edge_attr_size=[5])),
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
    from cogdl_b200.install import genconv_forward

    result = {"untouched_without_flag": None}
    cogdl_b200.install()
    result["untouched_without_flag"] = GENConv.forward is original
    patched = cogdl_b200.install(genconv=True)
    result["patched"] = patched
    result["rebound"] = GENConv.forward is genconv_forward and GENConv._cogdl_b200_original_forward is original
    dev = torch.device("cuda:0")
    for name, make in makers.items():
        torch.manual_seed(5)
        model = make()
        model.load_state_dict(states[name])
        model = model.to(dev).train()
        graph = copy.deepcopy(g_cpu).to(dev)
        out, grads = run(model, graph)
        gscale = max(float(g.abs().max()) for g in exact[name][1].values())
        result[name] = {
            "grad_errs_model_scale": {k: float((grads[k].double().cpu() - g).abs().max()) / gscale
                                      for k, g in exact[name][1].items()},
            "logits_vs_ref_cpu": rel(out, ref[name]),
            "logits_vs_fp64": rel(out, exact[name][0]),
            "grad_errs": {k: rel(grads[k], exact[name][1][k]) for k in exact[name][1]},
            "grads_present": sorted(grads) == sorted(exact[name][1]),
        }

    # uncovered case: max with an edge encoder must go to the original forward
    calls = []

    def spy(self, graph, x):
        calls.append(self.aggr)
        return original(self, graph, x)

    GENConv._cogdl_b200_original_forward = spy
    conv = GENConv(64, 7, aggr="max", edge_attr_size=[5]).to(dev)
    try:
        conv(copy.deepcopy(g_cpu).to(dev), g_cpu.x.to(dev))
    except Exception as e:  # the reference's own max path; only the dispatch decision is under test
        result["max_edge_original_error"] = type(e).__name__
    GENConv._cogdl_b200_original_forward = original
    result["max_edge_ran_original"] = calls == ["max"]
    print(json.dumps(result))


if __name__ == "__main__":
    main()

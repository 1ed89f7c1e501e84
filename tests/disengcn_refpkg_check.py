"""Child process of tests/test_gpu_disengcn.py: the UNMODIFIED reference DisenGCN (K = [16, 8], hidden 64, 7
iterations) through cogdl_b200.install(disengcn=True), against the reference's own CPU run made before install.
Runs in its own process because install() rebinds the reference's dispatch for the rest of the process.  Prints one
JSON line of measured errors.

Parameter gradients are compared with an fp64 restatement (tests/disengcn_ref.py in place of the routing, the
layer's own weight, bias and activation around it): the reference's CPU edge-softmax backward is inexact
(DESIGN.md section 3.8).  Dropout is 0 so the CPU and GPU runs see the same network.
"""
import copy
import json

import torch

from tests.disengcn_ref import disen_routing_fp64
from tests.refpkg import import_reference
from tests.test_gpu_refpkg import cora_shaped_graph, rel


def main():
    import_reference()
    from cogdl.data import Graph
    from cogdl.layers import DisenGCNLayer
    from cogdl.models.nn.disengcn import DisenGCN

    torch.backends.cuda.matmul.allow_tf32 = False
    torch.manual_seed(0)
    g_cpu = cora_shaped_graph(Graph, feats=64)
    n = g_cpu.num_nodes
    target = torch.randint(0, 7, (n,), generator=torch.Generator().manual_seed(1))

    def make():
        return DisenGCN(64, 64, 7, K=[16, 8], iterations=7, tau=1.0, dropout=0.0, activation="leaky_relu")

    def run(model, graph):
        model.zero_grad(set_to_none=True)
        out = model(graph)
        torch.nn.functional.cross_entropy(out, target.to(out.device)).backward()
        return out.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}

    def fp64_forward(self, graph, x):
        h = self.activation(torch.matmul(x, self.weight) + self.bias)
        return disen_routing_fp64(graph.row_indptr, graph.col_indices, h, self.K, self.iterations, self.tau)

    original = DisenGCNLayer.forward
    torch.manual_seed(5)
    model = make().train()
    state = copy.deepcopy(model.state_dict())
    ref_logits = run(model, copy.deepcopy(g_cpu))[0]
    m64 = make().double().train()
    m64.load_state_dict(state)
    g64 = copy.deepcopy(g_cpu)
    g64.x = g64.x.double()
    DisenGCNLayer.forward = fp64_forward
    try:
        exact_logits, exact_grads = run(m64, g64)
    finally:
        DisenGCNLayer.forward = original

    import cogdl_b200
    from cogdl_b200 import structure
    from cogdl_b200.install import disengcn_forward, uninstall_disengcn

    result = {}
    cogdl_b200.install()
    result["untouched_without_flag"] = DisenGCNLayer.forward is original
    result["patched"] = cogdl_b200.install(disengcn=True)
    result["rebound"] = DisenGCNLayer.forward is disengcn_forward and DisenGCNLayer._cogdl_b200_original_forward is original
    dev = torch.device("cuda:0")
    model = make()
    model.load_state_dict(state)
    model = model.to(dev).train()
    graph = copy.deepcopy(g_cpu).to(dev)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    misses = []
    for step in range(3):
        before = structure.cache_stats["miss"]
        out, grads = run(model, graph)
        misses.append(structure.cache_stats["miss"] - before)
        if step == 0:
            result["logits_vs_ref_cpu"] = rel(out, ref_logits)
            result["logits_vs_fp64"] = rel(out, exact_logits)
            result["grad_errs"] = {k: rel(grads[k], g) for k, g in exact_grads.items()}
            result["grads_present"] = sorted(grads) == sorted(exact_grads)
        opt.step()
    result["misses_per_step"] = misses

    # uncovered cases go to the original forward: CPU input, and a channel width without a kernel (d = 3)
    calls = []

    def spy(tag):
        def fwd(self, graph, x):
            calls.append(tag)
            return original(self, graph, x)
        return fwd

    layer = DisenGCNLayer(64, 32, 8, 2)
    DisenGCNLayer._cogdl_b200_original_forward = spy("cpu")
    try:
        layer(copy.deepcopy(g_cpu), g_cpu.x)
    except Exception as e:  # after install() the reference's edge_softmax is ours, which has no CPU path
        result["cpu_original_error"] = type(e).__name__
    layer3 = DisenGCNLayer(64, 24, 8, 2).to(dev)
    DisenGCNLayer._cogdl_b200_original_forward = spy("d3")
    try:
        layer3(copy.deepcopy(g_cpu).to(dev), g_cpu.x.to(dev))
    except Exception as e:  # the reference's own GPU path; only the dispatch decision is under test
        result["d3_original_error"] = type(e).__name__
    DisenGCNLayer._cogdl_b200_original_forward = original
    result["uncovered_ran_original"] = calls
    uninstall_disengcn()
    result["restored"] = DisenGCNLayer.forward is original
    print(json.dumps(result))


if __name__ == "__main__":
    main()

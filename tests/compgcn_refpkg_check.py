"""Child process of tests/test_gpu_compgcn.py: the UNMODIFIED reference LinkPredictCompGCN (2 layers, hidden 32, sub and
mult) through cogdl_b200.install(compgcn=True), against the reference's own CPU run made before install.  Runs in its
own process because install() rebinds the reference's dispatch for the rest of the process.  Prints one JSON line of
measured errors.

Parameter gradients are compared with an fp64 restatement (tests/compgcn_ref.py) of the whole model.  Gradients that
are exactly zero in exact arithmetic (training-mode BN cancels any shift shared by all rows: the layer biases, and
loop_rel under sub) are compared in absolute terms against the scale of the model's gradients instead.
"""
import copy
import json

import numpy as np
import torch

from tests.compgcn_ref import compgcn_layer_fp64
from tests.refpkg import import_reference
from tests.test_gpu_refpkg import rel

N_ENT, N_REL, TRIPLES, HIDDEN = 400, 6, 2500, 32


def make_kg():
    """Triples plus their reverses (type t + N_REL), shuffled COO on the host."""
    g = torch.Generator().manual_seed(31)
    h = torch.randint(0, N_ENT, (TRIPLES,), generator=g)
    t = torch.randint(0, N_ENT, (TRIPLES,), generator=g)
    r = torch.randint(0, N_REL, (TRIPLES,), generator=g)
    row, col, typ = torch.cat([h, t]), torch.cat([t, h]), torch.cat([r, r + N_REL])
    perm = torch.randperm(row.numel(), generator=g)
    return row[perm], col[perm], typ[perm]


def fp64_model(model, graph):
    """(node_embed, rel_embed) of LinkPredictCompGCN.predict in fp64, with a leaf per parameter."""
    params = {k: p.detach().double().requires_grad_(True) for k, p in model.named_parameters()}
    row, col = graph.edge_index
    x, rel_embed = params["emb.weight"], params["model.init_rel.weight"]
    for i, layer in enumerate(model.model.convs):
        pre = f"model.convs.{i}."
        p = {k[len(pre):]: v for k, v in params.items() if k.startswith(pre)}
        x, rel_embed = compgcn_layer_fp64(p, row, col, graph.edge_attr, x, rel_embed, layer.opn)
    return x, rel_embed, params


def main():
    import_reference()
    from cogdl.data import Graph
    from cogdl.models.nn.compgcn import CompGCNLayer, LinkPredictCompGCN
    from cogdl.utils.link_prediction_utils import DistMultLayer

    torch.backends.cuda.matmul.allow_tf32 = False
    row, col, typ = make_kg()
    g_cpu = Graph(edge_index=(row, col), edge_attr=typ)
    gen = torch.Generator().manual_seed(32)
    G, GR = torch.randn(N_ENT, HIDDEN, generator=gen), torch.randn(2 * N_REL, HIDDEN, generator=gen)
    scoring = DistMultLayer()

    def make(opn, dropout=0.0):
        torch.manual_seed(5)
        return LinkPredictCompGCN(N_ENT, N_REL, HIDDEN, layers=2, dropout=dropout, opn=opn, sampling_rate=0.2)

    def predict_grads(model, graph):
        model.zero_grad(set_to_none=True)
        node, relo = model.predict(graph)
        ((node * G.to(node.device)).sum() + (relo * GR.to(node.device)).sum()).backward()
        return node.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}

    def run_loss(model, graph):
        np.random.seed(7)
        torch.manual_seed(7)
        return model.loss(graph, scoring).detach()

    original = CompGCNLayer.forward
    ref = {}
    for opn in ("sub", "mult"):
        model = make(opn).train()
        node, grads = predict_grads(model, copy.deepcopy(g_cpu))
        ref[opn] = {"state": copy.deepcopy(model.state_dict()), "node": node}
        with torch.no_grad():            # before loss(), whose training-mode BN moves the running statistics
            ref[opn]["eval"] = model.eval().predict(copy.deepcopy(g_cpu))[0]
        ref[opn]["loss"] = run_loss(model.train(), copy.deepcopy(g_cpu))
        m64 = make(opn).train()
        m64.load_state_dict(ref[opn]["state"])
        node64, rel64, params = fp64_model(m64, g_cpu)
        ((node64 * G.double()).sum() + (rel64 * GR.double()).sum()).backward()
        ref[opn]["exact_grads"] = {k: p.grad for k, p in params.items() if p.grad is not None}
        ref[opn]["exact_node"] = node64.detach()

    import cogdl_b200
    from cogdl_b200 import structure
    from cogdl_b200.install import compgcn_forward, uninstall_compgcn

    result = {}
    cogdl_b200.install()
    result["untouched_without_flag"] = CompGCNLayer.forward is original
    result["patched"] = cogdl_b200.install(compgcn=True)
    result["rebound"] = CompGCNLayer.forward is compgcn_forward and CompGCNLayer._cogdl_b200_original_forward is original
    dev = torch.device("cuda:0")
    errs = {"predict_vs_ref_cpu": 0.0, "loss_vs_ref_cpu": 0.0, "node_vs_fp64": 0.0}
    grad_errs, zero_grads = {}, {}
    present = True
    untouched = True
    built = []
    for opn in ("sub", "mult"):
        model = make(opn)
        model.load_state_dict(ref[opn]["state"])
        model = model.to(dev).train()
        graph = copy.deepcopy(g_cpu).to(dev)
        edges_before = [t.clone() for t in graph.edge_index]
        before = structure.comp_cache_stats["miss"]
        node, grads = predict_grads(model, graph)
        built.append(structure.comp_cache_stats["miss"] - before)
        untouched &= all(torch.equal(a, b) for a, b in zip(graph.edge_index, edges_before))
        untouched &= graph._adj.row_ptr is None
        errs["node_vs_fp64"] = max(errs["node_vs_fp64"], rel(node, ref[opn]["exact_node"]))
        exact = ref[opn]["exact_grads"]
        present &= sorted(grads) == sorted(exact)
        scale = max(float(g.abs().max()) for g in exact.values())
        for k, g in exact.items():
            if float(g.abs().max()) < 1e-12:
                zero_grads[f"{opn}:{k}"] = float(grads[k].abs().max()) / scale
            else:
                grad_errs[f"{opn}:{k}"] = rel(grads[k], g)
        before = structure.comp_cache_stats["miss"]
        model.load_state_dict(ref[opn]["state"])    # BN running statistics as the reference's eval run saw them
        with torch.no_grad():
            errs["predict_vs_ref_cpu"] = max(errs["predict_vs_ref_cpu"], rel(model.eval().predict(graph)[0], ref[opn]["eval"]))
        built.append(structure.comp_cache_stats["miss"] - before)    # a second predict() on the graph: no build
        model.train()
        errs["loss_vs_ref_cpu"] = max(errs["loss_vs_ref_cpu"], rel(run_loss(model, copy.deepcopy(g_cpu).to(dev)),
                                                                   ref[opn]["loss"]))
    result.update(errs)
    result["grad_errs"] = grad_errs
    result["zero_grads_vs_scale"] = zero_grads
    result["grads_present"] = present
    result["graph_untouched"] = untouched
    result["structures_built_2layer"] = built[0]
    result["structures_rebuilt_on_repeat"] = max(built[1::2])

    # dropout > 0: under one seed the fused and the original GPU forward draw the same masks
    model = make("mult", dropout=0.3)
    model.load_state_dict(ref["mult"]["state"])
    model = model.to(dev).train()
    graph = copy.deepcopy(g_cpu).to(dev)
    torch.manual_seed(11)
    fused = model.predict(graph)[0].detach()
    CompGCNLayer.forward = original
    try:
        torch.manual_seed(11)
        plain = model.predict(graph)[0].detach()
    finally:
        CompGCNLayer.forward = compgcn_forward
    result["dropout_fused_vs_original_gpu"] = rel(fused, plain)

    # uncovered cases go to the original forward: CPU input, and an opn without a kernel
    calls = []

    def spy(tag):
        def fwd(self, *a):
            calls.append(tag)
            return original(self, *a)
        return fwd

    layer = CompGCNLayer(16, 8, N_REL, opn="sub")
    x_cpu, rel_cpu = torch.randn(N_ENT, 16), torch.randn(2 * N_REL, 16)
    CompGCNLayer._cogdl_b200_original_forward = spy("cpu")
    layer(copy.deepcopy(g_cpu), x_cpu, rel_cpu)
    layer_corr = CompGCNLayer(16, 8, N_REL, opn="corr").to(dev)
    CompGCNLayer._cogdl_b200_original_forward = spy("corr")
    try:
        layer_corr(copy.deepcopy(g_cpu).to(dev), x_cpu.to(dev), rel_cpu.to(dev))
    except NotImplementedError:
        pass
    CompGCNLayer._cogdl_b200_original_forward = original
    result["uncovered_ran_original"] = calls
    uninstall_compgcn()
    result["restored"] = CompGCNLayer.forward is original
    print(json.dumps(result))


if __name__ == "__main__":
    main()

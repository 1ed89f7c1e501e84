"""Child process of tests/test_gpu_rgcn.py: the UNMODIFIED reference RGCN and LinkPredictRGCN through
cogdl_b200.install(rgcn=True).  Runs in its own process because install() rebinds the reference's dispatch for the rest
of the process.  Prints one JSON line of measured errors.

  * T = 1, where the reference's indentation bug has no effect: RGCN (2 layers, basis) on the GPU against the
    reference's own CPU run made before install -- the output and every parameter gradient.
  * T > 1: LinkPredictRGCN.predict() (2 layers, num_bases < T) against the fp64 relational sum (tests/rgcn_ref.py) of
    the same parameters -- output and parameter gradients -- on a shuffled-COO cogdl.data.Graph, so each edge type
    must stay paired with its edge through the graph's CSR build.  One loss() step runs and builds one structure.
"""
import copy
import json

import numpy as np
import torch

from tests.refpkg import import_reference
from tests.rgcn_ref import rgcn_layer_fp64, row_norm_weights

N_ENT, N_REL, TRIPLES, HIDDEN, BASES = 300, 6, 2000, 32, 3


def rel(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp_min(1e-30))


def make_kg(n_rel):
    g = torch.Generator().manual_seed(41)
    h = torch.randint(0, N_ENT, (TRIPLES,), generator=g)
    t = torch.randint(0, N_ENT, (TRIPLES,), generator=g)
    r = torch.randint(0, n_rel, (TRIPLES,), generator=g)
    perm = torch.randperm(TRIPLES, generator=g)
    return h[perm], t[perm], r[perm]


def on_gpu(graph, dev):
    """A copy of graph on dev.  Graph.to() leaves edge_attr where it was (cogdl/data/data.py), so it is moved here."""
    g = copy.deepcopy(graph).to(dev)
    g.edge_attr = g.edge_attr.to(dev)
    return g


def grads_of(model, run, G):
    model.zero_grad(set_to_none=True)
    out = run()
    (out * G.to(out.device)).sum().backward()
    return out.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}


def main():
    import_reference()
    from cogdl.data import Graph
    from cogdl.layers.rgcn_layer import RGCNLayer
    from cogdl.models.nn.rgcn import RGCN, LinkPredictRGCN
    from cogdl.utils.link_prediction_utils import DistMultLayer

    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    gen = torch.Generator().manual_seed(42)
    G = torch.randn(N_ENT, HIDDEN, generator=gen)
    x0 = torch.randn(N_ENT, HIDDEN, generator=gen)

    # ---- reference runs before install
    h1, t1, r1 = make_kg(1)
    g1 = Graph(edge_index=(h1, t1), edge_attr=r1, x=x0)
    torch.manual_seed(5)
    m1 = RGCN(HIDDEN, HIDDEN, 2, 1, "basis", None)
    ref1_out, ref1_grads = grads_of(m1, lambda: m1(copy.deepcopy(g1), x0), G)
    state1 = copy.deepcopy(m1.state_dict())

    hn, tn, rn = make_kg(N_REL)
    gn = Graph(edge_index=(hn, tn), edge_attr=rn)
    torch.manual_seed(6)
    mn = LinkPredictRGCN(N_ENT, N_REL, HIDDEN, 2, "basis", BASES, sampling_rate=0.2)
    staten = copy.deepcopy(mn.state_dict())

    # fp64 relational sum of predict(), with a leaf per parameter
    params = {k: p.detach().double().requires_grad_(True) for k, p in mn.named_parameters()}
    w_hat = row_norm_weights(hn, N_ENT)
    h = params["emb.weight"]
    for i in range(2):
        pre = f"model.layers.{i}."
        p = {k[len(pre):]: v for k, v in params.items() if k.startswith(pre)}
        h = rgcn_layer_fp64(p, hn, tn, rn, w_hat, h, N_REL)
        if i < 1:
            h = torch.relu(h)
    (h * G.double()).sum().backward()
    exact_out, exact_grads = h.detach(), {k: p.grad for k, p in params.items() if p.grad is not None}

    import cogdl_b200
    from cogdl_b200 import structure
    from cogdl_b200.install import rgcn_forward, uninstall_rgcn

    original = RGCNLayer.forward
    result = {}
    cogdl_b200.install()
    result["untouched_without_flag"] = RGCNLayer.forward is original
    result["patched"] = cogdl_b200.install(rgcn=True)
    result["rebound"] = RGCNLayer.forward is rgcn_forward and RGCNLayer._cogdl_b200_original_forward is original

    m1g = RGCN(HIDDEN, HIDDEN, 2, 1, "basis", None)
    m1g.load_state_dict(state1)
    m1g = m1g.to(dev)
    out1, grads1 = grads_of(m1g, lambda: m1g(on_gpu(g1, dev), x0.to(dev)), G)
    t1 = {"out": rel(out1, ref1_out)}
    t1.update({k: rel(grads1[k], g) for k, g in ref1_grads.items()})
    result["t1_vs_ref_cpu"] = t1
    present = sorted(grads1) == sorted(ref1_grads)

    mng = LinkPredictRGCN(N_ENT, N_REL, HIDDEN, 2, "basis", BASES, sampling_rate=0.2)
    mng.load_state_dict(staten)
    mng = mng.to(dev)
    gdev = on_gpu(gn, dev)
    outn, gradsn = grads_of(mng, lambda: mng.predict(gdev)[0], G)
    tnr = {"out": rel(outn, exact_out)}
    tnr.update({k: rel(gradsn[k], g) for k, g in exact_grads.items()})
    result["tn_vs_fp64"] = tnr
    present &= sorted(gradsn) == sorted(exact_grads)
    result["grads_present"] = bool(present)

    np.random.seed(7)
    torch.manual_seed(7)
    before = structure.rgcn_cache_stats["miss"]
    loss = mng.loss(on_gpu(gn, dev), DistMultLayer())
    loss.backward()
    result["structures_built_per_step"] = structure.rgcn_cache_stats["miss"] - before
    result["loss_finite"] = bool(torch.isfinite(loss).item())

    # uncovered cases run the original forward: CPU input, and a regularizer other than basis
    calls = []

    def spy(tag):
        def fwd(self, *a):
            calls.append(tag)
            return original(self, *a)
        return fwd

    layer = RGCNLayer(HIDDEN, HIDDEN, N_REL, "basis", BASES)
    RGCNLayer._cogdl_b200_original_forward = spy("cpu")
    try:
        layer(copy.deepcopy(gn), x0)
    except RuntimeError:       # install() rebinds the reference's spmm to this package's, which has no CPU path
        pass
    layer_b = RGCNLayer(HIDDEN, HIDDEN, N_REL, "basis", BASES).to(dev)
    layer_b.regularizer = "bdd"
    RGCNLayer._cogdl_b200_original_forward = spy("bdd")
    try:
        layer_b(on_gpu(gn, dev), x0.to(dev))
    except AttributeError:     # the reference's bdd path cannot run on a basis layer's parameters
        pass
    RGCNLayer._cogdl_b200_original_forward = original
    result["fallbacks"] = calls
    uninstall_rgcn()
    result["restored"] = RGCNLayer.forward is original
    print(json.dumps(result))


if __name__ == "__main__":
    main()

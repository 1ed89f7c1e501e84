"""Child process of tests/test_gpu_gcnii.py: the UNMODIFIED reference GCNII (8 layers x 64, residual off and on) and
PPNP (appnp, K = 10) through cogdl_b200.install(gcnii=True, appnp=True), with the parameters and graphs of
tests/golden/gcnii_appnp.npz.  Runs in its own process because install() rebinds the reference's dispatch for the rest
of the process.  Prints one JSON line of measured errors.

Graphs: one built from CSR (sym_norm sets in_norm / out_norm, which the kernel applies as its row scale) and one from
edge_index (sym_norm rescales the edge weights).  Checked, in eval mode: the logits against the reference's CPU logits
of the golden file, and every parameter gradient (upstream gradient G of the file) against the fp64 restatement
tests/gcnii_ref.py, which tests/test_cpu_gcnii_golden.py pins to the reference.  In training mode: a seeded forward and
its gradients against the unfused forward on the GPU (the original forwards on this package's spmm): the same dropout
masks, since a different mask would differ by O(1).  Also: install() without the flags leaves both forwards alone, and
uninstall restores them.
"""
import copy
import json
import os

import numpy as np
import torch

from tests.refpkg import import_reference
from tests.test_cpu_gcnii_golden import GOLDEN, restated
from tests.test_gpu_refpkg import rel

F_IN, HID, C = 24, 64, 7


def make_graph(Graph, d, built_from):
    rp, col, x = (torch.from_numpy(d[k]) for k in ("rowptr", "col", "x"))
    if built_from == "csr":
        return Graph(x=x.clone(), row_ptr=rp.clone(), col=col.clone())
    row = torch.repeat_interleave(torch.arange(rp.shape[0] - 1), rp[1:] - rp[:-1])
    return Graph(x=x.clone(), edge_index=(row, col.clone()))


def run(model, graph, G, train=False, seed=None):
    """(logits, {name: grad}) of sum(logits * G)."""
    model.train(train)
    model.zero_grad(set_to_none=True)
    if seed is not None:
        torch.manual_seed(seed)
    out = model(graph)
    (out * G.to(out.device)).sum().backward()
    return out.detach(), {k: p.grad.detach().clone() for k, p in model.named_parameters() if p.grad is not None}


def main():
    import_reference()
    from cogdl.data import Graph
    from cogdl.layers.gcnii_layer import GCNIILayer
    from cogdl.models.nn.gcnii import GCNII
    from cogdl.models.nn.ppnp import PPNP

    import cogdl_b200

    torch.backends.cuda.matmul.allow_tf32 = False
    dev = torch.device("cuda:0")
    d = np.load(GOLDEN)
    G = torch.from_numpy(d["G"])

    base = {}
    for res in (False, True):
        base[f"gcnii_res{int(res)}"] = GCNII(F_IN, HID, C, 8, dropout=0.5, alpha=0.1, lmbda=0.5, residual=res)
    base["appnp"] = PPNP(F_IN, HID, C, 2, 0.5, "appnp", 0.1, 10)
    for m, model in base.items():
        model.load_state_dict({k: torch.from_numpy(d[f"p_{m}_{k}"]) for k, _ in model.named_parameters()})

    orig_gcnii, orig_ppnp = GCNIILayer.forward, PPNP.forward
    cogdl_b200.install()
    res = {"untouched_without_flag": GCNIILayer.forward is orig_gcnii and PPNP.forward is orig_ppnp}
    unfused = {(m, gk): run(copy.deepcopy(model).to(dev), make_graph(Graph, d, gk).to(dev), G, train=True, seed=77)
               for m, model in base.items() for gk in ("csr", "coo")}
    patched = cogdl_b200.install(gcnii=True, appnp=True)
    res["patched"] = patched[-2:]
    res["rebound"] = GCNIILayer.forward is not orig_gcnii and PPNP.forward is not orig_ppnp
    res["logits_vs_golden"], res["grads_vs_fp64"], res["train_logits"], res["train_grads"] = {}, {}, {}, {}
    for m, model in base.items():
        for gk in ("csr", "coo"):
            key = f"{m}_{gk}"
            md = copy.deepcopy(model).to(dev)
            out, grads = run(md, make_graph(Graph, d, gk).to(dev), G)
            res["logits_vs_golden"][key] = rel(out, torch.from_numpy(d[f"y_{m}_{gk}"]))
            _, g64 = restated(d, m, gk)
            res["grads_vs_fp64"][key] = max(rel(grads[k], torch.from_numpy(g64[k])) for k in g64)
            out, grads = run(md, make_graph(Graph, d, gk).to(dev), G, train=True, seed=77)
            u_out, u_grads = unfused[(m, gk)]
            res["train_logits"][key] = rel(out, u_out)
            res["train_grads"][key] = max(rel(grads[k], u_grads[k]) for k in u_grads)
    cogdl_b200.uninstall_gcnii()
    cogdl_b200.uninstall_appnp()
    res["restored"] = GCNIILayer.forward is orig_gcnii and PPNP.forward is orig_ppnp
    print(json.dumps(res))


if __name__ == "__main__":
    main()

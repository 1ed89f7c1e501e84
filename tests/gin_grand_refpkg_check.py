"""Child process of tests/test_gpu_gin_grand.py: the UNMODIFIED reference GINLayer, GINELayer, GIN and Grand through
cogdl_b200.install(gin=True, grand=True), on the graph of tests/golden/gin_grand.npz and on a batch of synthetic
graphs.  Runs in its own process because install() rebinds the reference's dispatch for the rest of the process.
Prints one JSON line.

Checked: the layers' outputs and d x, d eps, Grand.rand_prop (train, at the same seed, and eval, for every order) and
Grand.forward are bit-identical to the same reference code after install() without the flags (its loops on this
package's spmm) and within 1e-5 of the reference's CPU results; the GIN model's logits and gradients on a batch of
graphs agree within 1e-5 of the largest of their magnitudes (its sum pooling is a scatter_add_ with atomics, so
not bit for bit); the fused kernels ran;
install() without the flags leaves the originals alone, uninstall_gin() / uninstall_grand() restore them, and CPU or
fp64 features go to the originals.
"""
import json

import numpy as np
import torch

from tests.refpkg import import_reference
from tests.test_cpu_gin_grand_golden import DROPNODE, GIN_CASES, GOLDEN, ORDERS, SEED, rel


def golden_graph(Graph, d, dev):
    g = Graph(x=torch.from_numpy(d["x"]).clone(), edge_index=(torch.from_numpy(d["row"]).clone(),
                                                              torch.from_numpy(d["col"]).clone())).to(dev)
    g.row_indptr
    return g


def batch_graph(Graph, dev, n_graphs=6, seed=5):
    """n_graphs random symmetric graphs of 20-60 nodes as one disjoint union, with `batch` (as the GIN model reads it)."""
    rng = np.random.default_rng(seed)
    rows, cols, batch, off = [], [], [], 0
    for b in range(n_graphs):
        n = int(rng.integers(20, 60))
        e = int(rng.integers(2 * n, 5 * n))
        r, c = rng.integers(0, n, e), rng.integers(0, n, e)
        rows += [r + off, c + off]
        cols += [c + off, r + off]
        batch.append(np.full(n, b))
        off += n
    x = torch.from_numpy(rng.standard_normal((off, 8)).astype(np.float32))
    g = Graph(x=x, edge_index=(torch.from_numpy(np.concatenate(rows)), torch.from_numpy(np.concatenate(cols))),
              y=torch.from_numpy(rng.integers(0, 4, n_graphs)))
    g.batch = torch.from_numpy(np.concatenate(batch))
    g = g.to(dev)
    g.row_indptr
    return g


def run_all(Graph, d, dev):
    import cogdl_b200
    from cogdl.layers import GINELayer, GINLayer
    from cogdl.models.nn.gin import GIN
    from cogdl.models.nn.grand import Grand

    out, kernels = {}, {}
    G = torch.from_numpy(d["g"]).to(dev)
    for key, eps, train in GIN_CASES:
        layer = (GINELayer if key == "gine" else GINLayer)(None, eps, train).to(dev)
        x = torch.from_numpy(d["x"]).to(dev).requires_grad_(True)
        y = layer(golden_graph(Graph, d, dev), x)
        kernels[key] = cogdl_b200._cabi.last_kernel()
        y.backward(G)
        out[f"{key}_out"], out[f"{key}_dx"] = y.detach(), x.grad
        if train:
            out[f"{key}_deps"] = layer.eps.grad
    g = golden_graph(Graph, d, dev)
    g.sym_norm()
    for order in ORDERS:
        model = Grand(8, 16, 3, 0.0, 0.0, False, DROPNODE, order, 0.5).to(dev)
        torch.manual_seed(SEED)
        with torch.no_grad():
            out[f"grand_train_{order}"] = model.rand_prop(g, torch.from_numpy(d["x"]).to(dev))
        kernels[f"grand_{order}"] = cogdl_b200._cabi.last_kernel()
        model.eval()
        with torch.no_grad():
            out[f"grand_eval_{order}"] = model.rand_prop(g, torch.from_numpy(d["x"]).to(dev))
    torch.manual_seed(7)
    model = Grand(8, 16, 3, 0.2, 0.2, True, DROPNODE, 4, 0.5).to(dev)
    gf = golden_graph(Graph, d, dev)
    torch.manual_seed(8)
    out["grand_forward"] = model(gf).detach()
    torch.manual_seed(9)
    gin = GIN(3, 8, 4, 16, 2, 0.0, "sum", True, 0.5).to(dev)
    bg = batch_graph(Graph, dev)
    torch.manual_seed(10)
    logits = gin(bg)
    logits.backward(torch.ones_like(logits))
    model_out = {"gin_logits": logits.detach()}
    model_out.update({f"gin_grad_{n}": p.grad for n, p in gin.named_parameters() if p.grad is not None})
    return out, model_out, kernels


def main():
    cogdl = import_reference()
    import cogdl_b200
    from cogdl.data import Graph
    from cogdl.layers.gin_layer import GINLayer
    from cogdl.layers.gine_layer import GINELayer
    from cogdl.models.nn.grand import Grand

    dev = torch.device("cuda:0")
    d = np.load(GOLDEN)
    res = {}
    originals = (GINLayer.forward, GINELayer.forward, Grand.rand_prop)
    cogdl_b200.install()
    res["untouched_without_flag"] = (GINLayer.forward, GINELayer.forward, Grand.rand_prop) == originals
    base, base_model, _ = run_all(Graph, d, dev)
    res["patched"] = cogdl_b200.install(gin=True, grand=True)
    res["rebound"] = all(getattr(f, "_cogdl_b200", False) for f in (GINLayer.forward, GINELayer.forward, Grand.rand_prop))
    fused, fused_model, kernels = run_all(Graph, d, dev)
    res["bit_identical"] = {k: bool(torch.equal(base[k].view(torch.int32), fused[k].view(torch.int32))) for k in base}
    # relative to the largest magnitude over the logits and every gradient: the biases ahead of a BatchNorm have
    # gradients at the noise level of the pooling's atomics, which a per-tensor scale would magnify
    scale = max(float(v.abs().max()) for v in base_model.values())
    res["model_rel"] = {k: float((fused_model[k].double() - base_model[k].double()).abs().max()) / scale
                        for k in base_model}
    res["vs_golden"] = {k: rel(fused[k].cpu().numpy(), d[k]) for k in fused if k in d.files}
    res["fused_kernels"] = {k: ("dcoef_kernel" in v if k.startswith("gin") else
                                ("accum_kernel" in v if not k.endswith("_0") else True)) for k, v in kernels.items()}
    calls = []
    for cls, attr in ((GINLayer, "forward"), (GINELayer, "forward"), (Grand, "rand_prop")):
        orig = getattr(cls, "_cogdl_b200_original_" + attr)

        def counting(*a, _orig=orig, _name=f"{cls.__name__}.{attr}", **k):
            calls.append(_name)
            return _orig(*a, **k)
        setattr(cls, "_cogdl_b200_original_" + attr, counting)
    gcpu = Graph(x=torch.from_numpy(d["x"]).clone(), edge_index=(torch.from_numpy(d["row"]).clone(),
                                                                 torch.from_numpy(d["col"]).clone()))
    fb = {}
    # a CPU call reaches the original, whose spmm (rebound by install()) then refuses CPU tensors
    layer = GINLayer(None, 0.1, True)
    try:
        layer(gcpu, torch.from_numpy(d["x"]).clone())
    except RuntimeError as e:
        assert "CPU tensors are not supported" in str(e), e
    fb["gin_cpu"] = calls[-1:] == ["GINLayer.forward"]
    layer64 = GINELayer(None, 0.1, True).to(dev).double()
    try:    # the original's spmm (rebound by install()) has no fp64 kernel either
        layer64(golden_graph(Graph, d, dev), torch.from_numpy(d["x"]).to(dev).double())
    except TypeError as e:
        assert "float32 / float16" in str(e), e
    fb["gine_fp64"] = calls[-1:] == ["GINELayer.forward"]
    model = Grand(8, 16, 3, 0.0, 0.0, False, DROPNODE, 2, 0.5)
    gcpu.sym_norm()
    try:
        model.rand_prop(gcpu, torch.from_numpy(d["x"]).clone())
    except RuntimeError as e:
        assert "CPU tensors are not supported" in str(e), e
    fb["grand_cpu"] = calls[-1:] == ["Grand.rand_prop"]
    g64 = golden_graph(Graph, d, dev)
    try:
        model.to(dev).rand_prop(g64, torch.from_numpy(d["x"]).to(dev).double())
    except TypeError as e:
        assert "float32 / float16" in str(e), e
    fb["grand_fp64"] = calls[-1:] == ["Grand.rand_prop"]
    fb["only_fallbacks_counted"] = len(calls) == 4
    res["fallbacks"] = fb
    for cls, attr in ((GINLayer, "forward"), (GINELayer, "forward"), (Grand, "rand_prop")):
        setattr(cls, "_cogdl_b200_original_" + attr, originals[[GINLayer, GINELayer, Grand].index(cls)])
    from cogdl_b200 import uninstall_gin, uninstall_grand

    uninstall_gin()
    uninstall_grand()
    res["restored"] = (GINLayer.forward, GINELayer.forward, Grand.rand_prop) == originals
    del cogdl
    print(json.dumps(res))


if __name__ == "__main__":
    main()

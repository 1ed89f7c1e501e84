"""GAT with attention dropout: the fused kernels (install(gat=True)) against the reference's unfused path (CUDA events,
medians, variants alternated inside one run).

  (a) ogbn-arxiv shape (169,343 nodes, 1,166,243 power-law edges + self loops, 128 features, 40 classes): the
      reference GAT model, 2 layers, 8 heads x 16, attn_drop 0.5, feature dropout 0.6; one training step = forward,
      cross-entropy, backward, SGD step.  Variants: the original GATLayer.forward under install() (unfused: gathers,
      LeakyReLU, edge_softmax, nn.Dropout, mh_spmm), the rebound forward of install(gat=True) with attn_drop 0.5, and
      the rebound forward with attn_drop 0 (the floor: the same kernels without the mask).
  (b) ogbn-products shape (2,449,029 nodes, 61,859,140 edges + self loops, 100 features): one GATLayer (8 heads x 16,
      attn_drop 0.5) forward + backward, fused against unfused, as far as the unfused path fits.
For every variant: median step time and the peak of torch.cuda.max_memory_allocated above what was allocated before the
step.  Needs the reference package (oracle/_ref/pkg).  Writes time_gat_dropout.json to OUT_DIR with the card name and
power limit read in the same run.

    python tools/time_gat_dropout.py OUT_DIR [--steps K]
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F
from gpu_timing import event_times, peak_above, write_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cogdl_b200  # noqa: E402
from cogdl_b200 import synth  # noqa: E402
from tests.refpkg import import_reference  # noqa: E402

ap = argparse.ArgumentParser()
ap.add_argument("out_dir")
ap.add_argument("--steps", type=int, default=20)
args = ap.parse_args()
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda")

import_reference()
import cogdl.layers.gat_layer as gl  # noqa: E402
from cogdl.data import Graph  # noqa: E402
from cogdl.models.nn.gat import GAT  # noqa: E402

cogdl_b200.install()


def set_variant(name, modules):
    if name == "unfused":
        cogdl_b200.uninstall_gat()
    else:
        cogdl_b200.install(gat=True)
    for m in modules:
        m.dropout.p = 0.0 if name == "fused_p0" else 0.5


def measure(step, modules, variants, steps):
    """Alternates the variants step by step; returns {variant: (median us, peak MB above the baseline)}."""
    times = {v: [] for v in variants}
    peaks = {v: 0 for v in variants}
    for v in variants:                                   # warm every variant (module loads, plans, transposes)
        set_variant(v, modules)
        for _ in range(2):
            step()
    torch.cuda.synchronize()
    for _ in range(steps):
        for v in variants:
            set_variant(v, modules)
            peaks[v] = max(peaks[v], peak_above(lambda: times[v].extend(event_times(step, 1, 0, flush=False))))
    return {v: {"us": statistics.median(times[v]), "peak_mb": peaks[v] / 2 ** 20} for v in variants}


def power_law_graph(n, e, f, seed):
    rp, col = synth.powerlaw_csr(n, e, seed=seed, device=dev)
    row = torch.repeat_interleave(torch.arange(n, device=dev), rp[1:] - rp[:-1])
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(n, f, device=dev, generator=g)
    return Graph(x=x, edge_index=(row, col)), rp.numel() - 1, col.numel()


result = {}

# ---- (a) arxiv: 2-layer GAT training step
graph, n, nnz = power_law_graph(169343, 1166243, 128, seed=0)
graph.y = torch.randint(0, 40, (n,), device=dev)
torch.manual_seed(0)
model = GAT(128, 16, 40, 2, 0.6, 0.5, 0.2, 8, False, 1).to(dev).train()
opt = torch.optim.SGD(model.parameters(), lr=0.01)


def train_step():
    opt.zero_grad()
    loss = F.cross_entropy(model(graph), graph.y)
    loss.backward()
    opt.step()


res_a = measure(train_step, list(model.attentions), ["unfused", "fused_drop", "fused_p0"], args.steps)
res_a["shape"] = {"nodes": n, "edges": nnz, "features": 128, "heads": 8, "hidden": 16, "classes": 40}
result["arxiv_gat2_train_step"] = res_a
print("arxiv 2-layer GAT train step:", json.dumps(res_a), flush=True)
del graph, model, opt
torch.cuda.empty_cache()

# ---- (b) products: one layer forward + backward
graph, n, nnz = power_law_graph(2449029, 61859140, 100, seed=1)
torch.manual_seed(0)
layer = gl.GATLayer(100, 16, nhead=8, attn_drop=0.5).to(dev).train()
x = graph.x.requires_grad_(False)
g_out = torch.randn(n, 128, device=dev)


def layer_step():
    layer.zero_grad()
    layer(graph, x).backward(g_out)


res_b = {"shape": {"nodes": n, "edges": nnz, "features": 100, "heads": 8, "hidden": 16}}
res_b.update(measure(layer_step, [layer], ["fused_drop", "fused_p0"], max(args.steps // 2, 5)))
try:
    alt = measure(layer_step, [layer], ["unfused", "fused_drop"], 5)
    res_b["unfused"], res_b["fused_drop_alongside_unfused"] = alt["unfused"], alt["fused_drop"]
except torch.cuda.OutOfMemoryError as e:       # the unfused path does not fit: say so
    res_b["unfused"] = {"error": f"out of memory: {str(e).splitlines()[0]}"}
result["products_gat_layer_fwd_bwd"] = res_b
print("products GATLayer fwd+bwd:", json.dumps(res_b), flush=True)
write_result(args.out_dir, "time_gat_dropout", result)

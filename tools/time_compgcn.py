"""CompGCN: the fused composition aggregation and layer against the reference's per-edge message passing (CUDA events,
L2 flushed, medians).

  (a) FB15k-237 shape: 14,541 entities, 237 relations with Zipf(1) frequencies, 272,115 triples with entity ranks drawn
      from a power law, each plus its reverse (type t + 237), shuffled COO.
      - the fused aggregation (both halves, mult) at F = 100 and 200 against spmm_raw on the same stacked CSR and F;
      - CompGCNLayer (F_in = 100, F_out = 200, sub, dropout 0) forward and forward + backward, the original forward
        against install(compgcn=True)'s, with time and peak torch.cuda.max_memory_allocated above the inputs;
      - LinkPredictCompGCN.predict() with 2 layers and hidden 200, original against installed;
      - the structure build (CompStructure from the COO, plan included), since loss() samples new edges every step.
  (b) ogbl-wikikg2 shape: 2.5 M entities, 535 relations, 16.1 M triples plus reverses: the fused layer forward +
      backward, time and peak memory.  The reference is not run there; its edge-sized tensors are given as computed
      sizes.
Needs the reference package (oracle/_ref/pkg).  Inputs are seeded; the SHA-256 of every fused output is printed.
Writes time_compgcn.json to OUT_DIR with the card name and power limit read in the same run.

    python tools/time_compgcn.py OUT_DIR
"""
import json
import os
import statistics
import sys

import numpy as np
import torch
from gpu_timing import digest, event_times, peak_above, write_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cogdl_b200  # noqa: E402
from cogdl_b200 import structure  # noqa: E402
from cogdl_b200.operators._raw import comp_aggr_raw, spmm_raw  # noqa: E402
from tests.refpkg import import_reference  # noqa: E402

if len(sys.argv) != 2:
    sys.exit(__doc__)
out_dir = sys.argv[1]
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda")
def make_kg(n_ent, n_rel, n_tri, seed):
    """Seeded KG: relation frequencies Zipf(1) over a random relation order, entity ranks from a power law (hubs),
    each triple plus its reverse (type t + n_rel), the COO shuffled.  int64 tensors on the device."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rel_p = 1.0 / torch.arange(1, n_rel + 1, device=dev, dtype=torch.float64)
    r = torch.multinomial(rel_p, n_tri, replacement=True, generator=g)
    r = torch.randperm(n_rel, device=dev, generator=g)[r]
    ent_p = torch.arange(1, n_ent + 1, device=dev, dtype=torch.float64) ** -0.8
    pick = lambda: torch.randperm(n_ent, device=dev, generator=g)[torch.multinomial(ent_p, n_tri, True, generator=g)]  # noqa: E731
    h, t = pick(), pick()
    row, col, typ = torch.cat([h, t]), torch.cat([t, h]), torch.cat([r, r + n_rel])
    perm = torch.randperm(row.numel(), device=dev, generator=g)
    return row[perm].contiguous(), col[perm].contiguous(), typ[perm].contiguous()


import_reference()
from cogdl.data import Graph  # noqa: E402
from cogdl.models.nn.compgcn import CompGCNLayer, LinkPredictCompGCN  # noqa: E402

cogdl_b200.install(compgcn=True)
ORIGINAL = CompGCNLayer._cogdl_b200_original_forward
FUSED = CompGCNLayer.forward


def with_forward(fwd, fn):
    CompGCNLayer.forward = fwd
    try:
        return fn()
    finally:
        CompGCNLayer.forward = FUSED


res = {"fb15k237": {}, "wikikg2": {}, "sha256": {}}

# ---------------------------------------------------------------------------------------------- (a)
N, R = 14541, 237
row, col, typ = make_kg(N, R, 272115, seed=0)
E = row.numel()
fb = res["fb15k237"]
torch.cuda.synchronize()
structure.clear_structure_cache()
cs = structure.CompStructure(row, col, typ, N)
cs.csr.plan
torch.cuda.synchronize()


def build():
    c = structure.CompStructure(row, col, typ, N)
    c.csr.plan
    torch.cuda.synchronize()


fb["structure_build_us"] = statistics.median(event_times(build, 10, 3, flush=True))
fb["hub_rows_2N"] = cs.csr.plan.n_hub_rows
for F in (100, 200):
    gen = torch.Generator(device=dev).manual_seed(F)
    x = torch.randn(N, F, device=dev, generator=gen)
    relt = torch.randn(2 * R + 1, F, device=dev, generator=gen)
    t_sp = statistics.median(event_times(lambda: spmm_raw(cs.csr, cs.w, x), 20, 3, flush=True))
    t_mult = statistics.median(
        event_times(lambda: comp_aggr_raw(cs.csr, cs.type, cs.w, x, relt, "mult"), 20, 3, flush=True))
    t_sub = statistics.median(
        event_times(lambda: comp_aggr_raw(cs.csr, cs.type, cs.w, x, relt, "sub"), 20, 3, flush=True))
    fb[f"aggr_F{F}"] = {"spmm_us": t_sp, "fused_mult_us": t_mult, "fused_sub_us": t_sub,
                        "ratio_mult": t_mult / t_sp, "ratio_sub": t_sub / t_sp}
    res["sha256"][f"fb_aggr_mult_F{F}"] = digest(comp_aggr_raw(cs.csr, cs.type, cs.w, x, relt, "mult"))

# CompGCNLayer, F_in 100 -> F_out 200
F_IN, F_OUT = 100, 200
graph = Graph(edge_index=(row, col), edge_attr=typ)
torch.manual_seed(0)
layer = CompGCNLayer(F_IN, F_OUT, R, opn="sub", activation=torch.tanh).to(dev).train()
x = torch.randn(N, F_IN, device=dev, requires_grad=True)
rel_in = torch.randn(2 * R, F_IN, device=dev, requires_grad=True)
G = torch.randn(N, F_OUT, device=dev)


def layer_fwd():
    return layer(graph, x, rel_in)


def layer_fwd_bwd():
    out, r = layer(graph, x, rel_in)
    ((out * G).sum() + r.sum()).backward()


for name, fwd in (("original", ORIGINAL), ("fused", FUSED)):
    with torch.no_grad():
        t_f = with_forward(fwd, lambda: statistics.median(event_times(layer_fwd, 10, 3, flush=True)))
    t_fb = with_forward(fwd, lambda: statistics.median(event_times(layer_fwd_bwd, 10, 3, flush=True)))
    m_fb = with_forward(fwd, lambda: peak_above(layer_fwd_bwd))
    fb[f"layer_{name}"] = {"fwd_us": t_f, "fwd_bwd_us": t_fb, "fwd_bwd_peak_bytes": m_fb}
with torch.no_grad():
    y_o = with_forward(ORIGINAL, layer_fwd)[0]
    y_f = layer_fwd()[0]
fb["layer_fused_vs_original_max_rel"] = float((y_f - y_o).abs().max() / y_o.abs().max())
res["sha256"]["fb_layer_fused"] = digest(y_f)
fb["layer_fwd_bwd_speedup"] = fb["layer_original"]["fwd_bwd_us"] / fb["layer_fused"]["fwd_bwd_us"]
fb["layer_fwd_speedup"] = fb["layer_original"]["fwd_us"] / fb["layer_fused"]["fwd_us"]

# LinkPredictCompGCN.predict(), 2 layers, hidden 200
torch.manual_seed(1)
model = LinkPredictCompGCN(N, R, 200, layers=2, dropout=0.3, opn="sub").to(dev).eval()
with torch.no_grad():
    for name, fwd in (("original", ORIGINAL), ("fused", FUSED)):
        t = with_forward(fwd, lambda: statistics.median(event_times(lambda: model.predict(graph), 10, 3, flush=True)))
        m = with_forward(fwd, lambda: peak_above(lambda: model.predict(graph)))
        fb[f"predict_{name}"] = {"us": t, "peak_bytes": m}
fb["predict_speedup"] = fb["predict_original"]["us"] / fb["predict_fused"]["us"]
print(json.dumps(fb, indent=1), flush=True)
del graph, layer, model, x, rel_in, cs
torch.cuda.empty_cache()

# ---------------------------------------------------------------------------------------------- (b)
N, R = 2_500_000, 535
row, col, typ = make_kg(N, R, 16_100_000, seed=1)
E = row.numel()
wk = res["wikikg2"]
wk["E"] = E
wk["reference_edge_tensor_bytes"] = {"[E/2, F_out] fp32": (E // 2) * F_OUT * 4, "[E/2, F_out] int64 index": (E // 2) * F_OUT * 8,
                                     "[E/2, F_in] fp32": (E // 2) * F_IN * 4}
graph = Graph(edge_index=(row, col), edge_attr=typ)
torch.manual_seed(0)
layer = CompGCNLayer(F_IN, F_OUT, R, opn="sub", activation=torch.tanh).to(dev).train()
x = torch.randn(N, F_IN, device=dev, requires_grad=True)
rel_in = torch.randn(2 * R, F_IN, device=dev, requires_grad=True)
G = torch.randn(N, F_OUT, device=dev)
torch.cuda.synchronize()
structure.clear_structure_cache()
wk["first_fwd_bwd_peak_bytes"] = peak_above(layer_fwd_bwd)       # includes the structure build
wk["fwd_bwd_us"] = statistics.median(event_times(layer_fwd_bwd, 5, 1, flush=True))
with torch.no_grad():
    wk["fwd_us"] = statistics.median(event_times(layer_fwd, 5, 1, flush=True))
wk["fwd_bwd_peak_bytes"] = peak_above(layer_fwd_bwd)
res["sha256"]["wikikg2_layer"] = digest(layer_fwd()[0])
print(json.dumps(wk, indent=1), flush=True)
write_result(out_dir, "time_compgcn", res)
print(json.dumps({"card": res["card"], "sha256": res["sha256"]}))

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
import hashlib
import json
import os
import statistics
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cogdl_b200  # noqa: E402
from cogdl_b200 import structure  # noqa: E402
from cogdl_b200.operators._raw import comp_aggr_raw, spmm_raw  # noqa: E402
from tests.refpkg import import_reference  # noqa: E402

if len(sys.argv) != 2:
    sys.exit(__doc__)
out_dir = sys.argv[1]
os.makedirs(out_dir, exist_ok=True)
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda")
card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                      capture_output=True, text=True).stdout.strip()
flush = torch.empty(512 << 20, dtype=torch.uint8, device=dev)


def timed(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        flush.zero_()
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        fn()
        b.record()
        torch.cuda.synchronize()
        ts.append(a.elapsed_time(b) * 1e3)
    return statistics.median(ts)


def peak_above(fn):
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def sha(t):
    return hashlib.sha256(t.detach().contiguous().cpu().numpy().tobytes()).hexdigest()[:16]


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


res = {"card": card, "fb15k237": {}, "wikikg2": {}, "sha256": {}}

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


fb["structure_build_us"] = timed(build, reps=10)
fb["hub_rows_2N"] = cs.csr.plan.n_hub_rows
for F in (100, 200):
    gen = torch.Generator(device=dev).manual_seed(F)
    x = torch.randn(N, F, device=dev, generator=gen)
    relt = torch.randn(2 * R + 1, F, device=dev, generator=gen)
    t_sp = timed(lambda: spmm_raw(cs.csr, cs.w, x))
    t_mult = timed(lambda: comp_aggr_raw(cs.csr, cs.type, cs.w, x, relt, "mult"))
    t_sub = timed(lambda: comp_aggr_raw(cs.csr, cs.type, cs.w, x, relt, "sub"))
    fb[f"aggr_F{F}"] = {"spmm_us": t_sp, "fused_mult_us": t_mult, "fused_sub_us": t_sub,
                        "ratio_mult": t_mult / t_sp, "ratio_sub": t_sub / t_sp}
    res["sha256"][f"fb_aggr_mult_F{F}"] = sha(comp_aggr_raw(cs.csr, cs.type, cs.w, x, relt, "mult"))

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
        t_f = with_forward(fwd, lambda: timed(layer_fwd, reps=10))
    t_fb = with_forward(fwd, lambda: timed(layer_fwd_bwd, reps=10))
    m_fb = with_forward(fwd, lambda: peak_above(layer_fwd_bwd))
    fb[f"layer_{name}"] = {"fwd_us": t_f, "fwd_bwd_us": t_fb, "fwd_bwd_peak_bytes": m_fb}
with torch.no_grad():
    y_o = with_forward(ORIGINAL, layer_fwd)[0]
    y_f = layer_fwd()[0]
fb["layer_fused_vs_original_max_rel"] = float((y_f - y_o).abs().max() / y_o.abs().max())
res["sha256"]["fb_layer_fused"] = sha(y_f)
fb["layer_fwd_bwd_speedup"] = fb["layer_original"]["fwd_bwd_us"] / fb["layer_fused"]["fwd_bwd_us"]
fb["layer_fwd_speedup"] = fb["layer_original"]["fwd_us"] / fb["layer_fused"]["fwd_us"]

# LinkPredictCompGCN.predict(), 2 layers, hidden 200
torch.manual_seed(1)
model = LinkPredictCompGCN(N, R, 200, layers=2, dropout=0.3, opn="sub").to(dev).eval()
with torch.no_grad():
    for name, fwd in (("original", ORIGINAL), ("fused", FUSED)):
        t = with_forward(fwd, lambda: timed(lambda: model.predict(graph), reps=10))
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
wk["fwd_bwd_us"] = timed(layer_fwd_bwd, reps=5, warm=1)
with torch.no_grad():
    wk["fwd_us"] = timed(layer_fwd, reps=5, warm=1)
wk["fwd_bwd_peak_bytes"] = peak_above(layer_fwd_bwd)
res["sha256"]["wikikg2_layer"] = sha(layer_fwd()[0])
print(json.dumps(wk, indent=1), flush=True)
print(json.dumps({"card": card, "sha256": res["sha256"]}))
with open(os.path.join(out_dir, "time_compgcn.json"), "w") as f:
    json.dump(res, f, indent=1)

"""R-GCN: the fan-out aggregation and the installed RGCNLayer against the reference's forward (CUDA events, L2 flushed,
medians).

  (a) FB15k-237 shape: 14,541 entities, 237 relations with Zipf(1) frequencies, 272,115 triples with entity ranks drawn
      from a power law, shuffled COO, row-normalised weights.
      - the aggregation at F = 200, B = 5 against spmm_raw on the same structure and F, and against five separate
        weighted SpMMs (the per-basis values formed once, outside the timing);
      - RGCNLayer (200 -> 200, num_bases 5, dropout 0) forward and forward + backward for three versions: the original
        forward, a corrected unfused loop (the reference's loop with `return h_list` after it and the masked graph in
        the SpMM, on this package's spmm) and install(rgcn=True)'s, with peak torch.cuda.max_memory_allocated above the
        inputs;
      - LinkPredictRGCN.predict() with 2 layers, hidden 200, num_bases 5, original against installed;
      - one LinkPredictRGCN.loss() step with its backward (sampling rate 0.01, as the model's default), which builds a
        new graph every step: host-side sampling and the structure build are included.
  (b) ogbl-wikikg2 shape: 2.5 M entities, 535 relations, 16.1 M triples: the installed layer forward + backward, time
      and peak memory.  The original is not run there: its [T, N, F_out] tensor alone is given as a computed size.
Needs the reference package (oracle/_ref/pkg).  Inputs are seeded; the SHA-256 of the installed outputs is printed.
Writes time_rgcn.json to OUT_DIR with the card name and power limit read in the same run.

    python tools/time_rgcn.py OUT_DIR
"""
import json
import os
import statistics
import sys

import numpy as np
import torch
from gpu_timing import digest, event_times, host_times, peak_above, write_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cogdl_b200  # noqa: E402
from cogdl_b200 import structure  # noqa: E402
from cogdl_b200.operators._raw import rgcn_aggr_raw, spmm_raw  # noqa: E402
from tests.refpkg import import_reference  # noqa: E402

if len(sys.argv) != 2:
    sys.exit(__doc__)
out_dir = sys.argv[1]
torch.backends.cuda.matmul.allow_tf32 = False
dev = torch.device("cuda")
def make_kg(n_ent, n_rel, n_tri, seed):
    """Seeded KG: relation frequencies Zipf(1) over a random relation order, entity ranks from a power law (hubs), the
    COO shuffled.  int64 tensors on the device."""
    g = torch.Generator(device=dev).manual_seed(seed)
    rel_p = 1.0 / torch.arange(1, n_rel + 1, device=dev, dtype=torch.float64)
    r = torch.multinomial(rel_p, n_tri, replacement=True, generator=g)
    r = torch.randperm(n_rel, device=dev, generator=g)[r]
    ent_p = torch.arange(1, n_ent + 1, device=dev, dtype=torch.float64) ** -0.8
    pick = lambda: torch.randperm(n_ent, device=dev, generator=g)[torch.multinomial(ent_p, n_tri, True, generator=g)]  # noqa: E731
    h, t = pick(), pick()
    perm = torch.randperm(n_tri, device=dev, generator=g)
    return h[perm].contiguous(), t[perm].contiguous(), r[perm].contiguous()


import_reference()
from cogdl.data import Graph  # noqa: E402
from cogdl.layers.rgcn_layer import RGCNLayer  # noqa: E402
from cogdl.models.nn.rgcn import LinkPredictRGCN  # noqa: E402
from cogdl.utils import spmm as ref_spmm  # noqa: E402
from cogdl.utils.link_prediction_utils import DistMultLayer  # noqa: E402

cogdl_b200.install(rgcn=True)
ORIGINAL = RGCNLayer._cogdl_b200_original_forward
INSTALLED = RGCNLayer.forward


def corrected_forward(self, graph, x):
    """The reference forward with its loop corrected: every relation's masked graph in its SpMM, the list returned after
    the loop.  The masked graphs carry the row-normalised weights of their edges, without padding_self_loops()."""
    import torch.nn.functional as F

    edge_type = graph.edge_attr
    weight = torch.matmul(self.alpha, self.weight.view(self.num_bases, -1)).view(self.num_edge_types, self.in_feats,
                                                                               self.out_feats)
    graph.row_norm()
    edge_index = torch.stack(graph.edge_index)
    edge_type = graph.edge_attr
    edge_weight = graph.edge_weight
    h = torch.matmul(x, weight)
    h_result = 0
    for t in range(self.num_edge_types):
        m = edge_type == t
        g = Graph(edge_index=edge_index[:, m], edge_weight=edge_weight[m], num_nodes=x.shape[0])
        h_result = h_result + ref_spmm(g, h[t])
    h_result = F.dropout(h_result, p=self.dropout, training=self.training)
    if self.layer_norm is not None:
        h_result = self.layer_norm(h_result)
    if self.bias is not None:
        h_result = h_result + self.bias
    h_result += F.dropout(torch.matmul(x, self.weight_self_loop), p=self.self_dropout, training=self.training)
    return h_result


def with_forward(fwd, fn):
    RGCNLayer.forward = fwd
    try:
        return fn()
    finally:
        RGCNLayer.forward = INSTALLED


def on_gpu_graph(row, col, typ):
    g = Graph(edge_index=(row, col), edge_attr=typ)
    g.edge_attr = typ
    return g


res = {"fb15k237": {}, "wikikg2": {}, "sha256": {}}

# ---------------------------------------------------------------------------------------------- (a)
N, R, F, BASES = 14541, 237, 200, 5
row, col, typ = make_kg(N, R, 272115, seed=0)
fb = res["fb15k237"]
graph = on_gpu_graph(row, col, typ)
graph.row_norm()
st, val, _, _, _ = structure.graph_operands(graph)
rs = structure.rgcn_structure_for(st, graph.edge_attr)
fb["hub_rows"] = st.plan.n_hub_rows
gen = torch.Generator(device=dev).manual_seed(1)
x = torch.randn(N, F, device=dev, generator=gen)
coef = torch.randn(R, BASES, device=dev, generator=gen)
vals = [(val * coef[rs.type.long(), b]).contiguous() for b in range(BASES)]
t_sp = statistics.median(event_times(lambda: spmm_raw(st, val, x), 20, 3, flush=True))
t_agg = statistics.median(event_times(lambda: rgcn_aggr_raw(st, rs.type, val, coef, x), 20, 3, flush=True))


def five():
    for v in vals:
        spmm_raw(st, v, x)


t_five = statistics.median(event_times(five, 20, 3, flush=True))
fb["aggr_F200_B5"] = {"spmm_us": t_sp, "fanout_us": t_agg, "five_spmm_us": t_five, "vs_spmm": t_agg / t_sp,
                      "vs_five_spmm": t_agg / t_five}
res["sha256"]["fb_aggr"] = digest(rgcn_aggr_raw(st, rs.type, val, coef, x))
print(json.dumps(fb, indent=1), flush=True)

torch.manual_seed(0)
layer = RGCNLayer(F, F, R, "basis", BASES).to(dev).train()
xl = torch.randn(N, F, device=dev, requires_grad=True)
G = torch.randn(N, F, device=dev)


def layer_fwd():
    return layer(graph, xl)


def layer_fwd_bwd():
    (layer(graph, xl) * G).sum().backward()


for name, fwd in (("original", ORIGINAL), ("corrected_loop", corrected_forward), ("installed", INSTALLED)):
    with torch.no_grad():
        t_f = with_forward(fwd, lambda: statistics.median(event_times(layer_fwd, 10, 3, flush=True)))
    t_fb = with_forward(fwd, lambda: statistics.median(event_times(layer_fwd_bwd, 10, 3, flush=True)))
    m_fb = with_forward(fwd, lambda: peak_above(layer_fwd_bwd))
    fb[f"layer_{name}"] = {"fwd_us": t_f, "fwd_bwd_us": t_fb, "fwd_bwd_peak_bytes": m_fb}
    print(name, fb[f"layer_{name}"], flush=True)
with torch.no_grad():
    y_c = with_forward(corrected_forward, layer_fwd)
    y_i = layer_fwd()
fb["installed_vs_corrected_loop_max_rel"] = float((y_i - y_c).abs().max() / y_c.abs().max())
res["sha256"]["fb_layer_installed"] = digest(y_i)
for k in ("fwd_us", "fwd_bwd_us", "fwd_bwd_peak_bytes"):
    fb[f"layer_{k}_original_over_installed"] = fb["layer_original"][k] / fb["layer_installed"][k]
    fb[f"layer_{k}_corrected_over_installed"] = fb["layer_corrected_loop"][k] / fb["layer_installed"][k]

torch.manual_seed(1)
model = LinkPredictRGCN(N, R, 200, 2, "basis", BASES).to(dev).eval()
pgraph = on_gpu_graph(row, col, typ)
with torch.no_grad():
    for name, fwd in (("original", ORIGINAL), ("installed", INSTALLED)):
        t = with_forward(fwd, lambda: statistics.median(event_times(lambda: model.predict(pgraph), 10, 3, flush=True)))
        m = with_forward(fwd, lambda: peak_above(lambda: model.predict(pgraph)))
        fb[f"predict_{name}"] = {"us": t, "peak_bytes": m}
fb["predict_speedup"] = fb["predict_original"]["us"] / fb["predict_installed"]["us"]

model.train()
scoring = DistMultLayer()


def loss_step():
    model.zero_grad(set_to_none=True)
    model.loss(on_gpu_graph(row, col, typ), scoring).backward()


for name, fwd in (("original", ORIGINAL), ("installed", INSTALLED)):
    np.random.seed(3)
    try:
        fb[f"loss_step_{name}_us"] = statistics.median(host_times(lambda: with_forward(fwd, loss_step), 5, 1))
    except RuntimeError as e:    # the original raises on the GPU: loss() samples the edge types on the host
        fb[f"loss_step_{name}_us"] = f"raises: {str(e).splitlines()[0][:120]}"

print(json.dumps(fb, indent=1), flush=True)
del graph, pgraph, layer, model, xl, x, vals, rs, st, val
structure.clear_structure_cache()
torch.cuda.empty_cache()

# ---------------------------------------------------------------------------------------------- (b)
N, R = 2_500_000, 535
row, col, typ = make_kg(N, R, 16_100_000, seed=1)
wk = res["wikikg2"]
wk["E"] = row.numel()
wk["original_h_tensor_bytes"] = R * N * F * 4
graph = on_gpu_graph(row, col, typ)
torch.manual_seed(0)
layer = RGCNLayer(F, F, R, "basis", BASES).to(dev).train()
xl = torch.randn(N, F, device=dev, requires_grad=True)
G = torch.randn(N, F, device=dev)
wk["first_fwd_bwd_with_build_us"] = host_times(layer_fwd_bwd, 1, 0)[0]
wk["fwd_bwd_us"] = statistics.median(event_times(layer_fwd_bwd, 5, 1, flush=True))
wk["fwd_bwd_peak_bytes"] = peak_above(layer_fwd_bwd)
wk["inputs_bytes"] = torch.cuda.memory_allocated()
print(json.dumps(wk, indent=1), flush=True)

write_result(out_dir, "time_rgcn", res)
print(json.dumps(res["sha256"]))

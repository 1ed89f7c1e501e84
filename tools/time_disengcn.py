"""DisenGCN routing: fused kernels vs the reference's op sequence (CUDA events, L2 flushed, medians of alternating rounds).

  (a) arxiv shape without self loops, F = 64, K in {16, 8} (d = 4, 8), tau = 1, a 128 -> 64 layer:
      spmm_raw at F = 64 (the yardstick), one fused routing step forward, the fused layer (act(x W + b), then
      T = 7 steps) forward and forward + backward, and the reference layer's op sequence on the GPU
      (cogdl/layers/disengcn_layer.py:44-91 with our edge_softmax) forward and forward + backward; peak
      torch.cuda.max_memory_allocated above the inputs for both forward + backward;
  (b) a training step of the reference DisenGCN (K = [16, 8], hidden 64, T = 7, 128 features, 40 classes) on the
      arxiv shape, DisenGCNLayer's original forward against install(disengcn=True)'s (needs oracle/_ref/pkg);
  (c) the products shape, one fused layer forward (F = 64, K = 16, T = 7): time and peak memory.
Inputs are seeded; the SHA-256 of every output is printed.  Writes time_disengcn.json to OUT_DIR with the card name
and power limit read in the same run.

    python tools/time_disengcn.py OUT_DIR
"""
import json
import os
import statistics
import sys

import torch
from gpu_timing import digest, event_times, peak_above, write_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cogdl_b200  # noqa: E402
from cogdl_b200 import synth  # noqa: E402
from cogdl_b200.operators._raw import disen_route_fwd_raw, spmm_raw  # noqa: E402
from cogdl_b200.operators.edge_softmax import EdgeSoftmaxFunction  # noqa: E402

if len(sys.argv) != 2:
    sys.exit(__doc__)
out_dir = sys.argv[1]
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
PEAK = 3.35e12
T, TAU, F, IN = 7, 1.0, 64, 128

dev = torch.device("cuda")
def step_bytes(E, N, F, K):
    # per edge: column index + gathered c row; per row: rowptr, q and c rows, out row (+ lse2, r in training)
    return E * (4 + 4 * F) + N * (4 + 12 * F)


# ---------------------------------------------------------------------------------------------- (a)
n, e = synth.SHAPES["arxiv"]
rp, col = synth.powerlaw_csr(n, e, seed=0, device=dev, self_loops=False)
st = cogdl_b200.CSRStructure.from_int64(rp, col)
st.plan, st.csc()[0].plan
E = st.nnz
row = torch.repeat_interleave(torch.arange(n, device=dev), rp[1:] - rp[:-1])
colL = col.long()
gen = torch.Generator(device=dev).manual_seed(0)
x = torch.randn(n, IN, device=dev, generator=gen)
W = torch.nn.Parameter(0.1 * torch.randn(IN, F, device=dev, generator=gen))
b = torch.nn.Parameter(0.1 * torch.randn(F, device=dev, generator=gen))
r = torch.randn(n, F, device=dev, generator=gen)
xf = torch.randn(n, F, device=dev, generator=gen)


def act(xx):
    return torch.nn.functional.leaky_relu(xx @ W + b)


def fused_layer(K):
    return lambda xx: cogdl_b200.disen_routing(st, act(xx), K, T, TAU)


def reference_layer(K):
    d = F // K

    def run(xx):   # disengcn_layer.py:44-91, edge_softmax = ours
        h = act(xx)
        h = torch.cat([t.unsqueeze(0) for t in h.split(d, dim=-1)], dim=0)
        h_normed = h / h.pow(2).sum(dim=-1).sqrt().unsqueeze(-1)
        h_src = h_dst = h_normed.permute(1, 0, 2)
        for _ in range(T):
            s = (h_dst[row] * h_src[colL]).sum(dim=-1) / TAU
            w = EdgeSoftmaxFunction.apply(st, s.contiguous()).T.unsqueeze(-1)
            msg = h_src.index_select(0, colL).permute(1, 0, 2) * w
            idx = row.unsqueeze(-1).unsqueeze(0).repeat(K, 1, d)
            node = torch.zeros(h.shape, device=dev).scatter_add_(1, idx, msg) + h_normed
            h_dst = (node / node.pow(2).sum(-1).sqrt().unsqueeze(-1)).permute(1, 0, 2)
        return h_dst.reshape(n, -1)
    return run


def fwd_only(fn):
    def call():
        with torch.no_grad():
            fn(x)
    return call


def fwd_bwd(fn):
    def call():
        W.grad = b.grad = None
        fn(x).backward(r)
    return call


res = {"arxiv": {"n": n, "nnz": E, "F": F, "T": T}, "sha256": {}, "peak_bytes": {}, "parity": {},
       "bytes": {}, "rounds": []}
variants = {"spmm_raw_us": lambda: spmm_raw(st, None, xf)}
res["sha256"]["spmm_raw"] = digest(spmm_raw(st, None, xf))
for K in (16, 8):
    c = act(x).detach().reshape(n, K, F // K)
    c = (c / c.pow(2).sum(-1, keepdim=True).sqrt()).reshape(n, F).contiguous()
    variants[f"K{K}_fused_step_fwd_us"] = (lambda c_=c, K_=K: disen_route_fwd_raw(st, c_, c_, K_, TAU))
    variants[f"K{K}_fused_layer_fwd_us"] = fwd_only(fused_layer(K))
    variants[f"K{K}_reference_layer_fwd_us"] = fwd_only(reference_layer(K))
    variants[f"K{K}_fused_layer_fwd_bwd_us"] = fwd_bwd(fused_layer(K))
    variants[f"K{K}_reference_layer_fwd_bwd_us"] = fwd_bwd(reference_layer(K))
    res["bytes"][f"K{K}_step"] = step_bytes(E, n, F, K)
    with torch.no_grad():
        got, want = fused_layer(K)(x), reference_layer(K)(x)
    res["parity"][f"K{K}_fused_vs_reference_max_row_rel_err"] = float(
        ((got - want).abs() / want.abs().amax(1, keepdim=True).clamp_min(1e-30)).max())
    res["sha256"][f"K{K}_fused_step"] = digest(disen_route_fwd_raw(st, c, c, K, TAU)[0])
    res["sha256"][f"K{K}_fused_layer"] = digest(got)
    res["sha256"][f"K{K}_reference_layer"] = digest(want)
    for name, fn in (("fused", fused_layer(K)), ("reference", reference_layer(K))):
        res["peak_bytes"][f"K{K}_{name}_layer_fwd_bwd"] = peak_above(fwd_bwd(fn))
        W.grad = b.grad = None
    del got, want

# ---------------------------------------------------------------------------------------------- (b)
steps = {}
try:
    from tests.refpkg import import_reference

    import_reference()
    from cogdl.data import Graph
    from cogdl.layers import DisenGCNLayer
    from cogdl.models.nn.disengcn import DisenGCN

    cogdl_b200.install(disengcn=True)
    from cogdl_b200.install import disengcn_forward

    original = DisenGCNLayer._cogdl_b200_original_forward
    torch.manual_seed(0)
    model = DisenGCN(IN, 64, 40, K=[16, 8], iterations=T, tau=TAU, dropout=0.5, activation="leaky_relu").to(dev)
    model.train()
    graph = Graph(x=x, edge_index=(row, colL))
    graph.row_indptr
    y = torch.randint(0, 40, (n,), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    opt = torch.optim.SGD(model.parameters(), lr=0.01)

    def step_with(forward):
        def step():
            DisenGCNLayer.forward = forward
            opt.zero_grad(set_to_none=True)
            torch.nn.functional.cross_entropy(model(graph), y).backward()
            opt.step()
        return step

    steps = {"disengcn_step_original_ms": step_with(original), "disengcn_step_patched_ms": step_with(disengcn_forward)}
    for k, fn in steps.items():
        res["peak_bytes"][k.replace("_ms", "")] = peak_above(fn)
except ImportError as ex:
    print(f"(b) skipped: {ex}")

for rnd in range(2):
    rr = {k: statistics.median(event_times(fn, 20, 3, flush=True)) for k, fn in variants.items()}
    rr.update({k: statistics.median(event_times(fn, 10, 3, flush=True)) / 1e3 for k, fn in steps.items()})
    res["rounds"].append(rr)
    for k, v in rr.items():
        print(f"round {rnd} {k:40s} {v:10.1f}" if k.endswith("_us") else f"round {rnd} {k:40s} {v:10.3f}")
med = {k: statistics.median(rd[k] for rd in res["rounds"]) for k in res["rounds"][0]}
res["summary"] = {}
for K in (16, 8):
    res["summary"][f"K{K}_step_over_spmm"] = med[f"K{K}_fused_step_fwd_us"] / med["spmm_raw_us"]
    res["summary"][f"K{K}_step_hbm_fraction"] = res["bytes"][f"K{K}_step"] / (med[f"K{K}_fused_step_fwd_us"] * 1e-6) / PEAK
    res["summary"][f"K{K}_reference_over_fused_fwd"] = med[f"K{K}_reference_layer_fwd_us"] / med[f"K{K}_fused_layer_fwd_us"]
    res["summary"][f"K{K}_reference_over_fused_fwd_bwd"] = (med[f"K{K}_reference_layer_fwd_bwd_us"]
                                                           / med[f"K{K}_fused_layer_fwd_bwd_us"])
if steps:
    res["summary"]["disengcn_step_speedup"] = med["disengcn_step_original_ms"] / med["disengcn_step_patched_ms"]
    del model, graph, opt, steps
res["kernel"] = cogdl_b200._cabi.last_kernel()

# ---------------------------------------------------------------------------------------------- (c)
del variants
torch.cuda.empty_cache()
np_, ep = synth.SHAPES["products"]
rp2, col2 = synth.powerlaw_csr(np_, ep, seed=0, device=dev, self_loops=False)
st2 = cogdl_b200.CSRStructure.from_int64(rp2, col2)
del rp2, col2
st2.plan
h2 = torch.randn(np_, F, device=dev, generator=torch.Generator(device=dev).manual_seed(2))
with torch.no_grad():
    out2 = cogdl_b200.disen_routing(st2, h2, 16, T, TAU)
    res["products"] = {"n": np_, "nnz": st2.nnz, "F": F, "K": 16, "T": T, "sha256": digest(out2)}
    del out2
    res["products"]["peak_bytes_above_inputs"] = peak_above(lambda: cogdl_b200.disen_routing(st2, h2, 16, T, TAU))
    res["products"]["fused_layer_fwd_ms"] = statistics.median(
        event_times(lambda: cogdl_b200.disen_routing(st2, h2, 16, T, TAU), 5, 3, flush=True)) / 1e3
res["products"]["reference_one_EKd_tensor_bytes"] = st2.nnz * F * 4
print(json.dumps({k: res[k] for k in ("summary", "peak_bytes", "products", "parity", "sha256", "kernel")}, indent=1))
write_result(out_dir, "time_disengcn", res)

"""GENConv softmax aggregation: fused kernels vs the reference's op sequence (CUDA events, L2 flushed, median of 20).

  (a) arxiv shape, F = 128, beta = 1 (a CUDA parameter): the fused forward and forward + backward against the
      reference's op sequence on the GPU (cogdl/layers/deepergcn_layer.py:67-93: gather, relu + eps, our
      edge_softmax with F heads, multiply, scatter_add_), with spmm_raw on the same graph and F as the yardstick;
  (b) a training step of the reference DeeperGCN (softmax_sg, hidden 128, 4 layers, learnable beta) on the arxiv
      shape, GENConv's original forward against install(genconv=True)'s (needs oracle/_ref/pkg);
  (c) the fused forward on the products shape at F = 256: time and max_memory_allocated.  The unfused sequence
      is not run there; only the size of one of its [E, F] tensors is printed.
Algorithmic bytes per call (fp32 values, int32 indices) and their share of the H100 SXM data sheet's 3.35 TB/s are
printed beside the times.  Two rounds, variants alternating inside each.  Writes time_genconv.json to OUT_DIR with
the card name and power limit read in the same run.

    python tools/time_genconv.py OUT_DIR
"""
import json
import os
import statistics
import sys

import torch
from gpu_timing import event_times, peak_above, write_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cogdl_b200  # noqa: E402
from cogdl_b200 import synth  # noqa: E402
from cogdl_b200.operators._raw import spmm_raw  # noqa: E402
from cogdl_b200.operators.edge_softmax import EdgeSoftmaxFunction  # noqa: E402

if len(sys.argv) != 2:
    sys.exit(__doc__)
out_dir = sys.argv[1]
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
PEAK = 3.35e12

dev = torch.device("cuda")
def fwd_bytes(E, N, F, edge=False, lse=False):
    return E * (4 * F + 4) + N * (4 * F + 4) + (E * 4 * F if edge else 0) + (N * 4 * F if lse else 0)


def bwd_bytes(E, N, F, edge=False):
    # per edge: row index + 3 gathered rows (lse, g, out); per column: colptr, x row, dx row; edge term read + grad write
    return E * (4 + 3 * 4 * F) + N * (4 + 8 * F) + (E * (4 + 8 * F) if edge else 0)


# ---------------------------------------------------------------------------------------------- (a)
n, e = synth.SHAPES["arxiv"]
rp, col = synth.powerlaw_csr(n, e, seed=0, device=dev, self_loops=True)
st = cogdl_b200.CSRStructure.from_int64(rp, col)
st.plan, st.csc()[0].plan
E, F = st.nnz, 128
row = torch.repeat_interleave(torch.arange(n, device=dev), rp[1:] - rp[:-1])
x = torch.randn(n, F, device=dev)
r = torch.randn(n, F, device=dev)
beta = torch.nn.Parameter(torch.ones(1, device=dev))
eps = 1e-7


def reference_sequence(xx):
    msg = torch.relu(xx[col]) + eps
    w = EdgeSoftmaxFunction.apply(st, (beta * msg).contiguous())
    return torch.zeros_like(xx).scatter_add_(0, row.unsqueeze(-1).repeat(1, F), msg * w)


def fused(xx):
    return cogdl_b200.genconv_aggregate(st, xx, "softmax_sg", beta=beta, eps=eps)


def fwd_only(fn):
    def call():
        with torch.no_grad():
            fn(x)
    return call


def fwd_bwd(fn):
    xg = x.clone().requires_grad_(True)

    def call():
        xg.grad = beta.grad = None
        fn(xg).backward(r)
    return call


with torch.no_grad():
    got, want = fused(x), reference_sequence(x)
parity = float(((got - want).abs() / want.abs().amax(1, keepdim=True).clamp_min(1e-30)).max())
variants_a = {
    "spmm_raw_us": lambda: spmm_raw(st, None, x),
    "fused_fwd_us": fwd_only(fused),
    "reference_fwd_us": fwd_only(reference_sequence),
    "fused_fwd_bwd_us": fwd_bwd(fused),
    "reference_fwd_bwd_us": fwd_bwd(reference_sequence),
}

# ---------------------------------------------------------------------------------------------- (b)
variants_b = {}
try:
    from tests.refpkg import import_reference

    import_reference()
    from cogdl.data import Graph
    from cogdl.layers import GENConv
    from cogdl.models.nn.deepergcn import DeeperGCN

    cogdl_b200.install(genconv=True)
    from cogdl_b200.install import genconv_forward

    original = GENConv._cogdl_b200_original_forward
    torch.manual_seed(0)
    model = DeeperGCN(F, 128, 40, 4, aggr="softmax_sg", learn_beta=True).to(dev).train()
    rg = torch.repeat_interleave(torch.arange(n, device=dev), rp[1:] - rp[:-1])
    graph = Graph(x=x, edge_index=(rg, col))
    graph.row_indptr
    y = torch.randint(0, 40, (n,), device=dev, generator=torch.Generator(device=dev).manual_seed(1))
    opt = torch.optim.SGD(model.parameters(), lr=0.01)

    def step_with(forward):
        def step():
            GENConv.forward = forward
            opt.zero_grad(set_to_none=True)
            torch.nn.functional.cross_entropy(model(graph), y).backward()
            opt.step()
        return step

    variants_b = {"deepergcn_step_original_ms": step_with(original), "deepergcn_step_patched_ms": step_with(genconv_forward)}
except ImportError as ex:
    print(f"(b) skipped: {ex}")

res = {"arxiv": {"n": n, "nnz": E, "F": F}, "fused_vs_reference_fwd_max_row_rel_err": parity,
       "bytes": {"fwd": fwd_bytes(E, n, F), "fwd_train": fwd_bytes(E, n, F, lse=True), "bwd": bwd_bytes(E, n, F)},
       "rounds": []}
for rnd in range(2):
    rr = {k: statistics.median(event_times(fn, 20, 3, flush=True)) for k, fn in variants_a.items()}
    rr.update({k: statistics.median(event_times(fn, 20, 3, flush=True)) / 1e3 for k, fn in variants_b.items()})
    res["rounds"].append(rr)
    for k, v in rr.items():
        print(f"round {rnd} {k:34s} {v:10.1f}" if k.endswith("_us") else f"round {rnd} {k:34s} {v:10.3f}")
med = {k: statistics.median(rd[k] for rd in res["rounds"]) for k in res["rounds"][0]}
res["summary"] = {
    "fused_fwd_over_spmm": med["fused_fwd_us"] / med["spmm_raw_us"],
    "reference_over_fused_fwd_bwd": med["reference_fwd_bwd_us"] / med["fused_fwd_bwd_us"],
    "reference_over_fused_fwd": med["reference_fwd_us"] / med["fused_fwd_us"],
    "fused_fwd_hbm_fraction": res["bytes"]["fwd"] / (med["fused_fwd_us"] * 1e-6) / PEAK,
}
if variants_b:
    res["summary"]["deepergcn_step_speedup"] = med["deepergcn_step_original_ms"] / med["deepergcn_step_patched_ms"]
fused(x)
res["kernel"] = cogdl_b200._cabi.last_kernel()

# ---------------------------------------------------------------------------------------------- (c)
del variants_a, variants_b
torch.cuda.empty_cache()
np_, ep = synth.SHAPES["products"]
rp2, col2 = synth.powerlaw_csr(np_, ep, seed=0, device=dev, self_loops=False)
st2 = cogdl_b200.CSRStructure.from_int64(rp2, col2)
del rp2, col2
st2.plan
x2 = torch.randn(np_, 256, device=dev)
ts = []
with torch.no_grad():
    peak = peak_above(lambda: ts.extend(
        event_times(lambda: cogdl_b200.genconv_aggregate(st2, x2, "softmax_sg", beta=beta), 20, 3, flush=True)))
t2 = statistics.median(ts)
res["products"] = {"n": np_, "nnz": st2.nnz, "F": 256, "fused_fwd_us": t2, "peak_bytes_above_inputs": peak,
                   "unfused_one_EF_tensor_bytes": st2.nnz * 256 * 4,
                   "fwd_bytes": fwd_bytes(st2.nnz, np_, 256),
                   "fused_fwd_hbm_fraction": fwd_bytes(st2.nnz, np_, 256) / (t2 * 1e-6) / PEAK}
print(json.dumps({k: res[k] for k in ("summary", "products", "kernel", "fused_vs_reference_fwd_max_row_rel_err")}, indent=1))
write_result(out_dir, "time_genconv", res)

"""Fused GraphSAGE layer vs aggregation + cuBLAS on the arxiv shape (CUDA events, L2 flushed, median of 20, TF32 off).

Per aggregation (mean as 1/deg row scale on a CSR-only graph, max) and Fout in {128, 40}, one 128 -> Fout layer with
bias and ReLU:
  unfused_reference_order  aggregate -> cat[x, agg] -> fc            (cogdl/layers/sage_layer.py:69-87)
  unfused_two_addmm        aggregate -> x.W_self^T + b, += agg.W_neigh^T   (no cat)
  fused                    S = x.W_self^T + b, then the fused kernel
and a 2-layer SAGE training step (128 -> 128 -> 40, fwd + bwd + SGD), fused against unfused.  Two rounds, the
variants alternating inside each, so the spread is visible.  Writes time_fused_sage.json to the directory given
on the command line, with the card name and power limit read in the same run.

    python tools/time_fused_sage.py OUT_DIR
"""
import os
import statistics
import sys

import torch
import torch.nn.functional as F
from gpu_timing import event_times, write_result

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cogdl_b200  # noqa: E402
from cogdl_b200 import synth  # noqa: E402
from cogdl_b200.layers import SAGE  # noqa: E402
from cogdl_b200.operators._raw import scatter_max_fwd_raw, spmm_raw  # noqa: E402
from cogdl_b200.operators.fused_sage import fused_sage_raw  # noqa: E402

if len(sys.argv) != 2:
    sys.exit(__doc__)
out_dir = sys.argv[1]
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False

dev = torch.device("cuda")
n, e = synth.SHAPES["arxiv"]
rp, col = synth.powerlaw_csr(n, e, seed=0)
st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n)
st.plan
deg = (rp[1:] - rp[:-1]).float()
inv = torch.where(deg > 0, 1.0 / deg.clamp_min(1), torch.zeros_like(deg)).to(dev).view(n, 1)
x = torch.randn(n, 128, device=dev)


def agg_of(aggr):
    if aggr == "max":
        return lambda: scatter_max_fwd_raw(st, x)[0]
    return lambda: inv * spmm_raw(st, None, x)


def layer_variants(aggr, fout):
    lin = torch.nn.Linear(256, fout).to(dev)
    W, b = lin.weight.detach(), lin.bias.detach()
    Ws, Wn = W[:, :128], W[:, 128:]
    agg = agg_of(aggr)
    kw = ("max", None) if aggr == "max" else ("sum", inv)
    return {
        "unfused_reference_order": lambda: torch.relu_(F.linear(torch.cat([x, agg()], dim=1), W, b)),
        "unfused_two_addmm": lambda: torch.relu_(torch.addmm(torch.addmm(b, x, Ws.t()), agg(), Wn.t())),
        "fused": lambda: fused_sage_raw(st, None, kw[1], x, W, b, kw[0], True),
    }


def step_fn(aggr, fused):
    torch.manual_seed(0)
    model = SAGE(128, 128, 40, aggr=aggr, fused=fused).to(dev)
    graph = cogdl_b200.Graph(x=x, row_ptr=rp, col=col, num_nodes=n).to(dev)
    opt = torch.optim.SGD(model.parameters(), lr=0.01)
    y = torch.randint(0, 40, (n,), device=dev, generator=torch.Generator(device=dev).manual_seed(1))

    def step():
        opt.zero_grad(set_to_none=True)
        F.cross_entropy(model(graph), y).backward()
        opt.step()
    return step


res = {"shape": {"n": n, "nnz": st.nnz, "in_feats": 128}, "unit": "us (layer), ms (train step)",
       "rounds": []}
layers = {(a, f): layer_variants(a, f) for a in ("mean", "max") for f in (128, 40)}
steps = {(a, fu): step_fn(a, fu) for a in ("mean", "max") for fu in (False, True)}
for rnd in range(2):
    r = {}
    for (aggr, fout), variants in layers.items():
        for name, fn in variants.items():
            r[f"{aggr}_F{fout}_{name}_us"] = statistics.median(event_times(fn, 20, 3, flush=True))
    for (aggr, fused), fn in steps.items():
        r[f"train_step_{aggr}_{'fused' if fused else 'unfused'}_ms"] = statistics.median(event_times(fn, 20, 3, flush=True)) / 1e3
    res["rounds"].append(r)
    for k, v in r.items():
        print(f"round {rnd} {k:45s} {v:10.1f}" if k.endswith("_us") else f"round {rnd} {k:45s} {v:10.3f}")
layers[("mean", 128)]["fused"]()
res["kernel_mean"] = cogdl_b200._cabi.last_kernel()
write_result(out_dir, "time_fused_sage", res)

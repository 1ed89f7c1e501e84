"""Fused GCN layer vs SpMM + cuBLAS on the arxiv shape (CUDA events, L2 flushed, median of 20)."""
import os
import statistics
import sys

import torch
from gpu_timing import card, event_times

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cogdl_b200  # noqa: E402
from cogdl_b200 import synth  # noqa: E402
from cogdl_b200.operators._raw import spmm_raw  # noqa: E402
from cogdl_b200.operators.fused_gcn import fused_gcn_raw  # noqa: E402

dev = torch.device("cuda")
n, e = synth.SHAPES["arxiv"]
rp, col = synth.powerlaw_csr(n, e, seed=0)
w = synth.sym_norm_weights(rp, col).to(dev)
st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n)
st.plan
x = torch.randn(n, 128, device=dev)
print("card:", card(), flush=True)


def median_min(fn):
    ts = event_times(fn, 20, 3, flush=True)
    return statistics.median(ts), min(ts)


for fout in (128, 40):
    lin = torch.nn.Linear(128, fout).to(dev)
    W, b = lin.weight.detach().contiguous(), lin.bias.detach().contiguous()
    for tf32 in (False, True):
        torch.backends.cuda.matmul.allow_tf32 = tf32
        torch.backends.cudnn.allow_tf32 = tf32
        tag = "tf32" if tf32 else "fp32"
        print(f"Fout={fout} unfused gemm({tag})+bias -> spmm -> relu", median_min(lambda: torch.relu_(spmm_raw(st, w, torch.addmm(b, x, W.t())))))
        print(f"Fout={fout} unfused spmm -> gemm({tag}) -> relu      ", median_min(lambda: torch.relu_(spmm_raw(st, w, x) @ W.t())))
    torch.backends.cuda.matmul.allow_tf32 = False
    print(f"Fout={fout} spmm alone (F=128)                       ", median_min(lambda: spmm_raw(st, w, x)))
    print(f"Fout={fout} FUSED wgmma                               ", median_min(lambda: fused_gcn_raw(st, w, x, W, b, True)))

"""Run every op of the GAT / SAGE configs a few times on the arxiv shape (for `ncu` launch lists):
   ncu --metrics gpu__time_duration.sum --clock-control none --csv --log-file out.csv python tools/profile_ops.py"""
import os
import sys

import torch
from gpu_timing import flush_l2

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cogdl_b200  # noqa: E402
from cogdl_b200 import synth  # noqa: E402
from cogdl_b200.operators._raw import (edge_softmax_bwd_raw, edge_softmax_fwd_raw, gat_fwd_raw, mhsddmm_raw,  # noqa: E402
                                       mhspmm_raw, sddmm_raw, spmm_raw)

dev = torch.device("cuda")
n, e = synth.SHAPES["arxiv"]
rp, col = synth.powerlaw_csr(n, e, seed=0)
w = synth.sym_norm_weights(rp, col).to(dev)
st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n)
H, F = 8, 128
logits = (torch.randn(st.nnz, H, device=dev) * 3).clamp_(-10, 10)
x = torch.randn(n, F, device=dev)
h = torch.randn(n, H, F, device=dev)
hl, hr = torch.randn(n, H, device=dev), torch.randn(n, H, device=dev)
for it in range(3):
    flush_l2()
    att = edge_softmax_fwd_raw(st, logits)
    flush_l2()
    edge_softmax_bwd_raw(st, att, logits)
    flush_l2()
    gat_fwd_raw(st, hl, hr, h, 0.2, True)
    flush_l2()
    mhsddmm_raw(st, h, h)
    flush_l2()
    sddmm_raw(st, x, x)
    flush_l2()
    spmm_raw(st, w, x)
torch.cuda.synchronize()
print("done")

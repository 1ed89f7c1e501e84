"""Only the fused GCN layer, a few times (for ncu): python tools/profile_fused.py [Fout]"""
import os
import sys

import torch
from gpu_timing import flush_l2

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cogdl_b200  # noqa: E402
from cogdl_b200 import synth  # noqa: E402
from cogdl_b200.operators.fused_gcn import fused_gcn_raw  # noqa: E402

dev = torch.device("cuda")
n, e = synth.SHAPES["arxiv"]
rp, col = synth.powerlaw_csr(n, e, seed=0)
w = synth.sym_norm_weights(rp, col).to(dev)
st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n)
st.plan
fout = int(sys.argv[1]) if len(sys.argv) > 1 else 128
x = torch.randn(n, 128, device=dev)
lin = torch.nn.Linear(128, fout).to(dev)
W, b = lin.weight.detach().contiguous(), lin.bias.detach().contiguous()
for _ in range(4):
    flush_l2()
    fused_gcn_raw(st, w, x, W, b, True)
torch.cuda.synchronize()
print("done")

"""Ours vs the reference's OWN CUDA kernels (compiled unchanged for sm_90a into oracle/_ref/cuda) on the
same H100 and the same inputs -- the "existing GPU kernel" baseline of BASELINE.md 3.5.  Baseline tool,
not part of the product path or of bench.py.  Prints one RESULT line per op (median of 7, L2 flushed)."""
import os
import statistics
import sys

import torch
from gpu_timing import card, event_times

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cogdl_b200  # noqa: E402
import oracle  # noqa: E402
from cogdl_b200 import synth  # noqa: E402
from cogdl_b200.operators._raw import edge_softmax_fwd_raw, mhspmm_raw, scatter_max_fwd_raw, spmm_raw  # noqa: E402

dev = torch.device("cuda")
print("card:", card(), flush=True)


def median_us(fn):
    return statistics.median(event_times(fn, 7, 2, flush=True))


n, e = synth.SHAPES["arxiv"]
rp, col = synth.powerlaw_csr(n, e, seed=0)
w = synth.sym_norm_weights(rp, col).to(dev)
st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n)
x = torch.randn(n, 128, device=dev)
rows = []
ref = oracle.ref_module("spmm", "cuda")
rows.append(("spmm_F128", median_us(lambda: spmm_raw(st, w, x)), median_us(lambda: ref.csr_spmm(st.rowptr, st.colind, w, x))))
H = 8
logits = (torch.randn(st.nnz, H, device=dev) * 3).clamp_(-10, 10)
ref_es = oracle.ref_module("edge_softmax", "cuda")
rows.append(("edge_softmax_H8", median_us(lambda: edge_softmax_fwd_raw(st, logits)), median_us(lambda: ref_es.edge_softmax(st.rowptr, logits))))
att = edge_softmax_fwd_raw(st, logits)
h = torch.randn(n, H, 128, device=dev)
ref_mh = oracle.ref_module("mhspmm", "cuda")
rows.append(("mhspmm_H8_F128", median_us(lambda: mhspmm_raw(st, att, h)), median_us(lambda: ref_mh.mhspmm(st.rowptr, st.colind, att, h))))
xp = x.abs() + 0.01
ref_sm = oracle.ref_module("scatter_max", "cuda")
rows.append(("scatter_max_F128", median_us(lambda: scatter_max_fwd_raw(st, xp)), median_us(lambda: ref_sm.scatter_max_fp(st.rowptr, st.colind, xp))))
for name, ours, theirs in rows:
    print(f"RESULT {name}: ours {ours:.1f} us   reference CUDA kernel (sm_90a build) {theirs:.1f} us   speed-up {theirs / ours:.2f}x", flush=True)

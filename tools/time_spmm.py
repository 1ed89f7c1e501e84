"""Gather-kernel timings on the arxiv shape (CUDA events, L2 flushed, median of 30), with a SHA-256 of every output.

Inputs are seeded, so the hashes of two builds match exactly when the builds compute the same bits.

  python tools/time_spmm.py              # every workload below
  python tools/time_spmm.py 128 40       # only the SpMM (default plan) at these widths
"""
import os
import statistics
import sys

import torch
from gpu_timing import card, digest, event_times

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cogdl_b200  # noqa: E402
from cogdl_b200 import _cabi, synth  # noqa: E402
from cogdl_b200.operators._raw import mhspmm_raw, scatter_max_fwd_raw, spmm_raw  # noqa: E402

dev = torch.device("cuda")
n, e = synth.SHAPES["arxiv"]
rp, col = synth.powerlaw_csr(n, e, seed=0)
w = synth.sym_norm_weights(rp, col).to(dev)
st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n)
st.plan
st_noplan = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n, chunk_edges=0)
print("card:", card(), flush=True)


def randn(*shape, seed):
    return torch.randn(*shape, device=dev, generator=torch.Generator(device=dev).manual_seed(seed))


def report(label, fn, algo=None):
    out = fn()
    ts = event_times(fn, 30, 2, flush=True)
    med = statistics.median(ts)
    rate = f"{algo / med / 1e3:7.0f} GB/s" if algo else " " * 12
    out = out if isinstance(out, tuple) else (out,)
    print(f"{label:32s} median {med:8.1f} us min {min(ts):8.1f} us {rate}  sha256 {digest(*out)}  [{_cabi.last_kernel()}]")


def spmm(F, structure=st, tag="", weights=(w, None)):
    x = randn(n, F, seed=F)
    for wt in weights:
        algo = st.nnz * (4 * F + (8 if wt is not None else 4)) + n * (4 * F + 4)
        report(f"spmm F={F} {'weighted' if wt is not None else 'unweighted'}{tag}", lambda: spmm_raw(structure, wt, x), algo)


if sys.argv[1:]:
    for F in (int(a) for a in sys.argv[1:]):
        spmm(F)
    sys.exit(0)
for F in (7, 16, 32):
    spmm(F)
spmm(128, st_noplan, " chunk_edges=0")
for H, F in ((8, 8), (4, 8), (1, 16)):
    att, feat = torch.rand(st.nnz, H, device=dev, generator=torch.Generator(device=dev).manual_seed(H)), randn(n, H, F, seed=F)
    report(f"mhspmm H={H} F={F}", lambda: mhspmm_raw(st, att, feat))
for F in (4, 7, 8, 16, 40, 128, 256):
    x = randn(n, F, seed=F)
    report(f"scatter_max F={F}", lambda: scatter_max_fwd_raw(st, x))

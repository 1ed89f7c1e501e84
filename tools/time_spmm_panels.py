"""Column-panel SpMM on the arxiv shape (bench.py's N = 1 workload): how much of the time is L2 misses on X.

  python tools/time_spmm_panels.py fold  [--rounds R] [--steps S]
      the single-pass kernel (panels=1) on the same rowptr / hub plan / nnz with columns folded to `col % (n/k)` and an X of n/k
      rows, k in {1, 2, 4, 8}: only the X working set changes (87, 43, 22, 11 MB at F = 128).
  python tools/time_spmm_panels.py sweep [--F 128 256] [--rounds R] [--steps S]
      the same SpMM with the panel count forced to P in {1, 2, 4} (and 8 at F = 256) next to the automatic
      choice; every variant's output must be bitwise equal to P = 1.

Variants alternate round by round (R rounds x S steps each); CUDA events around each call, the L2 flushed
(512 MiB write) before each one, outside the interval.  Prints median, min and the spread of the per-round
medians, and the card's name, power limit and max SM clock.
"""
import argparse
import os
import statistics
import sys

import torch
from gpu_timing import alternate, card

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import cogdl_b200  # noqa: E402
from cogdl_b200 import _cabi, synth  # noqa: E402
from cogdl_b200.operators._raw import spmm_raw  # noqa: E402


def report(res, base, notes):
    t0 = statistics.median(res[base][0])
    for name, (ts, meds) in res.items():
        med = statistics.median(ts)
        print(f"  {name:>10}  median {med:7.1f} us  min {min(ts):7.1f}  round medians {min(meds):7.1f}..{max(meds):7.1f}"
              f"  x{t0 / med:5.2f} vs {base}  [{notes.get(name, '')}]", flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("mode", choices=["fold", "sweep"])
    ap.add_argument("--F", type=int, nargs="+", default=[128, 256])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    args = ap.parse_args()
    dev = torch.device("cuda")
    print("card:", card(), flush=True)
    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, self_loops=True)
    w = synth.sym_norm_weights(rp, col).to(dev)
    gen = torch.Generator(device=dev).manual_seed(0)

    if args.mode == "fold":
        F = 128
        variants, notes = {}, {}
        for k in (1, 2, 4, 8):
            m = n // k
            st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), (col % m).to(dev), n_cols=m)
            st.plan
            x = torch.randn(m, F, device=dev, generator=gen)
            variants[f"k={k}"] = (lambda st=st, x=x: spmm_raw(st, w, x, panels=1))   # the single-pass kernel
            notes[f"k={k}"] = f"X {m * F * 4 / 1e6:.1f} MB"
        res = alternate(variants, args.rounds, args.steps, 3, flush=True, sync_each=False)
        variants["k=1"]()
        notes["k=1"] += ", " + _cabi.last_kernel()
        print(f"fold curve: arxiv shape, weighted, F={F}, nnz={int(col.numel())}", flush=True)
        report(res, "k=1", notes)
        return

    st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n)
    st.plan
    for F in args.F:
        x = torch.randn(n, F, device=dev, generator=gen)
        ps = [1, 2, 4] + ([8] if F >= 256 else [])
        variants = {f"P={p}": (lambda p=p: spmm_raw(st, w, x, panels=p)) for p in ps}
        variants["auto"] = lambda: spmm_raw(st, w, x)
        notes = {}
        y1 = spmm_raw(st, w, x, panels=1)
        for name, fn in variants.items():
            y = fn()
            notes[name] = ("bitwise == P=1" if torch.equal(y.view(torch.int32), y1.view(torch.int32)) else "DIFFERS from P=1") + \
                ", " + _cabi.last_kernel()
        res = alternate(variants, args.rounds, args.steps, 3, flush=True, sync_each=False)
        print(f"panel sweep: arxiv shape, weighted, F={F}, X {n * F * 4 / 1e6:.1f} MB", flush=True)
        report(res, "P=1", notes)


if __name__ == "__main__":
    main()

"""SpMM on bench.py's N = 1 workload, several builds side by side: where the L2 goes in the column-panel passes.

  python tools/time_spmm_l2.py --base DIR [DIR ...] [--rounds R] [--steps S]

Each DIR is another tree of this project with its library built (for instance a checkout of the parent commit
after `make -C cogdl_b200/csrc`).  Each tree, this one included, runs in a worker process of its own that imports
cogdl_b200 from that tree; the workers take turns, variant by variant and round by round, so every build sees the
same card state.

Variants, all on the arxiv shape (169 343 rows, seed 0, self loops, sym-normalised weights), F = 128:
  bench   spmm(graph, x) with the automatic panel count (2 panels of 64 floats on a 50 MB L2): bench.py's value
  fold=k  the single-pass kernel (panels=1) with columns folded to `col % (n/k)` and an X of n/k rows,
          k in {1, 2, 4}: same rowptr, hub plan and nnz, only the X working set changes (87, 43, 22 MB).
  F40     the same SpMM at F = 40 (one pass, float4 lanes): bench.py's C2_spmm_F40.

Each step is timed with CUDA events, with the L2 flushed (512 MiB write) before it, outside the interval.  Prints
the median, min and per-round spread of every (build, variant), whether each build's output is bitwise equal
to this tree's, the launched kernel, the card's name, power limit and max SM clock, and the throttle reasons
active after the run.  No DRAM traffic is measured: the byte figures printed are computed from the shapes.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

from gpu_timing import card, digest, event_times

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
F = 128
FOLDS = (1, 2, 4)


def worker(tree, steps):
    """Serve timing commands on stdin for the build in `tree`; one JSON line out per line in."""
    sys.path.insert(0, tree)
    import torch

    import cogdl_b200
    from cogdl_b200 import _cabi, synth
    from cogdl_b200.operators._raw import spmm_raw

    assert os.path.realpath(cogdl_b200.__file__).startswith(os.path.realpath(tree)), cogdl_b200.__file__
    dev = torch.device("cuda")
    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, self_loops=True)
    w = synth.sym_norm_weights(rp, col).to(dev)
    gen = torch.Generator(device=dev).manual_seed(0)
    variants = {}
    st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n)
    st.plan
    x = torch.randn(n, F, device=dev, generator=gen)
    variants["bench"] = lambda: spmm_raw(st, w, x)
    for k in FOLDS:
        m = n // k
        stk = cogdl_b200.CSRStructure.from_int64(rp.to(dev), (col % m).to(dev), n_cols=m)
        stk.plan
        xk = torch.randn(m, F, device=dev, generator=gen)
        variants[f"fold={k}"] = (lambda stk=stk, xk=xk: spmm_raw(stk, w, xk, panels=1))
    x40 = torch.randn(n, 40, device=dev, generator=gen)
    variants["F40"] = lambda: spmm_raw(st, w, x40)
    info = {}
    for name, fn in variants.items():
        y = fn()
        torch.cuda.synchronize()
        info[name] = {"kernel": _cabi.last_kernel(), "sha256": digest(y)}
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    print(json.dumps({"ready": info, "nnz": int(col.numel()), "n": n}), flush=True)
    for line in sys.stdin:
        print(json.dumps(event_times(variants[line.strip()], steps, 0, flush=True, sync_each=False)), flush=True)


def single_use_bytes(n, nnz, panels, edge_row):
    """Bytes of one call that are read or written once per pass, from the shapes: colind + val (+ edge_row) per
    edge and the output rows; rowptr (4 (n + 1) per pass) only when row ends come from it."""
    per_pass = nnz * (4 + 4 + (4 if edge_row else 0)) + (0 if edge_row else 4 * (n + 1))
    return panels * per_pass + n * F * 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--base", required=True, nargs="+", help="other trees of this project with their library built")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--worker", default=None, help=argparse.SUPPRESS)
    args = ap.parse_args()
    if args.worker:
        worker(args.worker, args.steps)
        return

    print("card:", card(), flush=True)
    trees = {"this": ROOT}
    for d in args.base:
        trees[os.path.basename(os.path.normpath(d))] = os.path.abspath(d)
    procs, ready = {}, {}
    for tag, tree in trees.items():
        procs[tag] = subprocess.Popen([sys.executable, os.path.abspath(__file__), "--base", tree, "--worker", tree,
                                       "--steps", str(args.steps)], stdin=subprocess.PIPE, stdout=subprocess.PIPE,
                                      text=True)
        ready[tag] = json.loads(procs[tag].stdout.readline())
    names = list(ready["this"]["ready"])
    times = {(t, v): ([], []) for t in trees for v in names}
    try:
        for rnd in range(args.rounds):
            for v in names:
                for t in (list(trees) if rnd % 2 == 0 else list(trees)[::-1]):
                    procs[t].stdin.write(v + "\n")
                    procs[t].stdin.flush()
                    ts = json.loads(procs[t].stdout.readline())
                    times[(t, v)][0].extend(ts)
                    times[(t, v)][1].append(statistics.median(ts))
    finally:
        for p in procs.values():
            p.stdin.close()
            p.wait()
    print("throttle reasons after the run (hw, hw_thermal, sw_thermal, sw_power_cap):",
          card("clocks_event_reasons.hw_slowdown,clocks_event_reasons.hw_thermal_slowdown,"
               "clocks_event_reasons.sw_thermal_slowdown,clocks_event_reasons.sw_power_cap"), flush=True)
    n, nnz = ready["this"]["n"], ready["this"]["nnz"]
    print(f"arxiv shape, weighted, F={F}, n={n}, nnz={nnz}; {args.rounds} rounds x {args.steps} steps, L2 flushed")
    width = max(len(t) for t in trees)
    for v in names:
        m0 = statistics.median(times[("this", v)][0])
        for t in trees:
            ts, meds = times[(t, v)]
            m = statistics.median(ts)
            same = ready[t]["ready"][v]["sha256"] == ready["this"]["ready"][v]["sha256"]
            print(f"  {v:>7} {t:>{width}}  median {m:7.1f} us  min {min(ts):7.1f}  round medians {min(meds):7.1f}.."
                  f"{max(meds):7.1f}  this/{t} {m0 / m:.3f}  {'' if same else 'OUTPUT DIFFERS  '}"
                  f"[{ready[t]['ready'][v]['kernel']}]")
    for label, er in (("edge_row", True), ("rowptr", False)):
        print(f"single-use bytes per bench call (computed from shapes, 2 panels, row ends from {label}): "
              f"{single_use_bytes(n, nnz, 2, er) / 1e6:.1f} MB; X panel {n * F * 2 / 1e6:.1f} MB")


if __name__ == "__main__":
    main()

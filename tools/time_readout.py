"""Time the graph-level readouts on the GPU against the reference's own code, in one process:

- each pooling op (sum, mean, max; forward + backward, F = 64): cogdl_b200's against cogdl.utils.batch_*_pooling;
- the reference GIN graph-classification training step (5 layers, hidden 64, forward, cross-entropy, backward, Adam),
  under install(gin=True) with and without readout=True;
- the reference SortPool training step at k = 30, the same way;

at a molecular shape (128 graphs of about 26 nodes) and a large-graph shape (32 graphs of about 500 nodes), random graphs
with about 2 edges per node each way.  The readout path is timed on a batch vector it has seen (`cached`: the membership
is built once) and on a fresh copy of it per step (`fresh`: a data loader's new batch, so every step builds the
membership, its transpose and both hub plans).  Variants alternate for --rounds rounds after a warm-up, each timed over
--steps calls ending in a device synchronise (CUDA events); figures are medians in us.  The card's name and power limit
are read in the same run.  Prints one JSON line and writes it to --out/time_readout.json if given.
"""
import argparse
import json
import os
import statistics
import sys

import numpy as np
import torch
import torch.nn.functional as F
from gpu_timing import alternate, card, write_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"molecular": (128, 26), "large": (32, 500)}
HIDDEN, CLASSES, FEATS, K = 64, 2, 16, 30


def make_batch(Graph, n_graphs, mean_n, dev, seed=0):
    rng = np.random.default_rng(seed)
    rows, cols, batch, off = [], [], [], 0
    for b in range(n_graphs):
        n = int(rng.integers(mean_n // 2, 3 * mean_n // 2 + 1))
        r, c = rng.integers(0, n, 2 * n), rng.integers(0, n, 2 * n)
        rows += [r + off, c + off]
        cols += [c + off, r + off]
        batch.append(np.full(n, b))
        off += n
    g = Graph(x=torch.from_numpy(rng.standard_normal((off, FEATS)).astype(np.float32)),
              edge_index=(torch.from_numpy(np.concatenate(rows)), torch.from_numpy(np.concatenate(cols))),
              y=torch.from_numpy(rng.integers(0, CLASSES, n_graphs)))
    g.batch = torch.from_numpy(np.concatenate(batch))
    g = g.to(dev)
    g.row_indptr
    return g


def med(out):
    return {k: statistics.median(v[1]) for k, v in out.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--out")
    a = ap.parse_args()

    from tests.refpkg import import_reference

    import_reference()
    import cogdl.utils.utils as uu
    from cogdl.data import Graph
    from cogdl.models.nn.gin import GIN
    from cogdl.models.nn.sortpool import SortPool

    import cogdl_b200
    from cogdl_b200.install import install_readout

    ref_pool = {m: getattr(uu, f"batch_{m}_pooling") for m in ("sum", "mean", "max")}
    cogdl_b200.install(gin=True)
    dev = torch.device("cuda:0")
    res = {"card": card(), "rounds": a.rounds, "steps": a.steps, "unit": "us, median"}
    for shape, (B, n) in SHAPES.items():
        g = make_batch(Graph, B, n, dev)
        batch = g.batch
        x = torch.randn(batch.numel(), HIDDEN, device=dev, requires_grad=True)
        dy = torch.randn(B, HIDDEN, device=dev)
        ops = {}
        for m in ("sum", "mean", "max"):
            ours = getattr(cogdl_b200, f"batch_{m}_pooling")
            ops[f"{m}_readout_cached"] = lambda ours=ours: torch.autograd.grad(ours(x, batch), x, dy)
            ops[f"{m}_readout_fresh"] = lambda ours=ours: torch.autograd.grad(ours(x, batch.clone()), x, dy)
            try:
                torch.autograd.grad(ref_pool[m](x, batch), x, dy)
                ops[f"{m}_reference"] = lambda m=m: torch.autograd.grad(ref_pool[m](x, batch), x, dy)
            except Exception as ex:  # noqa: BLE001  (the reference's max falls back to torch_scatter when missing)
                res[f"{shape}_{m}_reference"] = f"does not run: {type(ex).__name__}: {ex}"[:200]
        res[f"{shape}_pool_F{HIDDEN}"] = med(alternate(ops, a.rounds, a.steps, a.warmup, flush=False))

        torch.manual_seed(0)
        gin = GIN(5, FEATS, CLASSES, HIDDEN, 2, 0.0, "sum", True, 0.5).to(dev)
        torch.manual_seed(1)
        sp = SortPool(FEATS, HIDDEN, CLASSES, 2, 32, 5, k=K, dropout=0.5).to(dev)
        opts = {id(gin): torch.optim.Adam(gin.parameters(), 1e-3), id(sp): torch.optim.Adam(sp.parameters(), 1e-3)}

        def step(model, fresh):
            if fresh:
                g.batch = g.batch.clone()       # a new batch vector: the membership cache misses
            opt = opts[id(model)]
            opt.zero_grad(set_to_none=True)
            loss = F.cross_entropy(model(g), g.y)
            loss.backward()
            opt.step()

        state = {"on": None}

        def flag(on, fn):
            """fn with the readout rebinding on or off; it changes at most once per round, so the rebinding's host work
            lands in one timed call of the round and not in its median."""
            def run():
                if state["on"] != on:
                    (install_readout if on else cogdl_b200.uninstall_readout)()
                    state["on"] = on
                fn()
            return run

        variants = {}
        for name, model in (("gin", gin), ("sortpool", sp)):
            variants[f"{name}_reference"] = flag(False, lambda model=model: step(model, False))
            variants[f"{name}_readout_cached"] = flag(True, lambda model=model: step(model, False))
            variants[f"{name}_readout_fresh"] = flag(True, lambda model=model: step(model, True))
        res[f"{shape}_train_step"] = med(alternate(variants, a.rounds, max(a.steps // 3, 5), a.warmup, flush=False))
        res[f"{shape}_nodes"] = int(batch.numel())
    cogdl_b200.uninstall_readout()
    print(json.dumps(res))
    if a.out:
        write_result(a.out, "time_readout", res)


if __name__ == "__main__":
    main()

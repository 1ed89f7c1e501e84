"""Time GIN's aggregation and GRAND's propagation on the GPU, fused against the reference's op sequence run with this
package's spmm, on synthetic power-law graphs (cogdl_b200/synth.py):

- GIN: `(1 + eps) * x + spmm(graph, x)` forward + backward (d x and d eps) at the arxiv shape, F = 128 and F = 64:
  cogdl_b200.gin_aggregate (one launch each way) against autograd through the expression;
- GRAND: rand_prop after DropNode with order = 8 at the Cora (F = 1433 and 128), PubMed (F = 500 and 128) and arxiv
  (F = 128) shapes on sym-normalised weights: cogdl_b200.random_propagate against the reference loop (spmm, add_, and a
  final div_).  random_propagate runs one fused launch per hop for F <= 128 (a multiple of 4) and the reference loop on
  this package's spmm otherwise; `path` says which.  And a GRAND forward with sample = 4 (normalize_x, DropNode,
  rand_prop, dropout and the two linear layers of cogdl/models/nn/grand.py, four times) on each shape.

Fused and unfused runs alternate for --rounds rounds after a warm-up, in one process; each figure is the median over
rounds of a loop of --iters calls (CUDA events), in ms per call.  The outputs of the two paths are compared bit for bit
at the timed size.  The card's name and power limit are read in the same run.  Prints one JSON line and writes it to
--out if given.
"""
import argparse
import json
import os
import statistics
import sys

import torch
import torch.nn.functional as F
from gpu_timing import card, event_times

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"cora": (2708, 10556, 1433), "pubmed": (19717, 88648, 500), "arxiv": (169343, 1166243, 128)}
GRAND_RUNS = [("cora", 1433), ("cora", 128), ("pubmed", 500), ("pubmed", 128), ("arxiv", 128)]
ORDER, SAMPLE, DROPNODE, HIDDEN, CLASSES = 8, 4, 0.5, 32, 7


def per_call_ms(fn, iters):
    """ms per call over one CUDA-event window of `iters` back-to-back calls of fn, after one warm-up call, and the last
    call's result."""
    fn()
    last = [None]

    def loop():
        for _ in range(iters):
            last[0] = fn()
    return event_times(loop, 1, 0, flush=False)[0] / 1e3 / iters, last[0]


def graph(name, dev, norm):
    import cogdl_b200
    from cogdl_b200 import synth

    n, e, _ = SHAPES[name]
    rp, col = synth.powerlaw_csr(n, e, seed=1, device=dev)
    row = torch.repeat_interleave(torch.arange(n, device=dev), rp[1:] - rp[:-1])
    g = cogdl_b200.Graph(edge_index=(row, col), num_nodes=n)
    if norm:
        g.sym_norm()
    g.row_indptr
    return g


def gin_step(g, x, eps, G, fused):
    import cogdl_b200

    out = cogdl_b200.gin_aggregate(g, x, eps) if fused else (1 + eps) * x + cogdl_b200.spmm(g, x)
    dx, deps = torch.autograd.grad(out, [x, eps], G)
    return out.detach(), dx


def rand_prop(g, x, fused):
    import cogdl_b200

    if fused:
        return cogdl_b200.random_propagate(g, x, ORDER)
    y = x
    for _ in range(ORDER):
        x = cogdl_b200.spmm(g, x).detach_()
        y.add_(x)
    return y.div_(ORDER + 1.0).detach_()


def grand_forward(g, x, l1, l2, fused):
    """GRAND's forward (cogdl/models/nn/grand.py) SAMPLE times, as GrandModelWrapper.train_step runs it."""
    outs = []
    for _ in range(SAMPLE):
        row_inv = x.sum(1).pow_(-1)
        row_inv.masked_fill_(row_inv == float("inf"), 0)
        h = x * row_inv[:, None]
        masks = torch.bernoulli(1.0 - torch.ones(h.shape[0]) * DROPNODE).unsqueeze(1)
        h = rand_prop(g, masks.to(h.device) * h, fused)
        h = F.dropout(h, 0.5, training=True)
        h = F.relu(l1(h))
        h = F.dropout(h, 0.5, training=True)
        outs.append(l2(h))
    return torch.stack(outs)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out")
    a = ap.parse_args()

    dev = torch.device("cuda:0")
    res = {"card": card(), "rounds": a.rounds, "iters": a.iters, "order": ORDER, "sample": SAMPLE}
    gen = torch.Generator(device=dev).manual_seed(0)
    g = graph("arxiv", dev, norm=False)
    n = SHAPES["arxiv"][0]
    for Fd in (128, 64):
        x = torch.randn(n, Fd, device=dev, generator=gen).requires_grad_(True)
        eps = torch.zeros(1, device=dev).requires_grad_(True)
        G = torch.randn(n, Fd, device=dev, generator=gen)
        t = {True: [], False: []}
        outs = {}
        for _ in range(a.rounds):
            for fused in (False, True):
                ms, outs[fused] = per_call_ms(lambda: gin_step(g, x, eps, G, fused), a.iters)
                t[fused].append(ms)
        same = all(torch.equal(p.view(torch.int32), q.view(torch.int32)) for p, q in zip(outs[True], outs[False]))
        res[f"gin_arxiv_F{Fd}"] = {"fused_ms": statistics.median(t[True]), "unfused_ms": statistics.median(t[False]),
                                   "ratio": statistics.median(t[True]) / statistics.median(t[False]),
                                   "bit_identical": bool(same)}
    from cogdl_b200.operators.grand import fused_hops

    for name, Fd in GRAND_RUNS:
        n = SHAPES[name][0]
        g = graph(name, dev, norm=True)
        x = torch.rand(n, Fd, device=dev, generator=gen)
        l1, l2 = torch.nn.Linear(Fd, HIDDEN).to(dev), torch.nn.Linear(HIDDEN, CLASSES).to(dev)
        t = {(k, f): [] for k in ("rand_prop", "forward") for f in (True, False)}
        outs = {}
        for _ in range(a.rounds):
            for fused in (False, True):
                ms, outs[fused] = per_call_ms(lambda: rand_prop(g, x.clone(), fused), a.iters)
                t[("rand_prop", fused)].append(ms)
                with torch.no_grad():
                    ms, _ = per_call_ms(lambda: grand_forward(g, x, l1, l2, fused), max(1, a.iters // 4))
                t[("forward", fused)].append(ms)
        same = torch.equal(outs[True].view(torch.int32), outs[False].view(torch.int32))
        for k in ("rand_prop", "forward"):
            f, u = statistics.median(t[(k, True)]), statistics.median(t[(k, False)])
            res[f"grand_{k}_{name}_F{Fd}"] = {"fused_ms": f, "unfused_ms": u, "ratio": f / u}
        res[f"grand_rand_prop_{name}_F{Fd}"]["bit_identical"] = bool(same)
        res[f"grand_rand_prop_{name}_F{Fd}"]["path"] = "fused" if fused_hops(x) else "spmm + add_"
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()

"""Time Correct & Smooth's label propagation on the GPU, fused (cogdl_b200.label_propagate: one SpMM launch per step,
the in_norm, scaling, addition, clamp and row reset in its store) against the reference's op sequence run with this
package's spmm (`alpha * spmm`, `+= (1 - alpha) * labels`, then torch.clamp or `x[nid] = labels[nid]`), on synthetic
power-law graphs (cogdl_b200/synth.py) of the arxiv shape (C = 40) and the products shape (C = 47):

- the two loops of one CorrectSmooth call at the reference's defaults: 50 correct steps (alpha 1.0, sym-normalised
  weights, the training rows reset) and 50 smooth steps (alpha 0.8, row-normalised weights, clamp to [0, 1]);
- a whole reference CorrectSmoothMLP.postprocess (softmax, both loops, the autoscale-free correction, the graph
  normalisations and one-hot set-up it does per call) through install() and install(correct_smooth=True).

Fused and unfused runs alternate for --rounds rounds after a warm-up, in one process; each figure is the median over
rounds (CUDA events).  The outputs of the two paths are compared bit for bit at the timed size.  The card's name and
power limit are read in the same run.  Prints one JSON line and writes it to --out if given.
"""
import argparse
import json
import os
import statistics
import sys

import torch
from gpu_timing import card, event_times

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = {"arxiv": (169343, 1166243, 40), "products": (2449029, 61859140, 47)}
NPROP, CORRECT_ALPHA, SMOOTH_ALPHA, TRAIN_SHARE = 50, 1.0, 0.8, 0.54


def loops(g1, g2, labels, nid, fused):
    import cogdl_b200

    if fused:
        r = cogdl_b200.label_propagate(g1, labels, CORRECT_ALPHA, NPROP, pinned=nid)
        return cogdl_b200.label_propagate(g2, r, SMOOTH_ALPHA, NPROP, lower=0, upper=1)
    r = labels.clone()
    for _ in range(NPROP):
        r = CORRECT_ALPHA * cogdl_b200.spmm(g1, r)
        r += (1 - CORRECT_ALPHA) * labels
        r[nid] = labels[nid]
    s0 = r
    r = s0.clone()
    for _ in range(NPROP):
        r = SMOOTH_ALPHA * cogdl_b200.spmm(g2, r)
        r += (1 - SMOOTH_ALPHA) * s0
        r = torch.clamp(r, 0, 1)
    return r


def postprocess_model(C):
    from cogdl.models.nn.correct_smooth import CorrectSmoothMLP

    p = argparse.ArgumentParser()
    CorrectSmoothMLP.add_args(p)
    args = p.parse_args(["--num-features", "8", "--num-classes", str(C), "--num-correct-prop", str(NPROP),
                         "--num-smooth-prop", str(NPROP), "--correct-norm", "sym", "--smooth-norm", "row"])
    args.dataset = "synthetic"
    return CorrectSmoothMLP(args)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--shapes", default="arxiv,products")
    ap.add_argument("--no-postprocess", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()

    import cogdl_b200
    from cogdl_b200 import synth

    dev = torch.device("cuda:0")
    res = {"card": card(), "rounds": a.rounds, "nprop": [NPROP, NPROP]}
    ref = None
    if not a.no_postprocess:
        from tests.refpkg import import_reference

        ref = import_reference()
        cogdl_b200.install()
    for name in a.shapes.split(","):
        n, e, C = SHAPES[name]
        rp, col = synth.powerlaw_csr(n, e, seed=1, device=dev)
        row = torch.repeat_interleave(torch.arange(n, device=dev), rp[1:] - rp[:-1])
        g1 = cogdl_b200.Graph(edge_index=(row, col), num_nodes=n)
        g1.sym_norm()
        g2 = cogdl_b200.Graph(edge_index=(row, col), num_nodes=n)
        g2.row_norm()
        gen = torch.Generator(device=dev).manual_seed(0)
        labels = torch.softmax(torch.randn(n, C, device=dev, generator=gen), -1)
        nid = torch.nonzero(torch.rand(n, device=dev, generator=gen) < TRAIN_SHARE).view(-1)
        with torch.no_grad():
            ref_out = loops(g1, g2, labels, nid, False)
            same = bool(torch.equal(ref_out.view(torch.int32), loops(g1, g2, labels, nid, True).view(torch.int32)))
            t = {False: [], True: []}
            for _ in range(a.rounds):
                for fused in (False, True):
                    t[fused].append(event_times(lambda: loops(g1, g2, labels, nid, fused), 1, 0, flush=False)[0] / 1e3)
        u, f = statistics.median(t[False]), statistics.median(t[True])
        r = {"nodes": n, "edges": int(rp[-1]), "C": C, "unfused_ms": round(u, 2), "fused_ms": round(f, 2),
             "ratio": round(f / u, 3), "bit_identical": same,
             "spread_ms": {"unfused": [round(min(t[False]), 2), round(max(t[False]), 2)],
                           "fused": [round(min(t[True]), 2), round(max(t[True]), 2)]}}
        del g1, g2, ref_out
        if ref is not None:
            from cogdl.data import Graph

            split = torch.rand(n)
            graph = Graph(x=torch.zeros(n, 1), y=torch.randint(0, C, (n,)), edge_index=(row.cpu(), col.cpu()),
                          train_mask=split < TRAIN_SHARE, val_mask=(split >= TRAIN_SHARE) & (split < 0.8),
                          test_mask=split >= 0.8).to(dev)
            model = postprocess_model(C)
            logits = torch.randn(n, C, device=dev)
            pt = {False: [], True: []}
            outs = {}

            def postprocess(fused):
                outs[fused] = model.postprocess(graph, logits)
            with torch.no_grad():
                for k in range(a.rounds + 1):
                    for fused in (False, True):
                        if fused:
                            cogdl_b200.install(correct_smooth=True)
                        ms = event_times(lambda: postprocess(fused), 1, 0, flush=False)[0] / 1e3
                        cogdl_b200.uninstall_correct_smooth()
                        if k > 0:
                            pt[fused].append(ms)
            r["postprocess"] = {"unfused_ms": round(statistics.median(pt[False]), 1),
                                "fused_ms": round(statistics.median(pt[True]), 1),
                                "ratio": round(statistics.median(pt[True]) / statistics.median(pt[False]), 3),
                                "bit_identical": bool(torch.equal(outs[False].view(torch.int32),
                                                                  outs[True].view(torch.int32)))}
            del graph, outs
        res[name] = r
        del row, col, rp, labels
        torch.cuda.empty_cache()
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as fh:
            fh.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()

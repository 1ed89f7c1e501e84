#!/usr/bin/env python
"""Time Simple-HGN's layer (myGATConv of CogDL's examples/simple_hgn) fused against unfused, in one process.

Fused: cogdl_b200.hgn_attention (the attention stage of simple_hgn.cu + the multi-head SpMM).  Unfused: the example's
op sequence on this package's unfused operators, which is what the example runs after cogdl_b200.install():
h_l[row] + h_r[col] + h_e[type] -> leakyrelu -> edge_softmax -> dropout -> (1 - alpha) a + alpha res -> mh_spmm.  Both
share the layer's prologue (x @ W, the attention terms, the type table).  Shapes, synthetic and seeded:

  mag    N = 1,939,743, E = 2 x 21,111,007 + N (four relations, their reverses, self loops: T = 9), H = 8, F = 64,
         x [N, 128], dropout 0.5, alpha 0.05
  small  N = 20,000, E = 250,000, T = 5, otherwise the same

Reports per shape: layer forward, layer forward + backward, its peak allocated memory above the step's start and the
memory the forward keeps alive for the backward (`held`, output included; with and without res_attn), the typed
attention stage against the plain GAT attention stage (gat_fwd - mh_spmm at the same shape), and a 3-conv training
step at the model's defaults (heads 8 / 8 / 1, hidden 64).  Prints the card name and power limit, and one JSON line per
shape.  Usage: python tools/time_simple_hgn.py [--shapes mag,small] [--reps 5]
"""
import argparse
import json
import os
import sys

import torch
from gpu_timing import card, host_times, peak_above

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import cogdl_b200  # noqa: E402
from cogdl_b200.operators._raw import gat_fwd_raw, hgn_attn_raw, mhspmm_raw  # noqa: E402

SHAPES = {"mag": (1939743, 21111007, 4), "small": (20000, 125000, 2)}
SLOPE, P, ALPHA, F_IN, HID = 0.2, 0.5, 0.05, 128, 64


def make_graph(N, E_half, R, dev, seed=0):
    """R relations of E_half / R edges each, their reverses and a self loop per node; T = 2R + 1."""
    g = torch.Generator(device=dev).manual_seed(seed)
    row = torch.randint(0, N, (E_half,), device=dev, generator=g)
    col = torch.randint(0, N, (E_half,), device=dev, generator=g)
    rel = torch.randint(0, R, (E_half,), device=dev, generator=g)
    loops = torch.arange(N, device=dev)
    r = torch.cat([row, col, loops])
    c = torch.cat([col, row, loops])
    t = torch.cat([rel, rel + R, torch.full((N,), 2 * R, device=dev, dtype=rel.dtype)])
    graph = cogdl_b200.Graph(edge_index=(r, c), num_nodes=N)
    order = torch.sort(r, stable=True).indices
    graph.row_indptr
    return graph, t[order].contiguous(), 2 * R + 1


class Conv(torch.nn.Module):
    """The example layer's parameters; forward(fused) runs the fused or the unfused attention."""

    def __init__(self, T, f_in, f_out, nhead, residual, alpha, edge_feats=64):
        super().__init__()
        self.nhead, self.f_out, self.edge_feats, self.alpha = nhead, f_out, edge_feats, alpha
        self.W = torch.nn.Parameter(torch.randn(f_in, f_out * nhead) / f_in ** 0.5)
        self.W_e = torch.nn.Parameter(torch.randn(edge_feats, edge_feats * nhead) / edge_feats ** 0.5)
        self.edge_emb = torch.nn.Parameter(torch.randn(T, edge_feats) * 0.1)
        self.a_l, self.a_r, self.a_e = (torch.nn.Parameter(torch.randn(1, nhead, d) * 0.1)
                                        for d in (f_out, f_out, edge_feats))
        self.residual = torch.nn.Linear(f_in, f_out * nhead) if residual else None

    def forward(self, graph, etype, x, res_attn, fused, p=P):
        h = (x @ self.W).view(-1, self.nhead, self.f_out)
        e = (self.edge_emb @ self.W_e).view(-1, self.nhead, self.edge_feats)
        h_l, h_r, h_e = (self.a_l * h).sum(-1), (self.a_r * h).sum(-1), (self.a_e * e).sum(-1)
        if fused:
            out, att = cogdl_b200.hgn_attention(graph, h, h_l, h_r, h_e, etype, SLOPE, p, res_attn, self.alpha)
            out = out.view(out.shape[0], -1)
        else:
            row, col = graph.edge_index
            a = torch.nn.functional.leaky_relu(h_l[row] + h_r[col] + h_e[etype], SLOPE)
            a = torch.nn.functional.dropout(cogdl_b200.edge_softmax(graph, a), p)
            if res_attn is not None:
                a = a * (1 - self.alpha) + res_attn * self.alpha
            out, att = cogdl_b200.mh_spmm(graph, a, h), a
        if self.residual is not None:
            out = out + self.residual(x)
        return out, att.detach()


def median_s(fn, reps):
    """Median seconds of fn() over reps runs, each ended by a device synchronise, after one warm-up run."""
    return sorted(host_times(fn, reps, 1))[reps // 2] / 1e6


def run_shape(name, reps, dev):
    N, E_half, R = SHAPES[name]
    graph, etype, T = make_graph(N, E_half, R, dev)
    E = etype.numel()
    torch.manual_seed(1)
    x = torch.randn(N, F_IN, device=dev)
    conv = Conv(T, F_IN, HID, 8, False, ALPHA).to(dev)
    res = torch.rand(E, 8, device=dev) / 8
    g = torch.randn(N, 8 * HID, device=dev)
    res_row = {"shape": name, "N": N, "E": E, "T": T, "H": 8, "F": HID}

    def fwd(fused):
        with torch.no_grad():
            conv(graph, etype, x, res, fused)

    def fwd_bwd(fused):
        out, _ = conv(graph, etype, x, res.requires_grad_(False), fused)
        out.backward(g)
        conv.zero_grad(set_to_none=True)

    fwd_bwd(True)                              # build the cached structures (transpose, plan, type grouping) first
    fwd_bwd(False)
    for fused in (True, False):
        res_row[f"peak_gb_{'fused' if fused else 'unfused'}"] = round(peak_above(lambda: fwd_bwd(fused)) / 1e9, 3)
    res_row["peak_saved_gb"] = round(res_row["peak_gb_unfused"] - res_row["peak_gb_fused"], 3)
    for r, tag in ((res, ""), (None, "_nores")):   # what the forward keeps alive for the backward (output included)
        for fused in (True, False):
            torch.cuda.synchronize()
            start = torch.cuda.memory_allocated()
            out, _ = conv(graph, etype, x, r, fused)
            torch.cuda.synchronize()
            key = f"held_gb_{'fused' if fused else 'unfused'}{tag}"
            res_row[key] = round((torch.cuda.memory_allocated() - start) / 1e9, 3)
            out.backward(g)
            conv.zero_grad(set_to_none=True)
            del out
        res_row[f"held_saved_gb{tag}"] = round(res_row[f"held_gb_unfused{tag}"] - res_row[f"held_gb_fused{tag}"], 3)
    res_row["EH_tensor_gb"] = round(E * 8 * 4 / 1e9, 3)
    for what, fn in (("fwd", fwd), ("fwd_bwd", fwd_bwd)):
        t = {}
        for _ in range(2):                    # alternate fused and unfused
            for fused in (True, False):
                t.setdefault(fused, []).append(median_s(lambda: fn(fused), reps))
        res_row[f"{what}_ms_fused"] = round(1e3 * min(t[True]), 3)
        res_row[f"{what}_ms_unfused"] = round(1e3 * min(t[False]), 3)
        res_row[f"{what}_speedup"] = round(min(t[False]) / min(t[True]), 3)

    # attention stage: typed (no dropout, no blend, no saved attention) against the plain GAT stage
    st = graph.structure()
    with torch.no_grad():
        h = (x @ conv.W).view(-1, 8, HID)
        hl, hr = (conv.a_l * h).sum(-1), (conv.a_r * h).sum(-1)
        he = (conv.a_e * (conv.edge_emb @ conv.W_e).view(-1, 8, conv.edge_feats)).sum(-1)
        rs = cogdl_b200.structure.rgcn_structure_for(st, etype)
        att = torch.rand(E, 8, device=dev)
        t_typed = median_s(lambda: hgn_attn_raw(st, rs.type, hl, hr, he, SLOPE, False), reps)
        t_gat = median_s(lambda: gat_fwd_raw(st, hl, hr, h, SLOPE, False), reps)
        t_agg = median_s(lambda: mhspmm_raw(st, att, h), reps)
    res_row["typed_attention_ms"] = round(1e3 * t_typed, 3)
    res_row["gat_attention_ms"] = round(1e3 * (t_gat - t_agg), 3)
    res_row["typed_over_gat"] = round(t_typed / max(t_gat - t_agg, 1e-9), 3)

    # 3-conv training step at the model's defaults
    convs = torch.nn.ModuleList([Conv(T, F_IN, HID, 8, False, ALPHA), Conv(T, 8 * HID, HID, 8, True, ALPHA),
                                 Conv(T, 8 * HID, 4, 1, True, ALPHA)]).to(dev)
    labels = torch.randint(0, 4, (N,), device=dev)

    def step(fused):
        o, a = convs[0](graph, etype, x, None, fused)
        o, a = convs[1](graph, etype, torch.nn.functional.elu(o), a, fused)
        o, _ = convs[2](graph, etype, torch.nn.functional.elu(o), None, fused)
        torch.nn.functional.cross_entropy(o, labels).backward()
        convs.zero_grad(set_to_none=True)

    t = {}
    for _ in range(2):
        for fused in (True, False):
            t.setdefault(fused, []).append(median_s(lambda: step(fused), reps))
    res_row["step_ms_fused"] = round(1e3 * min(t[True]), 3)
    res_row["step_ms_unfused"] = round(1e3 * min(t[False]), 3)
    res_row["step_speedup"] = round(min(t[False]) / min(t[True]), 3)
    return res_row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--shapes", default="mag,small")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_simple_hgn: needs a GPU")
    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = False
    print("card:", card())
    for name in args.shapes.split(","):
        print(json.dumps(run_shape(name, args.reps, dev)), flush=True)
    print("card:", card())


if __name__ == "__main__":
    main()

"""Time the initial-residual propagation of GCNII and APPNP on the GPU, fused (cogdl_b200.spmm_residual) against
unfused (cogdl_b200.spmm followed by torch's elementwise ops), on the arxiv shape (169 343 nodes, 1.17 M edges,
sym-normalised weights):

- a GCNII 16 x 256 training step (the restatement of CogDL's GCNII used by tools/time_actnn.py), unfused as the
  reference's GCNIILayer computes it, fused as install(gcnii=True) computes it: one spmm_residual and one addmm with
  beta * W + (1 - beta) * I per layer;
- an APPNP training step, K = 10 propagations at C = 40 classes after a 128 -> 64 -> 40 MLP, edge-weight dropout 0.5;
- the operator alone, forward, against the plain SpMM at F = 40, 128 and 256, on the raw entry points (the cached
  structure, no graph handling): with Z, without Z (the scaling only), with the row scale only, and with both.  Each
  window times 50 back-to-back launches, so the host's launch path overlaps the kernels and the per-launch time is
  the device's.  The epilogue's cost is the difference to the plain SpMM; reading Z once at HBM speed is given as
  arithmetic for comparison.

Fused and unfused runs alternate for --rounds rounds in one process; each figure is the median over rounds of the
per-round median (CUDA events).  The card's name and power limit are read in the same run.  Prints one JSON line and
writes it to --out if given.
"""
import argparse
import json
import math
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F
from gpu_timing import alternate, card

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BYTES_PER_S = 3.35e12      # H100 SXM data sheet


class GCNII(nn.Module):
    """CogDL's GCNII forward (gcnii.py:111-125) with GCNIILayer (gcnii_layer.py:24-30), alpha 0.1, lambda 0.5."""

    def __init__(self, fin, hid, out, layers, dropout, fused):
        super().__init__()
        self.fused = fused
        self.fc = nn.ModuleList([nn.Linear(fin, hid), nn.Linear(hid, out)])
        self.convs = nn.ModuleList(nn.Linear(hid, hid) for _ in range(layers))
        self.betas = [math.log(0.5 / (i + 1) + 1) for i in range(layers)]
        self.dropout = nn.Dropout(dropout)
        self.relu = nn.ReLU(inplace=True)

    def forward(self, g, x):
        import cogdl_b200

        h0 = self.relu(self.fc[0](self.dropout(x)))
        h = h0
        for lin, beta in zip(self.convs, self.betas):
            h = self.dropout(h)
            if self.fused:
                s = cogdl_b200.spmm_residual(g, h, h0, 1 - 0.1, 0.1)
                eye = torch.eye(lin.weight.shape[0], device=s.device)
                h = self.relu(torch.addmm(beta * lin.bias, s, (beta * lin.weight + (1 - beta) * eye).t()))
            else:
                hid = cogdl_b200.spmm(g, h)
                hid = (1 - 0.1) * hid + 0.1 * h0
                h = self.relu(beta * lin(hid) + (1 - beta) * hid)
        return self.fc[1](self.dropout(h))


class APPNP(nn.Module):
    """CogDL's PPNP forward (ppnp.py:56-87), propagation "appnp", on a graph with sym-normalised edge weights."""

    def __init__(self, fin, hid, out, dropout, alpha, niter, fused):
        super().__init__()
        self.mlp = nn.Sequential(nn.Dropout(dropout), nn.Linear(fin, hid), nn.ReLU(), nn.Dropout(dropout),
                                 nn.Linear(hid, out))
        self.dropout, self.alpha, self.niter, self.fused = dropout, alpha, niter, fused

    def forward(self, g, x):
        import cogdl_b200

        local = self.mlp(F.dropout(x, p=self.dropout, training=self.training))
        preds = local
        with g.local_graph():
            g.edge_weight = F.dropout(g.edge_weight, p=self.dropout, training=self.training)
            g.set_symmetric()
            for _ in range(self.niter):
                if self.fused:
                    preds = cogdl_b200.spmm_residual(g, preds, local, 1 - self.alpha, self.alpha)
                else:
                    preds = (1 - self.alpha) * cogdl_b200.spmm(g, preds) + self.alpha * local
        return preds


def burst(fn, n=50):
    """fn run n times back to back: one event window times all n launches."""
    def run():
        for _ in range(n):
            fn()
    return run


def train_step(model, g, x, y):
    def step():
        model.zero_grad(set_to_none=True)
        F.cross_entropy(model(g, x), y).backward()
    return step


def round_medians(fns, warmup, reps, rounds):
    """{name: median over rounds of the per-round median ms}, {name: per-round medians}; the names take turns within
    each round.  The median of an even count is its upper middle value."""
    upper_median = lambda v: sorted(v)[len(v) // 2]  # noqa: E731
    per = {k: [upper_median(ts[i:i + reps]) / 1e3 for i in range(0, len(ts), reps)]
           for k, (ts, _) in alternate(fns, rounds, reps, warmup, flush=False).items()}
    return {k: round(upper_median(v), 3) for k, v in per.items()}, {k: [round(t, 3) for t in v] for k, v in per.items()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--out")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_gcnii needs a GPU"
    import cogdl_b200
    from cogdl_b200 import synth

    torch.backends.cuda.matmul.allow_tf32 = False
    n, e = 169343, 1166243
    rp, col = synth.powerlaw_csr(n, e, seed=1)
    w = synth.sym_norm_weights(rp, col)
    g = cogdl_b200.Graph(row_ptr=rp, col=col, edge_weight=w, num_nodes=n).to("cuda")
    gen = torch.Generator().manual_seed(1)
    x = torch.randn(n, 128, generator=gen).cuda()
    y = torch.randint(0, 40, (n,), generator=gen).cuda()
    res = {"card": card()}

    models = {}
    for fused in (False, True):
        torch.manual_seed(0)
        models[fused] = GCNII(128, 256, 40, 16, 0.5, fused).cuda().train()
    models[True].load_state_dict(models[False].state_dict())
    med, raw = round_medians({"unfused": train_step(models[False], g, x, y), "fused": train_step(models[True], g, x, y)},
                         a.warmup, a.reps, a.rounds)
    res["gcnii_16x256_step_ms"] = med
    res["gcnii_ratio"] = round(med["fused"] / med["unfused"], 3)
    res["gcnii_rounds"] = raw
    with torch.no_grad():
        torch.manual_seed(5)
        models[False].eval(), models[True].eval()
        o0, o1 = models[False](g, x), models[True](g, x)
        res["gcnii_eval_logits_rel_diff"] = float((o0 - o1).abs().max() / o0.abs().max())
    del models
    torch.cuda.empty_cache()

    models = {}
    for fused in (False, True):
        torch.manual_seed(0)
        models[fused] = APPNP(128, 64, 40, 0.5, 0.1, 10, fused).cuda().train()
    models[True].load_state_dict(models[False].state_dict())
    med, raw = round_medians({"unfused": train_step(models[False], g, x, y), "fused": train_step(models[True], g, x, y)},
                         a.warmup, a.reps, a.rounds)
    res["appnp_k10_c40_step_ms"] = med
    res["appnp_ratio"] = round(med["fused"] / med["unfused"], 3)
    res["appnp_rounds"] = raw
    torch.manual_seed(9)
    with torch.no_grad():
        o0 = models[False](g, x)
        torch.manual_seed(9)
        o1 = models[True](g, x)
    res["appnp_seeded_train_forward_rel_diff"] = float((o0 - o1).abs().max() / o0.abs().max())
    del models
    torch.cuda.empty_cache()

    from cogdl_b200.operators._raw import spmm_raw, spmm_residual_raw

    st, val = g.structure(), g.raw_edge_weight
    r = torch.rand(n, device="cuda") + 0.5
    ops = {}
    B = 50
    for Fw in (40, 128, 256):
        h = torch.randn(n, Fw, device="cuda")
        z = torch.randn(n, Fw, device="cuda")
        fns = {"spmm": lambda: spmm_raw(st, val, h),
               "residual_z": lambda: spmm_residual_raw(st, val, h, z, 0.9, 0.1),
               "residual_no_z": lambda: spmm_residual_raw(st, val, h, None, 0.9, 0.1),
               "residual_row_scale_only": lambda: spmm_residual_raw(st, val, h, None, 1.0, 0.0, r),
               "residual_z_row_scale": lambda: spmm_residual_raw(st, val, h, z, 0.9, 0.1, r),
               "unfused_z": lambda: 0.9 * spmm_raw(st, val, h) + 0.1 * z}
        med, _ = round_medians({k: burst(f, B) for k, f in fns.items()}, 1, a.reps, a.rounds)
        med = {k + "_us": round(v / B * 1e3, 1) for k, v in med.items()}
        med["read_z_once_us_arithmetic"] = round(n * Fw * 4 / HBM_BYTES_PER_S * 1e6, 1)
        for k in ("residual_z", "residual_no_z", "residual_row_scale_only", "residual_z_row_scale"):
            med[f"epilogue_{k}_us"] = round(med[k + "_us"] - med["spmm_us"], 1)
        ops[f"F{Fw}"] = med
        del h, z
    res["operator"] = ops
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()

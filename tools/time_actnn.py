"""Time activation-compressed training (cogdl_b200.actnn) on the GPU: a GCNII 16 x 256 training step at the arxiv
shape (169 343 nodes, 1.17 M edges, 128 features) compressed at 2 bits against the uncompressed step, the per-row bit
allocation on the device against the reference's host greedy (restated by calc_precision_host, which includes the
copy of C to the host), and one compressed step at the products shape (2 449 029 nodes, 61.9 M edges, 100 features).
The uncompressed products step is not run: its saved activations are given as arithmetic.

The models are cogdl_b200's own restatement of CogDL's GCNII (cogdl/models/nn/gcnii.py) on cogdl_b200.spmm, so no
reference checkout is needed.  config.perlayer is off: allocate_perlayer's per-row branch runs on the host.  Reports
median step time (CUDA events), peak memory, and the card's name and power limit read in the same run; prints one
JSON line and writes it to --out if given.
"""
import argparse
import json
import math
import os
import sys

import torch
import torch.nn as nn
import torch.nn.functional as F
from gpu_timing import card, event_times

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


class GCNII(nn.Module):
    """CogDL's GCNII forward (gcnii.py:111-125) with its GCNIILayer / ActGCNIILayer (sym-normalised graph)."""

    def __init__(self, fin, hid, out, layers, dropout, act):
        super().__init__()
        from cogdl_b200.actnn.layers import QDropout, QLinear, QReLU

        Linear = QLinear if act else nn.Linear
        self.act = act
        self.fc = nn.ModuleList([Linear(fin, hid), Linear(hid, out)])
        self.convs = nn.ModuleList(Linear(hid, hid) for _ in range(layers))
        self.betas = [math.log(0.5 / (i + 1) + 1) for i in range(layers)]
        self.dropout = QDropout(dropout) if act else nn.Dropout(dropout)
        self.relu = QReLU() if act else nn.ReLU(inplace=True)

    def forward(self, g, x):
        import cogdl_b200

        h0 = self.relu(self.fc[0](self.dropout(x)))
        h = h0
        for lin, beta in zip(self.convs, self.betas):
            h = self.dropout(h)
            hid = cogdl_b200.spmm(g, h, actnn=self.act)
            hid = 0.9 * hid + 0.1 * h0
            h = self.relu(beta * lin(hid) + (1 - beta) * hid)
        return self.fc[1](self.dropout(h))


def step_time(model, g, x, y, warmup, reps):
    def step():
        model.zero_grad(set_to_none=True)
        F.cross_entropy(model(g, x), y).backward()

    for _ in range(warmup):
        step()
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times = sorted(event_times(step, reps, 0, flush=False))
    return times[len(times) // 2] / 1e3, torch.cuda.max_memory_allocated() / 2 ** 30


def graph(n, e, f, seed):
    import cogdl_b200
    from cogdl_b200 import synth

    rp, col = synth.powerlaw_csr(n, e, seed=seed)
    w = synth.sym_norm_weights(rp, col)
    g = cogdl_b200.Graph(row_ptr=rp, col=col, edge_weight=w, num_nodes=n).to("cuda")
    gen = torch.Generator().manual_seed(seed)
    return g, torch.randn(n, f, generator=gen).cuda(), torch.randint(0, 40, (n,), generator=gen).cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--skip-products", action="store_true")
    ap.add_argument("--out")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "time_actnn needs a GPU"
    from cogdl_b200.actnn import config, kernels
    from cogdl_b200.actnn.qscheme import calc_precision_host

    config.perlayer = False
    res = {"card": card()}
    g, x, y = graph(169343, 1166243, 128, 1)
    for tag, act in (("arxiv_fp32", False), ("arxiv_actnn2", True)):
        torch.manual_seed(0)
        m = GCNII(128, 256, 40, 16, 0.5, act).cuda().train()
        t, peak = step_time(m, g, x, y, a.warmup, a.reps)
        res[tag] = {"step_ms": round(t, 2), "peak_gib": round(peak, 3)}
        del m
        torch.cuda.empty_cache()

    C = torch.rand(169343, device="cuda") * 100
    target = 2 * C.numel()
    dev_bits = kernels.allocate_bits(C, target)
    for _ in range(3):
        kernels.allocate_bits(C, target)
    torch.cuda.synchronize()

    def twenty():     # each result is dropped before the next call, so its block is reused
        for _ in range(20):
            kernels.allocate_bits(C, target)
    res["alloc_device_ms"] = round(event_times(twenty, 1, 0, flush=False)[0] / 1e3 / 20, 3)
    import time

    t0 = time.perf_counter()
    host_bits = calc_precision_host(torch.full((C.numel(),), 8, dtype=torch.int32), C.cpu(),
                                    torch.ones(C.numel(), dtype=torch.int32), target)
    res["alloc_host_ms"] = round((time.perf_counter() - t0) * 1e3, 1)
    res["alloc_equal"] = bool(torch.equal(host_bits, dev_bits.cpu()))

    if not a.skip_products:
        del g, x, y
        torch.cuda.empty_cache()
        n = 2449029
        g, x, y = graph(n, 61859140 * 2, 100, 2)
        torch.manual_seed(0)
        m = GCNII(100, 256, 40, 16, 0.5, True).cuda().train()
        t, peak = step_time(m, g, x, y, 1, 3)
        res["products_actnn2"] = {"step_ms": round(t, 1), "peak_gib": round(peak, 2)}
        # uncompressed saved activations per GCNII layer: the linear input and the ReLU output (fp32) and the
        # dropout mask (1 byte per element)
        res["products_fp32_saved_gib_arithmetic"] = round(16 * n * 256 * (4 + 4 + 1) / 2 ** 30, 1)
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(json.dumps(res) + "\n")


if __name__ == "__main__":
    main()

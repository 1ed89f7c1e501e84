"""Child process of tests/test_gpu_readout.py: the UNMODIFIED reference pooling functions, GIN model, InfoGraph encoder,
SortPool and Set2Set through cogdl_b200.install(gin=True, readout=True), on the batch of tests/golden/readout.npz.  Runs
in its own process because install() rebinds the reference's functions for the rest of the process.  Prints one JSON
line.

Checked: every output within 1e-5 of the reference's CPU results (relative to the largest magnitude of the model's
outputs: the GIN biases ahead of a BatchNorm have gradients at the noise level of any summation order) and of the same
models under install(gin=True) alone (the reference's scatter_add_ pooling); two runs bit-identical; Set2Set, which the
reference cannot run, within 1e-5 of an fp64 torch run of the same LSTM with the softmax the layer documents;
install() without the flag leaves the originals alone, uninstall_readout() restores them, and CPU inputs go to them.
"""
import copy
import json

import numpy as np
import torch

from tests.golden.make_golden_readout import build_gin, build_infograph_encoder, build_sortpool, make_graph
from tests.refpkg import import_reference
from tests.test_cpu_readout_golden import GOLDEN

MODELS = {"gin": lambda k: k.startswith("gin_"), "ig": lambda k: k.startswith("ig_"), "sp": lambda k: k == "sp_logits",
          "sum": lambda k: k == "sum_x2", "mean": lambda k: k == "mean_x2"}


def run_all(Graph, d, dev):
    import cogdl.utils as cu

    out = {}
    x2, batch = torch.from_numpy(d["x2"]).to(dev), torch.from_numpy(d["batch"]).to(dev)
    out["sum_x2"] = cu.batch_sum_pooling(x2, batch)
    out["mean_x2"] = cu.batch_mean_pooling(x2, batch)
    gin = build_gin().to(dev)
    logits = gin(make_graph(Graph, d, dev))
    logits.backward(torch.from_numpy(d["g_logits"]).to(dev))
    out["gin_logits"] = logits.detach()
    out.update({f"gin_grad_{n}": p.grad for n, p in gin.named_parameters() if p.grad is not None})
    enc = build_infograph_encoder().to(dev)
    g = make_graph(Graph, d, dev)
    with torch.no_grad():
        out["ig_graph_rep"] = enc(g, g.x)[0]
        out["sp_logits"] = build_sortpool().to(dev).eval()(make_graph(Graph, d, dev))
    return out


def set2set_fp64(module, x, batch, B):
    m = copy.deepcopy(module).double().cpu()
    x, batch = x.double().cpu(), batch.cpu()
    h = (torch.zeros(m.num_layers, B, m.in_channels, dtype=torch.float64),) * 2
    q_star = torch.zeros(B, m.out_channels, dtype=torch.float64)
    for _ in range(m.processing_steps):
        q, h = m.lstm(q_star.unsqueeze(0), h)
        q = q.view(B, m.in_channels)
        e = (x * q[batch]).sum(-1)
        mx = torch.full((B,), -torch.inf, dtype=torch.float64).scatter_reduce(0, batch, e, "amax")
        w = torch.exp(e - mx[batch])
        a = w / torch.zeros(B, dtype=torch.float64).index_add(0, batch, w)[batch]
        q_star = torch.cat([q, torch.zeros(B, x.shape[1], dtype=torch.float64).index_add(0, batch, a[:, None] * x)], -1)
    return q_star


def scaled(a, b, keys):
    scale = max(float(b[k].abs().max()) for k in keys)
    return {k: float((a[k].double().cpu() - b[k].double().cpu()).abs().max()) / scale for k in keys}


def main():
    import_reference()
    import cogdl.layers.set2set as s2s
    import cogdl.models.nn.gin as gm
    import cogdl.models.nn.sortpool as spm
    import cogdl.utils as cu
    import cogdl_b200
    from cogdl.data import Graph

    dev = torch.device("cuda:0")
    torch.backends.cuda.matmul.allow_tf32 = torch.backends.cudnn.allow_tf32 = False   # fp32 GEMMs and conv1d
    d = np.load(GOLDEN)
    res = {}
    originals = (cu.batch_sum_pooling, gm.GIN.forward, spm.SortPool.forward, s2s.Set2Set.forward)
    cogdl_b200.install(gin=True)
    res["untouched_without_flag"] = (cu.batch_sum_pooling, gm.GIN.forward, spm.SortPool.forward,
                                     s2s.Set2Set.forward) == originals
    base = run_all(Graph, d, dev)
    res["patched"] = cogdl_b200.install(gin=True, readout=True)
    res["rebound"] = (all(getattr(f, "_cogdl_b200", False) for f in (gm.GIN.forward, spm.SortPool.forward,
                                                                      s2s.Set2Set.forward, cu.batch_sum_pooling,
                                                                      cu.batch_mean_pooling, cu.batch_max_pooling))
                      and s2s.batch_sum_pooling is cu.batch_sum_pooling)
    fused = run_all(Graph, d, dev)
    again = run_all(Graph, d, dev)
    res["bit_identical"] = {k: bool(torch.equal(fused[k].view(torch.int32), again[k].view(torch.int32))) for k in fused}
    res["vs_golden"], res["vs_gin_only"] = {}, {}
    gold = {k: torch.from_numpy(d[k]) for k in fused}
    for keys in ([k for k in fused if f(k)] for f in MODELS.values()):
        res["vs_golden"].update(scaled(fused, gold, keys))
        res["vs_gin_only"].update(scaled(fused, base, keys))
    torch.manual_seed(31)
    s2s_layer = s2s.Set2Set(8, 3).to(dev)
    x, batch = torch.from_numpy(d["x"]).to(dev), torch.from_numpy(d["batch"]).to(dev)
    got = s2s_layer(x, batch)
    want = set2set_fp64(s2s_layer, x, batch, int(d["batch"].max()) + 1)
    res["set2set_rel"] = float((got.double().cpu() - want).abs().max() / want.abs().max())

    calls = []
    orig = gm.GIN._cogdl_b200_original_forward

    def counting(*a, **k):
        calls.append("GIN.forward")
        return orig(*a, **k)
    gm.GIN._cogdl_b200_original_forward = counting
    fb = {}
    x2c, bc = torch.from_numpy(d["x2"]), torch.from_numpy(d["batch"])
    fb["pool_cpu"] = bool(np.allclose(cu.batch_sum_pooling(x2c, bc).numpy(), d["sum_x2"], rtol=1e-6, atol=1e-6))
    try:
        build_gin()(make_graph(Graph, d))       # the original's GIN layers (rebound by gin=True) refuse CPU tensors
    except RuntimeError as e:
        assert "CPU tensors are not supported" in str(e), e
    fb["gin_cpu"] = calls == ["GIN.forward"]
    gm.GIN._cogdl_b200_original_forward = orig
    res["fallbacks"] = fb

    cogdl_b200.uninstall_readout()
    res["restored"] = ((cu.batch_sum_pooling, gm.GIN.forward, spm.SortPool.forward, s2s.Set2Set.forward) == originals
                       and s2s.batch_sum_pooling is originals[0])
    print(json.dumps(res))


if __name__ == "__main__":
    main()

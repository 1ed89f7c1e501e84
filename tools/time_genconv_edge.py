"""GENConv with a linear edge encoder: the fused edge-encoder kernels against encoder GEMM + edge-term kernels (CUDA
events, L2 flushed, median of 20, two rounds with the variants alternating inside each).

  (a) ogbn-proteins shape (N = 132,534, E = 79,122,504, D = 8; a synthetic power-law graph built here), aggregation
      only, F = 64 and 128: the fused forward and forward + backward against `edge_attr @ W.T` plus the edge-term
      kernels, with spmm_raw at the same F as the yardstick.  A variant whose [E, F] tensors cannot fit on the card
      is not run; its computed size is printed.  Peak memory per variant, the byte model and its share of 3.35 TB/s,
      and the encoder FLOPs (2 E F D) against the FP32 rate (67 TFLOP/s) are printed beside the times.
  (b) a full-graph training step of the reference DeeperGCN at its defaults (14 layers, hidden 128, softmax_sg,
      edge_attr_size=[8]) on the proteins shape under install(genconv=True): time and max_memory_allocated
      (needs oracle/_ref/pkg).  The original forward would save one [E, 128] edge term per GENConv layer; only
      that size is printed.
  (c) the arxiv shape with D = 8, F = 128, fused against the existing path (the low-degree regime).
Writes time_genconv_edge.json to OUT_DIR with the card name and power limit read in the same run.

    python tools/time_genconv_edge.py OUT_DIR
"""
import json
import os
import statistics
import sys

import torch
from gpu_timing import event_times, peak_above, write_result

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import cogdl_b200  # noqa: E402
from cogdl_b200 import synth  # noqa: E402
from cogdl_b200.operators._raw import spmm_raw  # noqa: E402

if len(sys.argv) != 2:
    sys.exit(__doc__)
out_dir = sys.argv[1]
torch.backends.cuda.matmul.allow_tf32 = False
torch.backends.cudnn.allow_tf32 = False
PEAK_BW, PEAK_FP32 = 3.35e12, 67e12
PROTEINS = (132_534, 79_122_504)
D = 8

dev = torch.device("cuda")
HBM = torch.cuda.get_device_properties(dev).total_memory


def byte_model(E, N, F, fused, bwd=False):
    """Algorithmic bytes: fp32 values, int32 indices.  Forward: colind, x gather, the edge data (D features fused;
    the GEMM's read of the features and write of [E, F], then the kernel's read of it otherwise), out, lse2.
    Backward: rowind, perm, three gathered rows (lse2, g, out), the edge data (features fused; the edge term read
    and its gradient written, then the GEMM's read of the gradient and the features for dW otherwise), x and dx per
    column.  Gathered rows are counted in full, though part of them hits in the L2."""
    if not bwd:
        edge = 4 * D if fused else 4 * D + 2 * 4 * F
        return E * (4 + 4 * F + edge) + N * (4 + 8 * F)
    edge = 4 * D if fused else 3 * 4 * F + 4 * D
    return E * (8 + 12 * F + edge) + N * (4 + 8 * F)


def structures(n, e, self_loops):
    rp, col = synth.powerlaw_csr(n, e, seed=0, device=dev, self_loops=self_loops)
    st = cogdl_b200.CSRStructure.from_int64(rp, col)
    del rp, col
    st.plan, st.csc()[0].plan
    return st


def aggregation_variants(st, F, run_existing_bwd):
    g = torch.Generator(device=dev).manual_seed(F)
    x = torch.randn(st.n_cols, F, device=dev, generator=g)
    attr = torch.rand(st.nnz, D, device=dev, generator=g)
    w = torch.randn(F, D, device=dev, generator=g) / D ** 0.5
    r = torch.randn(st.n_rows, F, device=dev, generator=g)
    beta = torch.nn.Parameter(torch.ones(1, device=dev))
    xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)

    def fused(xx, ww):
        return cogdl_b200.genconv_aggregate(st, xx, "softmax_sg", beta=beta, edge_attr=attr, edge_weight=ww)

    def existing(xx, ww):
        return cogdl_b200.genconv_aggregate(st, xx, "softmax_sg", beta=beta, edge_term=attr @ ww.T)

    def fwd(fn):
        def call():
            with torch.no_grad():
                fn(x, w)
        return call

    def fwd_bwd(fn):
        def call():
            xg.grad = wg.grad = beta.grad = None
            fn(xg, wg).backward(r)
        return call

    with torch.no_grad():
        a, b = fused(x, w), existing(x, w)
    parity = float(((a - b).abs() / b.abs().amax(1, keepdim=True).clamp_min(1e-30)).max())
    del a, b
    v = {"spmm_raw_us": lambda: spmm_raw(st, None, x), "fused_fwd_us": fwd(fused), "existing_fwd_us": fwd(existing),
         "fused_fwd_bwd_us": fwd_bwd(fused)}
    if run_existing_bwd:
        v["existing_fwd_bwd_us"] = fwd_bwd(existing)
    return v, parity


def run_rounds(variants):
    rounds = []
    for rnd in range(2):
        rr = {k: statistics.median(event_times(fn, 20, 3, flush=True)) for k, fn in variants.items()}
        rounds.append(rr)
        for k, t in rr.items():
            print(f"round {rnd} {k:28s} {t:12.1f}")
    return rounds, {k: statistics.median(rd[k] for rd in rounds) for k in rounds[0]}


def report(st, F, variants, rounds, med, parity, skipped):
    E, N = st.nnz, st.n_rows
    peaks = {k.replace("_us", "_peak_bytes"): peak_above(fn) for k, fn in variants.items()}
    bm = {"fused_fwd": byte_model(E, N, F, True), "existing_fwd": byte_model(E, N, F, False),
          "fused_bwd": byte_model(E, N, F, True, bwd=True), "existing_bwd": byte_model(E, N, F, False, bwd=True)}
    flops = 2 * E * F * D
    s = {"fused_fwd_speedup": med["existing_fwd_us"] / med["fused_fwd_us"],
         "fused_fwd_over_spmm": med["fused_fwd_us"] / med["spmm_raw_us"],
         "fused_fwd_hbm_fraction": bm["fused_fwd"] / (med["fused_fwd_us"] * 1e-6) / PEAK_BW,
         "fused_fwd_fp32_fraction": flops / (med["fused_fwd_us"] * 1e-6) / PEAK_FP32,
         "fused_fwd_bound": "bytes" if bm["fused_fwd"] / PEAK_BW > flops / PEAK_FP32 else "fp32 FLOPs"}
    if "existing_fwd_bwd_us" in med:
        s["fused_fwd_bwd_speedup"] = med["existing_fwd_bwd_us"] / med["fused_fwd_bwd_us"]
    return {"n": N, "nnz": E, "F": F, "D": D, "fused_vs_existing_fwd_max_row_rel_err": parity, "rounds": rounds,
            "median": med, "peak_bytes": peaks, "bytes": bm, "encoder_flops": flops, "summary": s,
            "not_run": skipped}


res = {"hbm_bytes": HBM}

# ---------------------------------------------------------------------------------------------- (a)
st = structures(*PROTEINS, self_loops=False)
res["proteins"] = {}
for F in (64, 128):
    edge_tensor = st.nnz * F * 4
    # the existing forward + backward holds the edge term and its gradient at once
    fits_bwd = 2 * edge_tensor + st.nnz * (D + 6) * 4 < 0.9 * HBM
    skipped = {} if fits_bwd else {"existing_fwd_bwd": {"edge_term_bytes": edge_tensor,
                                                        "d_edge_term_bytes": edge_tensor}}
    if skipped:
        print(f"F={F}: the existing forward + backward needs two [E, F] tensors of {edge_tensor / 1e9:.1f} GB: not run")
    variants, parity = aggregation_variants(st, F, fits_bwd)
    rounds, med = run_rounds(variants)
    res["proteins"][F] = report(st, F, variants, rounds, med, parity, skipped)
    print(json.dumps({"F": F, **res["proteins"][F]["summary"], "peak_bytes": res["proteins"][F]["peak_bytes"]}))
    del variants
    torch.cuda.empty_cache()

# ---------------------------------------------------------------------------------------------- (b)
try:
    from tests.refpkg import import_reference

    import_reference()
    from cogdl.data import Graph
    from cogdl.models.nn.deepergcn import DeeperGCN

    cogdl_b200.install(genconv=True)
    n = st.n_rows
    rows = torch.repeat_interleave(torch.arange(n, device=dev, dtype=torch.int64),
                                   (st.rowptr[1:] - st.rowptr[:-1]).long())
    graph = Graph(x=torch.randn(n, 8, device=dev), edge_index=(rows, st.colind.long()))
    del rows
    graph.row_indptr
    graph.edge_attr = torch.rand(st.nnz, D, device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    torch.manual_seed(0)
    model = DeeperGCN(8, 128, 112, 14, aggr="softmax_sg", edge_attr_size=[D]).to(dev).train()
    y = (torch.rand(n, 112, device=dev) < 0.5).float()
    opt = torch.optim.SGD(model.parameters(), lr=0.01)

    def step():
        opt.zero_grad(set_to_none=True)
        torch.nn.functional.binary_cross_entropy_with_logits(model(graph), y).backward()
        opt.step()

    step_peak_above = peak_above(step)
    peak = torch.cuda.max_memory_allocated()
    times = [statistics.median(event_times(step, 10, 3, flush=True)) / 1e3 for _ in range(2)]
    res["deepergcn_step"] = {"layers": 14, "hidden": 128, "step_ms_rounds": times, "step_ms": statistics.median(times),
                             "max_memory_allocated": peak, "peak_above_inputs": step_peak_above, "kernel_after_step":
                             cogdl_b200._cabi.last_kernel(),
                             "original_saved_edge_terms_bytes": 13 * st.nnz * 128 * 4}
    print(json.dumps(res["deepergcn_step"]))
    del model, graph, opt, y
except ImportError as ex:
    print(f"(b) skipped: {ex}")
del st
torch.cuda.empty_cache()

# ---------------------------------------------------------------------------------------------- (c)
st = structures(*synth.SHAPES["arxiv"], self_loops=True)
variants, parity = aggregation_variants(st, 128, True)
rounds, med = run_rounds(variants)
res["arxiv"] = report(st, 128, variants, rounds, med, parity, {})
print(json.dumps({"arxiv": res["arxiv"]["summary"]}))
write_result(out_dir, "time_genconv_edge", res)

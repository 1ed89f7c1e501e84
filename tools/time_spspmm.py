"""Time cogdl_b200.spspmm (sm_90a SpGEMM) against torch.sparse.mm on CUDA (cuSPARSE through torch) for the products
CogDL's GTN and SRGCN make, and a reference GTN training step through install(spspmm=True).

Workloads: A.A on the arxiv-shaped synthetic graph; the GTN shape (4 relations, 9 000 nodes, 9 000 edges each: the
product of two mixtures, forward and forward + backward); the SRGCN nhop = 2 square of (A + I) at the Cora and PubMed
shapes.  Reports time (CUDA events, median of --reps after --warmup), peak memory, nnz(C) and products per second, with
the card's name and power limit read in the same run.  Prints one JSON line and writes it to --out if given.
"""
import argparse
import json
import os
import sys

import torch
from gpu_timing import card, event_times, peak_above

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def median_ms_peak(fn, warmup, reps):
    """Median ms (upper middle value of an even count) and peak GiB above the start over `reps` calls."""
    for _ in range(warmup):
        fn()
    times = []
    peak = peak_above(lambda: times.extend(event_times(fn, reps, 0, flush=False)))
    times.sort()
    return times[len(times) // 2] / 1e3, peak / 2**30


def products(index, n_rows, index_b):
    degb = torch.bincount(index_b[0], minlength=n_rows)
    return int(degb[index[1]].sum())


def compare(name, ia, va, ib, vb, m, k, n, warmup, reps, backward=False):
    import cogdl_b200

    dev = va.device
    A = torch.sparse_coo_tensor(ia, va, (m, k)).coalesce()
    B = torch.sparse_coo_tensor(ib, vb, (k, n)).coalesce()
    Ac, Bc = A.to_sparse_csr(), B.to_sparse_csr()

    def ours():
        if backward:
            a, b = va.detach().requires_grad_(True), vb.detach().requires_grad_(True)
            _, v = cogdl_b200.spspmm(ia, a, ib, b, m, k, n)
            v.sum().backward()
        else:
            cogdl_b200.spspmm(ia, va, ib, vb, m, k, n)

    # both sides start from structures built outside the timed window: spspmm from its cached CooStructure, torch
    # from prebuilt coalesced leaf tensors
    A_leaf, B_leaf = A.detach().requires_grad_(True), B.detach().requires_grad_(True)

    def torch_mm():
        if backward:
            torch.sparse.mm(A_leaf, B_leaf).coalesce().values().sum().backward()
        else:
            torch.sparse.mm(Ac, Bc)

    idx, _ = cogdl_b200.spspmm(ia, va, ib, vb, m, k, n)
    nnz = idx.shape[1]
    prods = products(A.indices(), k, B.indices())
    t_ours, mem_ours = median_ms_peak(ours, warmup, reps)
    try:
        t_ref, mem_ref = median_ms_peak(torch_mm, warmup, reps)
    except RuntimeError as e:            # torch's sparse backward may not cover a case: report it, do not hide it
        t_ref, mem_ref = None, str(e).splitlines()[0]
    return {"workload": name, "m": m, "k": k, "n": n, "nnz_a": int(A._nnz()), "nnz_b": int(B._nnz()), "nnz_c": nnz,
            "products": prods, "ms": round(t_ours, 4), "peak_gb": round(mem_ours, 4),
            "gproducts_per_s": round(prods / t_ours / 1e6, 3),
            "torch_sparse_mm_ms": None if t_ref is None else round(t_ref, 4),
            "torch_sparse_mm_peak_gb": mem_ref if isinstance(mem_ref, str) else round(mem_ref, 4),
            "speedup": None if t_ref is None else round(t_ref / t_ours, 3)}


def kernel_split(ia, va, n, warmup):
    """CUDA time per kernel name of one arxiv-shaped spspmm forward (torch.profiler, a run of its own)."""
    import cogdl_b200
    from torch.profiler import ProfilerActivity, profile

    for _ in range(warmup):
        cogdl_b200.spspmm(ia, va, ia, va, n, n, n)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        cogdl_b200.spspmm(ia, va, ia, va, n, n, n)
        torch.cuda.synchronize()
    rows = {}
    for ev in prof.key_averages():
        t = getattr(ev, "device_time_total", None)
        if t is None:
            t = ev.cuda_time_total
        if t > 0:
            rows[ev.key[:90]] = round(t / 1e3, 4)
    return dict(sorted(rows.items(), key=lambda kv: -kv[1])[:12])


def bin_counts(ia, n):
    """Rows of each bin of spgemm.cu for A.A (bound = min(sum of B row degrees, n); caps 256 and 4096)."""
    deg = torch.bincount(ia[0], minlength=n)
    ub = torch.zeros(n, dtype=torch.int64, device=ia.device).index_add_(0, ia[0], deg[ia[1]]).clamp(max=n)
    return {"warp": int(((ub > 0) & (ub <= 256)).sum()), "block": int(((ub > 256) & (ub <= 4096)).sum()),
            "bitmap": int((ub > 4096).sum()), "max_a_degree": int(deg.max())}


def plus_identity(ei, n):
    loops = torch.arange(n, device=ei.device)
    return torch.cat([ei[:, ei[0] != ei[1]], torch.stack([loops, loops])], dim=1)


def gtn_step(warmup, reps):
    sys.path.insert(0, ROOT)
    from tests.refpkg import import_reference

    import_reference()
    import cogdl_b200

    cogdl_b200.install(spspmm=True)
    from cogdl.data import Graph
    from cogdl.models.nn.gtn import GTN

    from tests.spspmm_models_ref import C_GTN, F_GTN, HID_GTN, N_GTN, gtn_inputs

    dev = torch.device("cuda:0")
    adj, x = gtn_inputs()
    model = GTN(4, 2, F_GTN, HID_GTN, C_GTN, N_GTN, 2).to(dev).train()
    graph = Graph(x=x, edge_index=adj[0][0]).to(dev)
    graph.adj = [(i.to(dev), v.to(dev)) for i, v in adj]
    y = torch.randint(0, C_GTN, (N_GTN,), device=dev)
    opt = torch.optim.Adam(model.parameters(), lr=0.01)

    def step():
        opt.zero_grad()
        torch.nn.functional.cross_entropy(model(graph), y).backward()
        opt.step()

    t, mem = median_ms_peak(step, warmup, reps)
    return {"workload": "reference GTN training step through install(spspmm=True)", "ms": round(t, 3),
            "peak_gb": round(mem, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--out")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("time_spspmm.py needs a GPU")
    import cogdl_b200  # noqa: F401
    from cogdl_b200 import synth

    dev = torch.device("cuda:0")
    res = {"card": card(), "results": []}
    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, self_loops=True)
    row = torch.repeat_interleave(torch.arange(n), rp[1:] - rp[:-1])
    ia = torch.stack([row, col]).to(dev)
    va = torch.rand(ia.shape[1], device=dev)
    res["results"].append(compare("arxiv A.A", ia, va, ia, va, n, n, n, args.warmup, args.reps))
    from cogdl_b200.structure import coo_structure_for

    merged = coo_structure_for(ia, n, n).csr
    mrow = torch.repeat_interleave(torch.arange(n, device=dev), (merged.rowptr[1:] - merged.rowptr[:-1]).long())
    res["arxiv_bins_after_merge"] = bin_counts(torch.stack([mrow, merged.colind.long()]), n)
    res["arxiv_forward_kernel_ms"] = kernel_split(ia, va, n, args.warmup)

    from tests.spspmm_models_ref import E_REL, N_GTN

    g = torch.Generator().manual_seed(1)
    mix = []
    for _ in range(2):     # one GTConv channel: the 4 relations stacked with their filter weights, coalesced
        ei = torch.randint(0, N_GTN, (2, 4 * E_REL), generator=g).to(dev)
        mix.append((ei, torch.rand(ei.shape[1], device=dev)))
    (ga, gva), (gb, gvb) = mix
    res["results"].append(compare("GTN layer product", ga, gva, gb, gvb, N_GTN, N_GTN, N_GTN, args.warmup, args.reps))
    res["results"].append(compare("GTN layer product fwd+bwd", ga, gva, gb, gvb, N_GTN, N_GTN, N_GTN, args.warmup,
                                  args.reps, backward=True))
    for name in ("cora", "pubmed"):
        nn_, ee = synth.SHAPES.get(name, (19717, 88648))
        gg = torch.Generator().manual_seed(2)
        ei = torch.randint(0, nn_, (2, ee // 2), generator=gg)
        ei = plus_identity(torch.cat([ei, ei.flip(0)], dim=1), nn_).to(dev)
        v = torch.ones(ei.shape[1], device=dev)
        res["results"].append(compare(f"SRGCN nhop=2 (A+I)^2 {name}", ei, v, ei, v, nn_, nn_, nn_, args.warmup, args.reps))
    try:
        res["results"].append(gtn_step(args.warmup, args.reps))
    except ImportError as e:
        res["results"].append({"workload": "reference GTN training step", "skipped": str(e)})
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()

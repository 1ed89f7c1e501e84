"""Child process of tests/test_gpu_correct_smooth.py: the UNMODIFIED reference Correct & Smooth
(CorrectSmoothMLP.postprocess and diffusion) through cogdl_b200.install(correct_smooth=True), on the graph and logits
of tests/golden/correct_smooth.npz.  Runs in its own process because install() rebinds the reference's dispatch for
the rest of the process.  Prints one JSON line.

Checked: every (autoscale, correct norm, smooth norm) case of postprocess and the p = 1 diffusion are bit-identical
to the same reference code after install() without the flag (its loops on this package's spmm) and within 1e-5 of the
reference's CPU results; the propagation ran in the label-propagation kernels; install() without the flag leaves the
originals alone, uninstall_correct_smooth() restores them, and CPU labels, fp64 labels, labels requiring grad, an
unknown post step and p != 1 go to the originals.
"""
import argparse
import functools
import json

import numpy as np
import torch

from tests.refpkg import import_reference
from tests.test_cpu_correct_smooth_golden import CASES, GOLDEN, NPROP, rel


def make_graph(Graph, d, dev):
    g = Graph(x=torch.from_numpy(d["x"]).clone(), y=torch.from_numpy(d["y"]).clone(),
              edge_index=(torch.from_numpy(d["row"]).clone(), torch.from_numpy(d["col"]).clone()),
              train_mask=torch.from_numpy(d["train_mask"]).clone(), val_mask=torch.from_numpy(d["val_mask"]).clone(),
              test_mask=torch.from_numpy(~(d["train_mask"] | d["val_mask"])).clone())
    return g.to(dev)


def make_model(autoscale, correct_norm, smooth_norm):
    from cogdl.models.nn.correct_smooth import CorrectSmoothMLP

    parser = argparse.ArgumentParser()
    CorrectSmoothMLP.add_args(parser)
    argv = ["--num-features", "6", "--num-classes", "5", "--num-correct-prop", str(NPROP), "--num-smooth-prop",
            str(NPROP), "--correct-norm", correct_norm, "--smooth-norm", smooth_norm] + (["--autoscale"] if autoscale else [])
    args = parser.parse_args(argv)
    args.dataset = "golden"
    return CorrectSmoothMLP(args)


def run_all(Graph, d, dev):
    import cogdl.models.nn.correct_smooth as csm

    out = {}
    logits = torch.from_numpy(d["logits"]).to(dev)
    for a, cn, sn in CASES:
        graph = make_graph(Graph, d, dev)
        # put the graph in CSR order before the first SpMM: cogdl_b200.spmm reads the edge weights before it asks for
        # the CSR, so on a graph still held as COO its first call would pair them with the unsorted order
        graph.row_indptr
        with torch.no_grad():
            out[(a, cn, sn)] = make_model(a, cn, sn).postprocess(graph, logits.clone())
    g = make_graph(Graph, d, dev)
    g.row_indptr
    g.row_norm()
    with torch.no_grad():
        out["diffusion"] = csm.diffusion(g, torch.from_numpy(d["x"]).to(dev), nhtop=10)
    return out


def main():
    import_reference()
    import cogdl.models.nn.correct_smooth as csm
    from cogdl.data import Graph

    import cogdl_b200
    from cogdl_b200 import _cabi

    dev = torch.device("cuda:0")
    d = np.load(GOLDEN)
    orig_oc, orig_diff = csm.outcome_correlation, csm.diffusion
    cogdl_b200.install()
    res = {"untouched_without_flag": csm.outcome_correlation is orig_oc and csm.diffusion is orig_diff}
    unfused = run_all(Graph, d, dev)
    res["patched"] = cogdl_b200.install(correct_smooth=True)[-2:]
    res["rebound"] = csm.outcome_correlation is not orig_oc and csm.diffusion is not orig_diff
    n0 = _cabi.launch_count()
    fused = run_all(Graph, d, dev)
    res["launches"] = _cabi.launch_count() - n0
    res["bit_identical"], res["vs_golden"] = {}, {}
    for k, v in fused.items():
        name = k if isinstance(k, str) else f"cs_{int(k[0])}_{k[1]}_{k[2]}"
        res["bit_identical"][name] = bool(torch.equal(v.view(torch.int32), unfused[k].view(torch.int32)))
        res["vs_golden"][name] = rel(v.double().cpu().numpy(), d[name].astype(np.float64))
    # the label-propagation kernels ran: the last propagation of a postprocess is one of them
    with torch.no_grad():
        make_model(True, "sym", "row").postprocess(make_graph(Graph, d, dev), torch.from_numpy(d["logits"]).to(dev))
    res["last_kernel"] = _cabi.last_kernel()

    # fallbacks: the originals get every case without a kernel
    calls = []
    spy_oc = lambda *a, **k: calls.append("outcome_correlation") or "original"  # noqa: E731
    spy_diff = lambda *a, **k: calls.append("diffusion") or "original"  # noqa: E731
    csm._cogdl_b200_original_outcome_correlation, csm._cogdl_b200_original_diffusion = spy_oc, spy_diff
    g = make_graph(Graph, d, dev)
    lab = torch.rand(g.num_nodes, 5, device=dev)
    clamp = functools.partial(csm.autoscale_post, lower=0, upper=1)
    fallbacks = {
        "cpu": csm.outcome_correlation(g, lab.cpu(), 0.8, 3, clamp),
        "fp64": csm.outcome_correlation(g, lab.double(), 0.8, 3, clamp),
        "requires_grad": csm.outcome_correlation(g, lab.clone().requires_grad_(True), 0.8, 3, clamp),
        "unknown_post_step": csm.outcome_correlation(g, lab, 0.8, 3, lambda x: x.clamp(0, 1)),
        "fixed_post_other_y": csm.outcome_correlation(g, lab, 0.8, 3, functools.partial(
            csm.fixed_post, y=lab.clone(), nid=torch.arange(3, device=dev))),
        "p2": csm.diffusion(g, lab, 3, p=2),
        "diffusion_cpu": csm.diffusion(g, lab.cpu(), 3),
    }
    res["fallbacks"] = {k: v == "original" if isinstance(v, str) else False for k, v in fallbacks.items()}
    res["fallback_calls"] = calls
    csm._cogdl_b200_original_outcome_correlation, csm._cogdl_b200_original_diffusion = orig_oc, orig_diff
    cogdl_b200.uninstall_correct_smooth()
    res["restored"] = csm.outcome_correlation is orig_oc and csm.diffusion is orig_diff
    print(json.dumps(res))


if __name__ == "__main__":
    main()

"""Child process of tests/test_gpu_spspmm.py: the UNMODIFIED reference GTN, SRGCN and Graph U-Net through
cogdl_b200.install(spspmm=True).  torch_sparse is not installed, so first the imports are shown to fail; then the models
run on the GPU through install from the parameters of the golden CPU run (tests/golden/gtn_srgcn.npz).  Logits are
compared with that run, parameter gradients with the fp64 restatements of tests/spspmm_models_ref.py (pinned to the
same golden run by test_cpu_spspmm_models_golden.py).  Runs in its own process because install() rebinds the
reference's dispatch for the rest of the process.  Prints one JSON line of measured errors.
"""
import json
import os
import sys

import numpy as np
import torch

from tests import spspmm_models_ref as R
from tests.golden.make_golden_spspmm_models import run_gtn, run_srgcn
from tests.refpkg import import_reference

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gtn_srgcn.npz")


def rel(got, want):
    got, want = torch.as_tensor(got).detach().double().cpu(), torch.as_tensor(want).detach().double().cpu()
    return float((got - want).abs().max() / want.abs().max().clamp_min(1e-30))


def fp64_grads(tag, gold, logits_fn):
    p = {k[len(f"{tag}_p_"):]: torch.from_numpy(gold[k]).double().requires_grad_(True) for k in gold.files
         if k.startswith(f"{tag}_p_")}
    (logits_fn(p) * torch.from_numpy(gold[f"{tag}_G"]).double()).sum().backward()
    return {k: v.grad for k, v in p.items() if v.grad is not None}


def state_of(tag, gold):
    return {k[len(f"{tag}_p_"):]: torch.from_numpy(gold[k]) for k in gold.files if k.startswith(f"{tag}_p_")}


def grad_err(model, want):
    got = {k: p.grad for k, p in model.named_parameters() if p.grad is not None}
    assert sorted(got) == sorted(want), (sorted(got), sorted(want))
    return max(rel(got[k], want[k]) for k in want), got


def main():
    import_reference()
    gold = np.load(GOLDEN)
    result = {}
    try:
        import cogdl.models.nn.gtn  # noqa: F401
        result["import_failed_before_install"] = False
    except ModuleNotFoundError as e:
        result["import_failed_before_install"] = e.name == "torch_sparse"

    import cogdl_b200

    result["patched"] = cogdl_b200.install(spspmm=True)
    from cogdl.data import Graph
    from cogdl.models.nn.gtn import GTN
    from cogdl.models.nn.srgcn import SRGCN

    dev = torch.device("cuda:0")
    adj = [(torch.from_numpy(gold[f"gtn_index_{r}"]).long(), torch.from_numpy(gold[f"gtn_value_{r}"])) for r in range(4)]
    want = fp64_grads("gtn", gold, lambda p: R.gtn_fp64(p, adj, torch.from_numpy(gold["gtn_x"]).double()))
    model, out, _ = run_gtn(GTN, Graph, dev, state_of("gtn", gold))
    result["gtn_logits_vs_cpu"] = rel(out, gold["gtn_logits"])
    result["gtn_grad_vs_fp64"], got = grad_err(model, want)
    conv = [k for k in got if ".conv" in k]
    result["gtn_conv_grad_nonzero"] = len(conv) == 3 and all(float(got[k].abs().max()) > 0 for k in conv)
    ei = torch.from_numpy(gold["srgcn_index"]).long()
    want = fp64_grads("srgcn", gold, lambda p: R.srgcn_fp64(p, ei, torch.from_numpy(gold["srgcn_x"]).double()))
    model, out, _ = run_srgcn(SRGCN, Graph, dev, state_of("srgcn", gold))
    result["srgcn_logits_vs_cpu"] = rel(out, gold["srgcn_logits"])
    result["srgcn_grad_vs_fp64"], _ = grad_err(model, want)

    from cogdl.models.nn.graph_unet import GraphUnet

    ei, x = R.cora_inputs()
    torch.manual_seed(0)
    unet = GraphUnet(R.F_CORA, 16, R.C_CORA, 2, [0.8, 0.6]).to(dev).eval()
    out = unet(Graph(x=x, edge_index=ei).to(dev))
    result["unet_ran"] = tuple(out.shape) == (R.N_CORA, R.C_CORA) and bool(torch.isfinite(out).all())
    unet_aug = GraphUnet(R.F_CORA, 16, R.C_CORA, 2, [0.8, 0.6], aug_adj=True).to(dev).eval()
    try:
        unet_aug(Graph(x=x, edge_index=ei).to(dev))
        result["unet_aug_adj_error"] = False
    except RuntimeError as e:       # graph_unet.py:38 moves edge_index to the CPU: no CPU path here
        result["unet_aug_adj_error"] = "CUDA" in str(e)

    from cogdl_b200.install import uninstall_spspmm

    uninstall_spspmm()
    try:
        import torch_sparse  # noqa: F401
        result["restored"] = False
    except ModuleNotFoundError:
        result["restored"] = "torch_sparse" not in sys.modules
    print(json.dumps(result))


if __name__ == "__main__":
    main()

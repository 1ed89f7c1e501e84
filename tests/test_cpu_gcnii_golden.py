"""The fp64 restatement of the reference GCNII and APPNP (tests/gcnii_ref.py) against the reference's own CPU run
(tests/golden/gcnii_appnp.npz, tests/golden/make_golden_gcnii.py): logits of every (model, graph) case, and every
parameter gradient the golden file holds (all but GCNII on the CSR-built graph, see the generator), within 1e-5 of
the largest magnitude.  test_gpu_gcnii.py then holds the fused GPU models to this restatement."""
import os

import numpy as np
import pytest
import torch

from tests import gcnii_ref
from tests.gpu_util import rel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gcnii_appnp.npz")
CASES = [(m, g) for m in ("gcnii_res0", "gcnii_res1", "appnp") for g in ("csr", "coo")]


def restated(d, model, built_from):
    """(logits, {param: grad}) of the fp64 restatement for one golden case."""
    params = gcnii_ref.leaves({k[len(f"p_{model}_"):]: d[k] for k in d.files if k.startswith(f"p_{model}_")})
    A, in_norm, out_norm = gcnii_ref.propagation(d["rowptr"], d["col"], built_from, model)
    x = torch.from_numpy(d["x"]).double()
    if model == "appnp":
        y = gcnii_ref.appnp_fp64(params, A, x, 2, 0.1, 10)
    else:
        y = gcnii_ref.gcnii_fp64(params, A, in_norm, out_norm, x, 8, 0.1, 0.5, model == "gcnii_res1")
    (y * torch.from_numpy(d["G"]).double()).sum().backward()
    return y.detach().numpy(), {k: p.grad.numpy() for k, p in params.items()}


@pytest.mark.parametrize("model,built_from", CASES)
def test_restatement_matches_the_reference(model, built_from):
    d = np.load(GOLDEN)
    y, grads = restated(d, model, built_from)
    assert rel(y, d[f"y_{model}_{built_from}"]) <= 1e-5
    keys = [k for k in d.files if k.startswith(f"g_{model}_{built_from}_")]
    assert bool(keys) == (model == "appnp" or built_from == "coo")
    for k in keys:
        name = k[len(f"g_{model}_{built_from}_"):]
        assert rel(grads[name], d[k]) <= 1e-5, name

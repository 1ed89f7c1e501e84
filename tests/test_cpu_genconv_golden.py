"""The fp64 restatement of GENConv's aggregation (tests/genconv_ref.py), which the GPU tests use as their yardstick,
against the reference GENConv's own CPU output (tests/golden/genconv.npz, made by make_golden_genconv.py)."""
import os

import numpy as np
import pytest
import torch

from tests.genconv_ref import genconv_aggregate_fp64
from tests.golden.make_golden_genconv import CASES, case_key

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "genconv.npz"))


def row_scaled_err(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = np.maximum(np.abs(want), np.abs(want).max(axis=1, keepdims=True))
    return float((np.abs(got - want) / np.maximum(scale, 1e-30)).max())


@pytest.mark.parametrize("edge", [False, True])
@pytest.mark.parametrize("aggr,beta", CASES)
def test_fp64_restatement_matches_reference_genconv(aggr, beta, edge):
    key = case_key(aggr, beta, edge)
    x = torch.from_numpy(GOLDEN["x"])
    a = torch.from_numpy(GOLDEN["edge_" + key]) if edge else None
    h = genconv_aggregate_fp64(torch.from_numpy(GOLDEN["rowptr"]), torch.from_numpy(GOLDEN["colind"]), x, aggr,
                               beta=1.0 if beta is None else beta, edge_term=a, p=2.0)
    want = GOLDEN["h_" + key]
    assert want.shape == tuple(h.shape)
    deg0 = np.diff(GOLDEN["rowptr"]) == 0
    assert deg0.any() and np.all(want[deg0] == 0), "the golden graph has degree-0 rows, aggregated to 0"
    assert row_scaled_err(h.numpy(), want) <= 1e-5, key

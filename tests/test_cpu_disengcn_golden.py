"""The fp64 restatement of DisenGCN's routing (tests/disengcn_ref.py), which the GPU tests use as their yardstick,
against the reference DisenGCNLayer's own CPU output (tests/golden/disengcn.npz, made by make_golden_disengcn.py)."""
import os

import numpy as np
import pytest
import torch

from tests.disengcn_ref import disen_routing_fp64
from tests.golden.make_golden_disengcn import CASES, case_key

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "disengcn.npz"))


def row_scaled_err(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = np.maximum(np.abs(want), np.abs(want).max(axis=1, keepdims=True))
    return float((np.abs(got - want) / np.maximum(scale, 1e-30)).max())


@pytest.mark.parametrize("K,d,T,tau", CASES)
def test_fp64_restatement_matches_reference_disengcn_layer(K, d, T, tau):
    key = case_key(K, d, T, tau)
    x = torch.from_numpy(GOLDEN["x"]).double()
    W, b = torch.from_numpy(GOLDEN["W_" + key]).double(), torch.from_numpy(GOLDEN["b_" + key]).double()
    h = torch.nn.functional.leaky_relu(x @ W + b)
    rowptr = torch.from_numpy(GOLDEN["rowptr"])
    got = disen_routing_fp64(rowptr, torch.from_numpy(GOLDEN["colind"]), h, K, T, tau)
    want = GOLDEN["out_" + key]
    assert want.shape == tuple(got.shape) == (x.shape[0], K * d)
    assert (np.diff(GOLDEN["rowptr"]) == 0).any(), "the golden graph has degree-0 rows"
    assert row_scaled_err(got.numpy(), want) <= 1e-5, key

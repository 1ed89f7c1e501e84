"""The fp64 restatement of CompGCNLayer (tests/compgcn_ref.py), which the GPU tests use as their yardstick, against the
reference CompGCNLayer's own CPU forward and backward (tests/golden/compgcn.npz, made by make_golden_compgcn.py)."""
import os

import numpy as np
import pytest
import torch

from tests.compgcn_ref import compgcn_layer_fp64
from tests.golden.make_golden_compgcn import CASES, case_key

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "compgcn.npz"))


def row_scaled_err(got, want):
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    if want.ndim == 1:
        got, want = got[None, :], want[None, :]
    scale = np.maximum(np.abs(want), np.abs(want).max(axis=1, keepdims=True))
    return float((np.abs(got - want) / np.maximum(scale, 1e-30)).max())


def test_golden_kg_shape():
    row, col, typ = GOLDEN["row"], GOLDEN["col"], GOLDEN["type"]
    E, N = row.size, GOLDEN["x"].shape[0]
    assert E % 2 == 1
    assert not np.array_equal(row[: E // 2], np.sort(row[: E // 2])), "the COO is shuffled"
    for h in (slice(0, E // 2), slice(E // 2, E)):
        deg = np.bincount(row[h], minlength=N)
        assert (deg == 0).any() and (deg > 1).any()
    assert np.intersect1d(row[: E // 2], row[E // 2:]).size > 0, "some rows have edges in both halves"
    assert typ.max() < 2 * GOLDEN["rel"].shape[0]


@pytest.mark.parametrize("opn,bases", CASES)
def test_fp64_restatement_matches_reference_compgcn_layer(opn, bases):
    key = case_key(opn, bases)
    prefix = f"p_{key}_"
    p = {k[len(prefix):]: torch.from_numpy(GOLDEN[k]).double().requires_grad_(True)
         for k in GOLDEN.files if k.startswith(prefix)}
    x = torch.from_numpy(GOLDEN["x"]).double().requires_grad_(True)
    rel = torch.from_numpy(GOLDEN["rel"]).double().requires_grad_(True)
    y, yr = compgcn_layer_fp64(p, GOLDEN["row"], GOLDEN["col"], GOLDEN["type"], x, rel, opn)
    ((y * torch.from_numpy(GOLDEN["G"]).double()).sum() + (yr * torch.from_numpy(GOLDEN["GR"]).double()).sum()).backward()
    assert row_scaled_err(y.detach(), GOLDEN["y_" + key]) <= 1e-5, key
    assert row_scaled_err(yr.detach(), GOLDEN["yr_" + key]) <= 1e-5, key
    assert row_scaled_err(x.grad, GOLDEN["dx_" + key]) <= 1e-5, key
    if not bases:
        assert row_scaled_err(rel.grad, GOLDEN["drel_" + key]) <= 1e-5, key
    names = [k[len(f"g_{key}_"):] for k in GOLDEN.files if k.startswith(f"g_{key}_")]
    assert set(names) == set(p), key
    for name in names:
        got, want = p[name].grad, GOLDEN[f"g_{key}_{name}"]
        if float(got.abs().max()) < 1e-12:
            # exactly zero in exact arithmetic: training-mode BN removes any shift shared by all rows (the bias,
            # and loop_rel under sub); the fp32 reference leaves rounding noise there
            assert float(np.abs(want).max()) <= 1e-5, (key, name)
        else:
            assert row_scaled_err(got, want) <= 1e-5, (key, name)

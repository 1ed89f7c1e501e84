"""An fp64 restatement of the reference's GINLayer / GINELayer aggregation (with d x and d eps) and Grand.rand_prop
against the reference's own CPU run (tests/golden/gin_grand.npz, tests/golden/make_golden_gin_grand.py), within 1e-5 of
the largest magnitude.  test_gpu_gin_grand.py then holds the reference layers and rand_prop run through
install(gin=True, grand=True) to the golden file."""
import os

import numpy as np
import pytest
import scipy.sparse as sp
import torch

from tests.gpu_util import rel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gin_grand.npz")
GIN_CASES = (("gin", 0.1, True), ("gin_fixed", -1.0, False), ("gine", -0.3, True))
ORDERS = (0, 1, 2, 8)
DROPNODE, SEED = 0.5, 123


def gin_fp64(row, col, n, x, g, eps):
    """(1 + eps) x + A x with A[i, j] the number of edges i -> j (cogdl's spmm sums x[col] into row), and for the
    upstream gradient g: d x = (1 + eps) g + A^T g, d eps = sum(g * x)."""
    A = sp.coo_matrix((np.ones(len(row)), (row, col)), shape=(n, n)).tocsr()
    x, g = x.astype(np.float64), g.astype(np.float64)
    return (1 + eps) * x + A @ x, (1 + eps) * g + A.T @ g, float((g * x).sum())


def rand_prop_fp64(row, col, w, n, x0, order):
    """x0 + A x0 + ... + A^order x0, over order + 1 (GRAND's propagation after DropNode)."""
    A = sp.coo_matrix((w.astype(np.float64), (row, col)), shape=(n, n)).tocsr()
    h = x0.astype(np.float64)
    y = h.copy()
    for _ in range(order):
        h = A @ h
        y += h
    return y / (order + 1)


def dropnode_mask(n):
    """The mask Grand.drop_node draws in train mode after torch.manual_seed(SEED)."""
    torch.manual_seed(SEED)
    return torch.bernoulli(1.0 - torch.ones(n) * DROPNODE).numpy()


@pytest.mark.parametrize("key,eps,train", GIN_CASES)
def test_gin_restatement_matches_the_reference(key, eps, train):
    d = np.load(GOLDEN)
    n = d["x"].shape[0]
    out, dx, deps = gin_fp64(d["row"], d["col"], n, d["x"], d["g"], np.float64(np.float32(eps)))
    assert rel(out, d[f"{key}_out"]) <= 1e-5
    assert rel(dx, d[f"{key}_dx"]) <= 1e-5
    if train:
        assert abs(deps - float(d[f"{key}_deps"][0])) <= 1e-5 * np.abs(d["g"] * d["x"]).sum()


@pytest.mark.parametrize("order", ORDERS)
def test_rand_prop_restatement_matches_the_reference(order):
    d = np.load(GOLDEN)
    n = d["x"].shape[0]
    mask = d[f"mask_{order}"]
    assert np.array_equal(mask, dropnode_mask(n)), "the seed draws another DropNode mask"
    train = rand_prop_fp64(d["srow"], d["scol"], d["sw"], n, mask[:, None] * d["x"], order)
    assert rel(train, d[f"grand_train_{order}"]) <= 1e-5
    ev = rand_prop_fp64(d["srow"], d["scol"], d["sw"], n, d["x"] * (1.0 - DROPNODE), order)
    assert rel(ev, d[f"grand_eval_{order}"]) <= 1e-5


def test_golden_graph_has_a_hub_and_an_isolated_node():
    d = np.load(GOLDEN)
    deg = np.bincount(d["row"], minlength=d["x"].shape[0])
    assert deg.max() >= 100 and (deg == 0).sum() >= 1
    assert 0 < d["mask_8"].sum() < d["x"].shape[0]

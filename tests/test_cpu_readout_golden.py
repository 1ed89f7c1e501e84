"""The fp64 restatements of the graph-level readouts (tests/readout_ref.py) against the reference's own CPU run
(tests/golden/readout.npz, tests/golden/make_golden_readout.py): sum and mean pooling, the GIN model's pooled layer
outputs, the InfoGraph encoder's graph_rep and the [B, k, F] tensor SortPool pools, within 1e-5 of the largest
magnitude.  test_gpu_readout.py then holds the kernels to these restatements, and readout_refpkg_check.py the reference
models run through install(readout=True) to the golden file.

Max pooling and Set2Set have no golden entry: the reference's batch_max_pooling needs torch_scatter, which is not
installed, and its Set2Set.forward crashes (it calls edge_softmax(graph, edge_val) with the logits for the graph).  They
are pinned here against torch's own fp64 formulations of the same readouts: scatter_reduce's amax and autograd through
an index_add_ softmax."""
import os

import numpy as np
import pytest
import torch

from tests import readout_ref as R
from tests.gpu_util import rel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "readout.npz")
K = 25          # SortPool's k in the golden file (make_golden_readout.K)


def _golden():
    d = np.load(GOLDEN)
    return d, d["batch"], int(d["batch"].max()) + 1


def test_sum_and_mean_restatements_match_the_reference():
    d, batch, B = _golden()
    assert rel(R.sum_pool(d["x2"], batch, B), d["sum_x2"]) <= 1e-5
    assert rel(R.mean_pool(d["x2"], batch, B), d["mean_x2"]) <= 1e-5


def test_gin_pooled_layer_outputs_are_sum_pools():
    d, batch, B = _golden()
    reps = [d["x"], d["gin_rep_1"], d["gin_rep_2"]]
    for i, rep in enumerate(reps):
        assert rel(R.sum_pool(rep, batch, B), d[f"gin_pooled_{i}"]) <= 1e-5, i


def test_infograph_graph_rep_is_the_concatenated_sum_pools():
    d, batch, B = _golden()
    node_rep = d["ig_node_rep"]
    assert node_rep.shape[1] == 48
    want = np.concatenate([R.sum_pool(node_rep[:, 16 * i:16 * (i + 1)], batch, B) for i in range(3)], axis=1)
    assert rel(want, d["ig_graph_rep"]) <= 1e-5


def test_sort_pool_restatement_matches_the_reference():
    d, batch, B = _golden()
    n = np.bincount(batch, minlength=B)
    assert (n < K).any() and (n > K).any(), "the golden batch must have graphs on both sides of k"
    out, idx = R.sort_pool(d["sp_h"], batch, B, K)
    assert rel(out, d["sp_pooled"]) <= 1e-5
    assert ((idx >= 0).sum(1) == np.minimum(n, K)).all()


def test_max_restatement_is_scatter_reduce_amax():
    rng = np.random.default_rng(3)
    batch = np.sort(rng.integers(0, 9, 200))
    batch[batch == 4] = 5                                   # graph 4 has no nodes
    x = rng.standard_normal((200, 7)).astype(np.float32)
    x[10, 2] = x[11, 2] = 5.0                               # a tie inside one graph (batch is sorted)
    out, arg = R.max_pool(x, batch, 9)
    t = torch.zeros(9, 7, dtype=torch.float64).scatter_reduce(
        0, torch.from_numpy(batch)[:, None].expand(-1, 7), torch.from_numpy(x).double(), "amax", include_self=False)
    assert np.array_equal(out, t.numpy())
    assert (arg[4] == -1).all() and (out[4] == 0).all()
    if batch[10] == batch[11]:
        assert arg[batch[10], 2] == 10
    sel = arg >= 0
    assert np.array_equal(x[arg[sel], np.nonzero(sel)[1]], out[sel])
    dy = rng.standard_normal((9, 7))
    dx = R.max_pool_grad(dy, arg, 200)
    assert np.isclose(dx.sum(), dy[sel].sum())


def test_max_restatement_nan_and_empty_rules():
    x = np.array([[np.nan, 1.0], [np.nan, np.inf], [2.0, -np.inf]], np.float32)
    out, arg = R.max_pool(x, np.array([0, 0, 2]), 3)
    assert np.isneginf(out[0, 0]) and arg[0, 0] == -1      # a column of NaN alone
    assert out[0, 1] == np.inf and arg[0, 1] == 1
    assert (out[1] == 0).all() and (arg[1] == -1).all()    # no nodes
    assert out[2, 1] == -np.inf and arg[2, 1] == -1     # -inf is never above the start value


@pytest.mark.parametrize("F", [1, 6])
def test_set2set_restatement_and_gradients_match_autograd(F):
    rng = np.random.default_rng(F)
    batch = np.array([0, 0, 0, 2, 2, 3, 0, 3, 3, 3])       # unsorted, graph 1 empty
    B = 4
    x, q, dr = rng.standard_normal((10, F)), rng.standard_normal((B, F)), rng.standard_normal((B, F))
    xt = torch.from_numpy(x).requires_grad_(True)
    qt = torch.from_numpy(q).requires_grad_(True)
    bt = torch.from_numpy(batch)
    e = (xt * qt[bt]).sum(-1)
    m = torch.full((B,), -torch.inf, dtype=torch.float64).scatter_reduce(0, bt, e, "amax")
    w = torch.exp(e - m[bt])
    a = w / torch.zeros(B, dtype=torch.float64).index_add(0, bt, w)[bt]
    r = torch.zeros(B, F, dtype=torch.float64).index_add(0, bt, a[:, None] * xt)
    r.backward(torch.from_numpy(dr))
    got_r, got_a = R.set2set(x, q, batch, B)
    assert np.allclose(got_r, r.detach().numpy(), rtol=1e-12, atol=1e-12)
    assert np.allclose(got_a, a.detach().numpy(), rtol=1e-12, atol=1e-12)
    assert (got_r[1] == 0).all()
    dx, dq = R.set2set_grad(x, q, batch, B, dr)
    assert np.allclose(dx, xt.grad.numpy(), rtol=1e-10, atol=1e-12)
    assert np.allclose(dq, qt.grad.numpy(), rtol=1e-10, atol=1e-12)


def test_sort_pool_restatement_is_a_stable_descending_sort():
    h = np.zeros((9, 2))
    h[:, 1] = [1.0, np.nan, 3.0, 1.0, -np.inf, np.inf, -0.0, 0.0, np.nan]
    batch = np.array([0, 0, 0, 0, 0, 0, 0, 0, 2])
    out, idx = R.sort_pool(h, batch, 3, 10)
    assert list(idx[0, :8]) == [1, 5, 2, 0, 3, 6, 7, 4] and (idx[0, 8:] == -1).all()
    assert (idx[1] == -1).all() and list(idx[2, :1]) == [8]
    t = torch.sort(torch.from_numpy(h[:8, 1]), descending=True, stable=True).indices.numpy()
    assert list(t) == list(idx[0, :8])
    dy = np.arange(30 * 2, dtype=np.float64).reshape(3, 10, 2)
    dx = R.sort_pool_grad(dy, idx, 9)
    assert np.array_equal(dx[5], dy[0, 1]) and np.array_equal(dx[8], dy[2, 0])

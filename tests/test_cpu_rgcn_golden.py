"""The fp64 restatement of R-GCN's basis layer (tests/rgcn_ref.py) against the reference's own CPU run
(tests/golden/rgcn.npz, tests/golden/make_golden_rgcn.py), within 1e-5 of the largest magnitude:

  * at T = 1 the reference layer (with layer_norm, bias and self loop) is the relational sum;
  * at T > 1 the relational sum is the sum of the reference's own per-relation spmm pieces;
  * at T > 1 the reference layer's output is the first present relation's weight applied to every edge, and not the
    relational sum (the indentation of `return h_list` in RGCNLayer.basis_forward)."""
import os

import numpy as np
import torch

from tests.gpu_util import rel
from tests.rgcn_ref import first_present, layer_post, relational_sum, row_norm_weights, type_weights

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "rgcn.npz")


def load():
    d = np.load(GOLDEN)
    return {k: d[k] for k in d.files}


def params(d, T):
    pre = f"p_t{T}_"
    return {k[len(pre):]: torch.from_numpy(v).double() for k, v in d.items() if k.startswith(pre)}


def test_row_norm_weights_are_the_references():
    d = load()
    n = d["x"].shape[0]
    assert rel(row_norm_weights(d["srow"], n).numpy(), d["sw"]) <= 1e-6
    assert rel(row_norm_weights(d["row"], n).numpy()[np.argsort(d["row"], kind="stable")], d["sw"]) <= 1e-6


def test_single_relation_layer_is_the_relational_sum():
    d = load()
    x = torch.from_numpy(d["x"]).double()
    p = params(d, 1)
    w_hat = row_norm_weights(d["row"], x.shape[0])
    h = relational_sum(d["row"], d["col"], d["type_t1"], w_hat, x, type_weights(None, p["weight"], 1))
    assert rel(layer_post(h, x, p).numpy(), d["out_t1"]) <= 1e-5


def test_relational_sum_is_the_sum_of_the_reference_pieces():
    d = load()
    x = torch.from_numpy(d["x"]).double()
    p = params(d, 4)
    W = type_weights(p["alpha"], p["weight"], 4)
    w_hat = row_norm_weights(d["row"], x.shape[0])
    h = relational_sum(d["row"], d["col"], d["type_t4"], w_hat, x, W).numpy()
    pieces = sum(d[f"piece_{t}"].astype(np.float64) for t in range(4))
    assert rel(h, pieces) <= 1e-5
    # the same sum from the graph's CSR-order copy, whose types were reordered with the edges
    h_csr = relational_sum(d["srow"], d["scol"], d["stype_t4"], torch.from_numpy(d["sw"]).double(), x, W).numpy()
    assert rel(h_csr, h) <= 1e-5


def test_reference_multi_relation_layer_uses_the_first_present_relation():
    d = load()
    x = torch.from_numpy(d["x"]).double()
    p = params(d, 4)
    W = type_weights(p["alpha"], p["weight"], 4)
    w_hat = row_norm_weights(d["row"], x.shape[0])
    assert int(d["type_t4"].min()) == 1
    fp = first_present(d["row"], d["col"], d["type_t4"], w_hat, x, W).numpy()
    assert rel(d["out_t4"], fp) <= 1e-5
    rs = relational_sum(d["row"], d["col"], d["type_t4"], w_hat, x, W).numpy()
    assert rel(d["out_t4"], rs) > 1e-2

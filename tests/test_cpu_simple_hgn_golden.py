"""The fp64 restatement of Simple-HGN's layer (tests/simple_hgn_ref.py) against the reference's own CPU run of
myGATConv (tests/golden/simple_hgn.npz, tests/golden/make_golden_simple_hgn.py): three stacked convs (the second with
res_attn and a residual Linear, the third with one head) on a shuffled COO with types and empty rows, run on the
graph's CSR with the types put through the same stable sort by row (the edge-order rule the installed layer follows).
The restatement computes the CSR from the COO itself: outputs and returned attentions (CSR order) within 1e-5,
gradients of x and every parameter within 2e-5, all relative to the largest magnitude."""
import os

import numpy as np
import torch

from tests.gpu_util import rel
from tests.simple_hgn_ref import conv_fp64

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "simple_hgn.npz")
SLOPE, ALPHA = 0.2, 0.05
HEADS = (8, 8, 1)


def load():
    d = np.load(GOLDEN)
    return {k: d[k] for k in d.files}


def csr_of(d):
    """(rowptr, colind, type, order): the stable sort by row that building the CSR applies to the COO."""
    n = d["x"].shape[0]
    order = np.argsort(d["row"], kind="stable")
    rowptr = np.zeros(n + 1, np.int64)
    rowptr[1:] = np.cumsum(np.bincount(d["row"], minlength=n))
    return rowptr, d["col"][order], d["type"][order], order


def run_fp64(d):
    rowptr, colind, etype, _ = csr_of(d)
    x = torch.from_numpy(d["x"]).double().requires_grad_(True)
    prm = [{k[3:]: torch.from_numpy(v).double().requires_grad_(True) for k, v in d.items() if k.startswith(f"c{i}_")}
           for i in (1, 2, 3)]
    act = torch.tanh
    out1, m1 = conv_fp64(prm[0], rowptr, colind, etype, x, HEADS[0], SLOPE, act=act)
    out2, m2 = conv_fp64(prm[1], rowptr, colind, etype, out1, HEADS[1], SLOPE, ALPHA, res_attn=m1.detach(), act=act)
    out3, m3 = conv_fp64(prm[2], rowptr, colind, etype, out2, HEADS[2], SLOPE)
    ((out2 * torch.from_numpy(d["g2"]).double()).sum() + (out3 * torch.from_numpy(d["g3"]).double()).sum()).backward()
    return (out1, out2, out3), (m1, m2, m3), x, prm


def test_outputs_and_attentions_match_the_reference():
    d = load()
    outs, atts, _, _ = run_fp64(d)
    assert np.array_equal(csr_of(d)[3], d["order"])
    for k in range(3):
        assert rel(outs[k].detach().numpy(), d[f"out{k + 1}"]) <= 1e-5, f"out{k + 1}"
        assert rel(atts[k].detach().numpy(), d[f"att{k + 1}"]) <= 1e-5, f"att{k + 1}"


def test_gradients_match_the_reference():
    d = load()
    _, _, x, prm = run_fp64(d)
    assert rel(x.grad.numpy(), d["grad_x"]) <= 2e-5
    for i, p in enumerate(prm, 1):
        for name, t in p.items():
            assert rel(t.grad.numpy(), d[f"grad_c{i}_{name}"]) <= 2e-5, f"c{i}.{name}"


def test_types_follow_their_edges():
    """Restating on the CSR with the types left in COO order pairs logits with other edges' types: the fixture tells
    the two apart, so the order rule above is what makes the match."""
    d = load()
    rowptr, colind, _, _ = csr_of(d)
    x = torch.from_numpy(d["x"]).double()
    prm = {k[3:]: torch.from_numpy(v).double() for k, v in d.items() if k.startswith("c1_")}
    out, _ = conv_fp64(prm, rowptr, colind, d["type"], x, HEADS[0], SLOPE, act=torch.tanh)
    assert rel(out.numpy(), d["out1"]) > 1e-3

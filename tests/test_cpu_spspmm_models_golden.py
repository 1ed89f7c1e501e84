"""The fp64 restatements of GTN and SRGCN (tests/spspmm_models_ref.py), which the GPU check of spspmm uses as its
gradient yardstick, against the reference models' own CPU run (tests/golden/gtn_srgcn.npz, made by
make_golden_spspmm_models.py with fp64 sparse products)."""
import os

import numpy as np
import pytest
import torch

from tests.gpu_util import rel
from tests import spspmm_models_ref as R

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gtn_srgcn.npz"))


def params(tag):
    pre = f"{tag}_p_"
    return {k[len(pre):]: torch.from_numpy(GOLDEN[k]).double().requires_grad_(True) for k in GOLDEN.files
            if k.startswith(pre)}


def check(tag, p, logits):
    assert rel(logits.detach(), GOLDEN[f"{tag}_logits"]) <= 1e-5
    (logits * torch.from_numpy(GOLDEN[f"{tag}_G"]).double()).sum().backward()
    names = [k[len(f"{tag}_g_"):] for k in GOLDEN.files if k.startswith(f"{tag}_g_")]
    assert names and set(names) <= set(p)
    for name in names:
        # 2e-5: a one-element bias gradient is a signed sum over every node, which the fp32 reference run knows only
        # to about 1e-5 of its value (SRGCN's out_att.attention.p.bias sits at 1.01e-5)
        assert rel(p[name].grad, GOLDEN[f"{tag}_g_{name}"]) <= 2e-5, name


def test_golden_inputs_are_the_seeded_ones():
    adj, x = R.gtn_inputs()
    for r, (e, v) in enumerate(adj):
        assert np.array_equal(GOLDEN[f"gtn_index_{r}"], e.numpy()) and np.array_equal(GOLDEN[f"gtn_value_{r}"], v.numpy())
    assert np.array_equal(GOLDEN["gtn_x"], x.numpy())
    ei, xc = R.cora_inputs()
    assert np.array_equal(GOLDEN["srgcn_index"], ei.numpy()) and np.array_equal(GOLDEN["srgcn_x"], xc.numpy())
    # the relations overlap, so GTConv's coalesce takes its duplicate branch
    allidx = np.concatenate([GOLDEN[f"gtn_index_{r}"] for r in range(4)], axis=1)
    assert np.unique(allidx, axis=1).shape[1] < allidx.shape[1]


@pytest.mark.parametrize("tag", ["gtn", "srgcn"])
def test_fp64_restatement_matches_the_reference_model(tag):
    p = params(tag)
    if tag == "gtn":
        adj = [(torch.from_numpy(GOLDEN[f"gtn_index_{r}"]).long(), torch.from_numpy(GOLDEN[f"gtn_value_{r}"]))
               for r in range(4)]
        logits = R.gtn_fp64(p, adj, torch.from_numpy(GOLDEN["gtn_x"]).double())
    else:
        logits = R.srgcn_fp64(p, torch.from_numpy(GOLDEN["srgcn_index"]).long(),
                              torch.from_numpy(GOLDEN["srgcn_x"]).double())
    check(tag, p, logits)
    if tag == "gtn":     # the GTConv filters train only through the values of the product
        assert all(float(p[f"layers.{i}.{c}.weight"].grad.abs().max()) > 0
                   for i, c in ((0, "conv1"), (0, "conv2"), (1, "conv1")))

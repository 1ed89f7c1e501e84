"""The fp64 restatement of the reference's Correct & Smooth (tests/correct_smooth_ref.py) against the reference's own
CPU run (tests/golden/correct_smooth.npz, tests/golden/make_golden_correct_smooth.py): every (autoscale, correct norm,
smooth norm) case and the p = 1 diffusion, within 1e-5 of the largest magnitude.  test_gpu_correct_smooth.py then holds
the reference model run through install(correct_smooth=True) to the golden file."""
import os

import numpy as np
import pytest

from tests import correct_smooth_ref as ref
from tests.gpu_util import rel

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "correct_smooth.npz")
CASES = [(a, cn, sn) for a in (False, True) for cn in ("sym", "row") for sn in ("row", "col")]
NPROP, CORRECT_ALPHA, SMOOTH_ALPHA = 20, 1.0, 0.8


def softmax(z):
    e = np.exp(z - z.max(axis=1, keepdims=True))
    return e / e.sum(axis=1, keepdims=True)


@pytest.mark.parametrize("autoscale,correct_norm,smooth_norm", CASES)
def test_restatement_matches_the_reference(autoscale, correct_norm, smooth_norm):
    d = np.load(GOLDEN)
    n = d["logits"].shape[0]
    got = ref.correct_smooth_fp64(d["row"], d["col"], n, softmax(d["logits"].astype(np.float64)), d["y"],
                                  d["train_mask"], autoscale, correct_norm, smooth_norm, CORRECT_ALPHA, SMOOTH_ALPHA,
                                  NPROP, NPROP)
    assert rel(got, d[f"cs_{int(autoscale)}_{correct_norm}_{smooth_norm}"]) <= 1e-5


def test_diffusion_restatement_matches_the_reference():
    d = np.load(GOLDEN)
    n = d["logits"].shape[0]
    got = ref.diffusion_fp64(ref.adjacency(d["row"], d["col"], n, "row"), d["x"], 10)
    assert rel(got, d["diffusion"]) <= 1e-5


def test_golden_graph_has_a_hub_and_an_isolated_node():
    d = np.load(GOLDEN)
    deg = np.bincount(d["row"], minlength=d["logits"].shape[0])
    assert deg.max() >= 100 and (deg == 0).sum() >= 1

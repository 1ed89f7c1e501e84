"""The attention-dropout mask contract of the fused GAT, without a GPU: the numpy keep rule (tests/gat_dropout_ref.py)
against the library's exported draw function and its expected keep rate, and the fp64 restatement of the dropout
GATLayer against the reference layer's own CPU output (tests/golden/gat_dropout.npz, make_golden_gat_dropout.py)."""
import os

import numpy as np
import pytest
import torch

from tests.gat_dropout_ref import draw, drop_below, gat_layer_fp64, keep_mask

GOLDEN = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "gat_dropout.npz"))


def test_numpy_draw_matches_library_draw():
    from cogdl_b200 import _cabi

    lib = _cabi.load()
    for seed in (0, 1, 0x5EED0001, 2 ** 63 + 12345, 2 ** 64 - 1):
        for e in (0, 1, 2, 1000, 2 ** 31 - 1, 61_859_140):
            for h in range(8):
                assert int(draw(seed, e, h)) == int(lib.cogdl_b200_sample_draw(seed, e, h)), (seed, e, h)


def test_drop_threshold_and_scale():
    from cogdl_b200.operators._raw import attn_dropout_args

    for p in (0.0, 0.1, 0.5, 0.9, 0.999):
        below, scale = attn_dropout_args(p)
        assert below == drop_below(p) == int(np.floor(np.float64(p) * 2.0 ** 64))
        assert scale == 1.0 / (1.0 - p)
    assert attn_dropout_args(0.5)[0] == 2 ** 63
    for bad in (1.0, -0.1, 1.5, float("nan")):
        with pytest.raises(ValueError):
            attn_dropout_args(bad)


@pytest.mark.parametrize("p", [0.1, 0.5, 0.9])
def test_keep_fraction_within_6_sigma(p):
    n = 125_000
    keep = keep_mask(0xC0FFEE + int(p * 10), n, 8, p)          # 10^6 draws
    sigma = np.sqrt(p * (1 - p) / keep.size)
    assert abs(keep.mean() - (1 - p)) <= 6 * sigma
    # no head or edge stripe is biased either (each head: 125 000 draws)
    assert np.all(np.abs(keep.mean(axis=0) - (1 - p)) <= 6 * np.sqrt(p * (1 - p) / n))


def test_p_zero_keeps_everything():
    assert keep_mask(123, 10_000, 8, 0.0).all()


def test_golden_graph_shape():
    row, col, rowptr = GOLDEN["row"], GOLDEN["col"], GOLDEN["rowptr"]
    n = GOLDEN["x"].shape[0]
    deg = np.diff(rowptr)
    assert (deg == 0).sum() >= 50 and deg.max() >= 200, "degree-0 rows and a hub row"
    assert np.array_equal(np.repeat(np.arange(n), deg), row), "edges in CSR order"
    assert set(zip(row.tolist(), col.tolist())) != set(zip(col.tolist(), row.tolist()))


@pytest.mark.parametrize("key", ["h8", "h1"])
def test_fp64_restatement_matches_reference_gat_layer(key):
    p, slope = float(GOLDEN["p"]), float(GOLDEN["slope"])
    seed = int(GOLDEN[f"seed_{key}"])
    mask = GOLDEN[f"mask_{key}"]
    assert np.array_equal(mask, keep_mask(seed, GOLDEN["col"].size, mask.shape[1], p)), "the golden mask is the keep rule"
    assert 0.4 < mask.mean() < 0.6
    x = torch.from_numpy(GOLDEN["x"]).double()
    W, a_l, a_r = (torch.from_numpy(GOLDEN[f"{k}_{key}"]).double() for k in ("W", "a_l", "a_r"))
    y = gat_layer_fp64(x, W, a_l, a_r, GOLDEN["rowptr"], GOLDEN["col"], slope, mask, p).numpy()
    want = GOLDEN[f"y_{key}"].astype(np.float64)
    assert np.abs(y - want).max() <= 1e-5 * np.abs(want).max()
    # the mask matters: without it (or with another seed) the output is far off
    y_nodrop = gat_layer_fp64(x, W, a_l, a_r, GOLDEN["rowptr"], GOLDEN["col"], slope, np.ones_like(mask), 0.0).numpy()
    assert np.abs(y_nodrop - want).max() > 0.05 * np.abs(want).max()

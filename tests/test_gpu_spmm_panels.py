"""Column-panel form of the fp32 SpMM (X larger than the L2): one pass per column panel of X, panel-major.

Whatever the panel count, the output must be bitwise equal to the single-pass kernel on every row (hub rows
included: per-panel partials are combined in the same chunk order) and bitwise equal to the oracle on rows
the hub plan does not split.
"""
import numpy as np
import pytest
import torch

import oracle
from tests.gpu_util import bits, dev, plan_structure
from tests.graphs import case

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["hub", "two_hubs", "ragged", "rect"])
@pytest.mark.parametrize("F", [128, 256])
@pytest.mark.parametrize("weighted", [True, False])
@pytest.mark.parametrize("chunk", [64, 256])
def test_panels_bitwise_equal_single_pass(dev, name, F, weighted, chunk):
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n_cols = case(name)
    rng = np.random.default_rng(3)
    X = rng.standard_normal((n_cols, F)).astype(np.float32)
    val = rng.random(ci.shape[0]).astype(np.float32) if weighted else None
    ref = oracle.spmm_csr(rp, ci, val, X)
    st = plan_structure(rp, ci, n_cols, dev, chunk=chunk)
    assert st.plan.n_segs > 0
    x_d = torch.from_numpy(X).to(dev)
    v_d = None if val is None else torch.from_numpy(val).to(dev)
    y1 = spmm_raw(st, v_d, x_d, panels=1)
    assert "panels=" not in _cabi.last_kernel()
    unsplit = np.diff(rp) <= chunk
    for P in [2, 4] + ([8] if F == 256 else []):
        y = spmm_raw(st, v_d, x_d, panels=P)
        assert f",panels={P}" in _cabi.last_kernel()
        assert torch.equal(bits(y), bits(y1)), f"panels={P} differs from the single-pass kernel"
        assert np.array_equal(y.cpu().numpy()[unsplit], ref[unsplit]), f"panels={P}: unsplit rows differ from the oracle"
        assert torch.equal(bits(spmm_raw(st, v_d, x_d, panels=P)), bits(y)), "second call differs"
        assert int(st.plan.counters.abs().sum()) == 0, "per-panel arrival counters must be left zero"


def test_forced_panels_out_of_range_is_an_error(dev):
    from cogdl_b200._cabi import CogdlB200Error
    from cogdl_b200.operators._raw import spmm_raw

    rp, ci, n_cols = case("hub")
    st = plan_structure(rp, ci, n_cols, dev, chunk=256)
    for F, P in ((128, 3), (128, 8), (40, 2), (512, 2), (192, 2), (384, 4)):
        with pytest.raises(CogdlB200Error):
            spmm_raw(st, None, torch.randn(n_cols, F, device=dev), panels=P)


def expected_auto_panels(x_bytes, F):
    """The selection rule: smallest power of two whose panel takes at most 7/8 of the L2, else 1."""
    budget = torch.cuda.get_device_properties(0).L2_cache_size * 7 // 8
    if x_bytes <= budget:
        return 1
    P = 2
    while P <= 8 and 32 * P <= F:
        if F % (32 * P) == 0 and F // P <= 128 and x_bytes // P <= budget:
            return P
        P *= 2
    return 1


@pytest.mark.parametrize("x_rows,F", [(169343, 128), (169343, 40), (20000, 128), (2449029, 128)])
def test_automatic_panel_count_follows_x_size(dev, x_rows, F):
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import spmm_raw

    rng = np.random.default_rng(4)
    rp = np.arange(0, 4001 * 6, 6, dtype=np.int32)[:4001]
    ci = rng.integers(0, x_rows, int(rp[-1])).astype(np.int32)
    st = plan_structure(rp, ci, x_rows, dev, chunk=256)
    x = torch.randn(x_rows, F, device=dev)
    y = spmm_raw(st, None, x)
    P = expected_auto_panels(x_rows * F * 4, F)
    if torch.cuda.get_device_properties(0).L2_cache_size == 50 << 20:   # H100 SXM
        assert P == {(169343, 128): 2}.get((x_rows, F), 1)
    note = _cabi.last_kernel()
    assert (f",panels={P}" in note) if P > 1 else ("panels=" not in note), note
    assert torch.equal(bits(y), bits(spmm_raw(st, None, x, panels=1)))


def test_arxiv_shape_automatic_equals_single_pass(dev):
    import cogdl_b200
    from cogdl_b200 import _cabi, synth
    from cogdl_b200.operators._raw import spmm_raw

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, self_loops=True)
    w = synth.sym_norm_weights(rp, col).to(dev)
    st = cogdl_b200.CSRStructure.from_int64(rp.to(dev), col.to(dev), n_cols=n)
    x = torch.randn(n, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(0))
    y = spmm_raw(st, w, x)
    assert ",panels=" in _cabi.last_kernel()
    assert torch.equal(bits(y), bits(spmm_raw(st, w, x, panels=1)))

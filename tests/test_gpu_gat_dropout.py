"""Fused GAT with attention dropout on the GPU: the dropout entry points against the fp64 restatement with the
numpy-regenerated mask (tests/gat_dropout_ref.py), the sign-bit carrier, bit identity at p = 0 and in eval mode,
reproducibility, argument errors, and the reference GAT through install(gat=True) (tests/gat_refpkg_check.py)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.gat_dropout_ref import drop_below, gat_attention_fp64, gat_dropout_fp64, keep_mask
from tests.gpu_util import dev, plan_structure, rel
from tests.graphs import case

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "gat_dropout.npz")
TOL = 1e-5
# (graph, chunk_edges): hub rows split into 16- and 64-edge chunks, 30 % degree-0 rows, no plan at all (warp kernels)
GRAPHS = [("hub", 16), ("hub", 256), ("two_hubs", 64), ("ragged", 256), ("ragged", 0), ("tiny", 0)]
# (H, F): the widths of the existing GAT tests; F = 8 at H = 1 takes the narrow-group gather, H = 3 the generic softmax
SHAPES = [(8, 16), (8, 128), (1, 64), (1, 8), (3, 5)]


def inputs(name, H, F, dev, seed=12):
    rp, ci, n = case(name)
    rng = np.random.default_rng(seed)
    h_l = torch.from_numpy(rng.standard_normal((n, H)).astype(np.float32)).to(dev)
    h_r = torch.from_numpy(rng.standard_normal((n, H)).astype(np.float32)).to(dev)
    feat = torch.from_numpy(rng.standard_normal((n, H, F)).astype(np.float32)).to(dev)
    return rp, ci, n, h_l, h_r, feat


def signbits(att):
    return (att.contiguous().view(torch.int32) < 0).cpu().numpy()


def drop_args(seed, p):
    return (seed, drop_below(p), 1.0 / (1.0 - p))


@pytest.mark.parametrize("name,chunk", GRAPHS)
@pytest.mark.parametrize("H,F", SHAPES)
def test_p0_through_dropout_entry_points_is_bit_identical(dev, name, chunk, H, F):
    from cogdl_b200.operators._raw import gat_attn_bwd_raw, gat_fwd_raw, mhsddmm_raw, mhspmm_raw

    rp, ci, n, h_l, h_r, feat = inputs(name, H, F, dev)
    st = plan_structure(rp, ci, n, dev, chunk=chunk)
    out0, att0 = gat_fwd_raw(st, h_l, h_r, feat, 0.2, True)
    out1, att1 = gat_fwd_raw(st, h_l, h_r, feat, 0.2, True, drop=drop_args(987654321, 0.0))
    assert torch.equal(out0, out1) and torch.equal(att0, att1)
    g = torch.randn(n, H, F, device=dev)
    st_t, perm = st.csc()
    assert torch.equal(mhspmm_raw(st_t, att0, g, perm=perm), mhspmm_raw(st_t, att1, g, perm=perm, drop_scale=1.0))
    d_att = mhsddmm_raw(st, g, feat)
    de0, gr0 = gat_attn_bwd_raw(st, att0, d_att, h_l, h_r, 0.2)
    de1, gr1 = gat_attn_bwd_raw(st, att1, d_att, h_l, h_r, 0.2, drop_scale=1.0)
    assert torch.equal(de0, de1) and torch.equal(gr0, gr1)


@pytest.mark.parametrize("name,chunk", GRAPHS)
@pytest.mark.parametrize("H,F", SHAPES)
@pytest.mark.parametrize("p", [0.5, 0.1, 0.9])
def test_forward_and_mask_vs_fp64(dev, name, chunk, H, F, p):
    from cogdl_b200.operators._raw import gat_fwd_raw

    rp, ci, n, h_l, h_r, feat = inputs(name, H, F, dev)
    st = plan_structure(rp, ci, n, dev, chunk=chunk)
    seed = 0xABCDEF0123 + 7 * H + F
    out, att = gat_fwd_raw(st, h_l, h_r, feat, 0.2, True, drop=drop_args(seed, p))
    keep = keep_mask(seed, ci.size, H, p)
    # the mask travels in the sign bits of the saved attention, exactly where the numpy keep rule puts it
    sb = signbits(att)
    assert int(sb.sum()) == int((~keep).sum())
    assert np.array_equal(sb, ~keep)
    a64 = gat_attention_fp64(rp, ci, h_l.double().cpu(), h_r.double().cpu(), 0.2).numpy()
    assert rel(att.abs().cpu().numpy(), a64) <= TOL
    ref = gat_dropout_fp64(rp, ci, h_l.double().cpu(), h_r.double().cpu(), feat.double().cpu(), 0.2, keep, p)
    assert out.shape == ref.shape
    assert rel(out.cpu().numpy(), ref.numpy()) <= TOL
    if n > 0 and (np.diff(rp) == 0).any():
        assert torch.all(out[torch.from_numpy(np.diff(rp) == 0).to(dev)] == 0)


@pytest.mark.parametrize("name,chunk", GRAPHS)
@pytest.mark.parametrize("H,F", SHAPES)
def test_gradients_vs_fp64_autograd(dev, name, chunk, H, F):
    from cogdl_b200.operators.fused_gat import FusedGATFunction

    p, seed = 0.5, 4242 + H
    rp, ci, n, h_l, h_r, feat = inputs(name, H, F, dev)
    st = plan_structure(rp, ci, n, dev, chunk=chunk)
    xs = [t.clone().requires_grad_(True) for t in (h_l, h_r, feat)]
    out = FusedGATFunction.apply(xs[0], xs[1], st, None, None, None, 0.2, xs[2], p, seed)
    G = torch.randn_like(out)
    out.backward(G)
    keep = keep_mask(seed, ci.size, H, p)
    ys = [t.double().cpu().requires_grad_(True) for t in (h_l, h_r, feat)]
    ref = gat_dropout_fp64(rp, ci, ys[0], ys[1], ys[2], 0.2, keep, p)
    ref.backward(G.double().cpu())
    assert rel(out.detach().cpu().numpy(), ref.detach().numpy()) <= TOL
    assert rel(xs[2].grad.cpu().numpy(), ys[2].grad.numpy()) <= TOL                    # d feat: CSC pass, perm fused
    # d h_l / d h_r are row / column sums of the per-edge logit gradients, which cancel (exactly, for a row whose
    # logits share one LeakyReLU branch at H = 1): their error is scaled by the fp64 sums of |per-edge gradient|,
    # obtained by giving every edge its own column
    cols = torch.from_numpy(ci.astype(np.int64))
    hr_e = ys[1].detach()[cols].requires_grad_(True)
    gat_dropout_fp64(rp, np.arange(ci.size), ys[0].detach(), hr_e, ys[2].detach()[cols], 0.2, keep, p).backward(
        G.double().cpu())
    d_e = hr_e.grad.abs()
    rows = torch.repeat_interleave(torch.arange(n), torch.from_numpy(np.diff(rp).astype(np.int64)))
    for got, want, idx in ((xs[0], ys[0], rows), (xs[1], ys[1], cols)):               # softmax bwd after fp32 mhsddmm
        scale = torch.zeros_like(want.grad).index_add_(0, idx, d_e).clamp_min(want.grad.abs())
        err = (got.grad.cpu().double() - want.grad).abs().max() / max(float(scale.max()), 1e-30) if n else 0.0
        assert err <= 2e-5


def test_fused_layer_with_the_golden_seed_matches_reference_layer(dev):
    """The reference GATLayer's CPU output with the keep rule's mask (tests/golden/gat_dropout.npz) against the fused
    operator called with the same seed."""
    import cogdl_b200

    gd = np.load(GOLDEN)
    graph = cogdl_b200.Graph(row_ptr=torch.from_numpy(gd["rowptr"]).to(dev), col=torch.from_numpy(gd["col"]).to(dev),
                             num_nodes=gd["x"].shape[0])
    x = torch.from_numpy(gd["x"]).to(dev)
    for key in ("h8", "h1"):
        W, a_l, a_r = (torch.from_numpy(gd[f"{k}_{key}"]).to(dev) for k in ("W", "a_l", "a_r"))
        h = (x @ W).view(x.shape[0], a_l.shape[1], a_l.shape[2])
        h_l, h_r = (a_l * h).sum(dim=-1), (a_r * h).sum(dim=-1)
        y = cogdl_b200.fused_gat_op(h_l, h_r, graph, float(gd["slope"]), h, attn_drop=float(gd["p"]),
                                    seed=int(gd[f"seed_{key}"]))
        assert rel(y.reshape(y.shape[0], -1).cpu().numpy(), gd[f"y_{key}"]) <= 2 * TOL, key


def _fused_layer(dev, attn_drop):
    from cogdl_b200.layers import GATLayer

    torch.manual_seed(0)
    a = GATLayer(24, 16, nhead=8, attn_drop=attn_drop, fused=True).to(dev)
    return a


def _graph(dev, name="two_hubs"):
    import cogdl_b200

    rp, ci, n = case(name)
    return cogdl_b200.Graph(row_ptr=torch.from_numpy(rp.astype(np.int64)).to(dev),
                            col=torch.from_numpy(ci.astype(np.int64)).to(dev), num_nodes=n), n


def test_training_is_reproducible_under_manual_seed_and_seeds_differ(dev):
    gr, n = _graph(dev)
    layer = _fused_layer(dev, 0.5).train()
    x = torch.randn(n, 24, device=dev)
    G = torch.randn(n, 8 * 16, device=dev)

    def step(seed):
        layer.zero_grad()
        torch.manual_seed(seed)
        y = layer(gr, x)
        y.backward(G)
        return y.detach().clone(), [p.grad.clone() for p in layer.parameters()]

    y1, g1 = step(3)
    y2, g2 = step(3)
    assert torch.equal(y1, y2) and all(torch.equal(a, b) for a, b in zip(g1, g2))
    y3, _ = step(4)
    assert not torch.equal(y1, y3)
    # without reseeding, every call draws a fresh mask
    torch.manual_seed(3)
    assert not torch.equal(layer(gr, x), layer(gr, x))


def test_eval_and_p0_are_bit_identical_to_the_plain_fused_op(dev):
    gr, n = _graph(dev)
    x = torch.randn(n, 24, device=dev)
    drop = _fused_layer(dev, 0.5)
    plain = _fused_layer(dev, 0.0)
    plain.load_state_dict(drop.state_dict())
    drop.eval(), plain.eval()
    assert torch.equal(drop(gr, x), plain(gr, x))
    plain.train()
    ya = plain(gr, x)
    from cogdl_b200.operators.fused_gat import FusedGATFunction

    h = torch.matmul(x, plain.W).view(-1, 8, 16)
    h_l, h_r = (plain.a_l * h).sum(dim=-1), (plain.a_r * h).sum(dim=-1)
    yb = FusedGATFunction.apply(h_l, h_r, gr.structure(), None, None, None, 0.2, h).view(n, -1)
    assert torch.equal(ya, yb)


def test_kernel_names_list_every_launch_with_the_dropout_flag(dev):
    """The attention backward names the statistics kernel and the main kernel it launched, the GAT forward its
    attention launches and then the aggregation; each instantiation carries the dropout flag."""
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import gat_attn_bwd_raw, gat_fwd_raw, mhsddmm_raw

    rp, ci, n, h_l, h_r, feat = inputs("hub", 8, 128, dev)
    st = plan_structure(rp, ci, n, dev, chunk=256)
    _, att = gat_fwd_raw(st, h_l, h_r, feat, 0.2, True, drop=drop_args(1, 0.5))
    assert _cabi.last_kernel() == ("cogdl_b200::es_stats_kernel<MODE=2> + cogdl_b200::es_main_kernel<MODE=2,CAP=2048,WARPS=8,DROP>"
                                   " + cogdl_b200::stream_kernel<float4,NV=1,multihead+drop,SRC_ONE,U=8,MINB=3,prefetch>"
                                   " block=128")
    d_att = mhsddmm_raw(st, torch.randn(n, 8, 128, device=dev), feat)
    gat_attn_bwd_raw(st, att, d_att, h_l, h_r, 0.2, drop_scale=2.0)
    assert _cabi.last_kernel() == ("cogdl_b200::es_stats_kernel<MODE=3,DROP> + "
                                   "cogdl_b200::es_main_kernel<MODE=3,CAP=2048,WARPS=8,DROP> cp.async.bulk tiles")
    rp1, ci1, n1, hl1, hr1, f1 = inputs("hub", 1, 8, dev)
    gat_fwd_raw(plan_structure(rp1, ci1, n1, dev, chunk=256), hl1, hr1, f1, 0.2, True, drop=drop_args(1, 0.5))
    assert _cabi.last_kernel() == ("cogdl_b200::es_stats_kernel<MODE=2> + cogdl_b200::es_main_kernel<MODE=2,CAP=512,WARPS=8,DROP>"
                                   " + cogdl_b200::mhspmm_kernel<float4,GROUP=2,no_perm,drop>")


def test_bad_arguments_raise_the_library_error(dev):
    import cogdl_b200
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import _scratch
    from cogdl_b200.structure import _ptr, _stream

    rp, ci, n, h_l, h_r, feat = inputs("tiny", 8, 16, dev)
    st = plan_structure(rp, ci, n, dev, chunk=256)
    out = torch.empty(n, 8, 16, device=dev)
    att = torch.empty(ci.size, 8, device=dev)
    plan, keep = st.plan_struct(_scratch("gat_fwd", st, 8, 16))
    fwd = ("cogdl_b200_gat_fwd_dropout_f32", _ptr(st.rowptr), _ptr(st.colind), _ptr(h_l), _ptr(h_r), _ptr(feat), 0.2,
           1, 2 ** 63)
    for scale in (0.0, -1.0, float("inf"), float("nan")):
        with pytest.raises(_cabi.CogdlB200Error) as e:
            _cabi.call(*fwd, scale, _ptr(out), _ptr(att), n, 8, 16, plan, _stream(dev))
        assert e.value.code == _cabi.EINVAL
        with pytest.raises(_cabi.CogdlB200Error) as e:
            _cabi.call("cogdl_b200_mhspmm_dropout_f32", _ptr(st.rowptr), _ptr(st.colind), None, _ptr(att), _ptr(feat),
                       scale, _ptr(out), n, 8, 16, plan, _stream(dev))
        assert e.value.code == _cabi.EINVAL
        with pytest.raises(_cabi.CogdlB200Error) as e:
            _cabi.call("cogdl_b200_gat_attn_bwd_dropout_f32", _ptr(st.rowptr), _ptr(st.colind), _ptr(att), _ptr(att),
                       _ptr(h_l), _ptr(h_r), 0.2, scale, _ptr(att), _ptr(h_l), n, 8, plan, _stream(dev))
        assert e.value.code == _cabi.EINVAL
    with pytest.raises(_cabi.CogdlB200Error) as e:
        _cabi.call(*fwd, 2.0, _ptr(out), None, n, 8, 16, plan, _stream(dev))
    assert e.value.code == _cabi.EINVAL
    del keep
    gr, _ = _graph(dev, "tiny")
    for p in (1.0, 1.5, -0.5):
        with pytest.raises(ValueError):
            cogdl_b200.fused_gat_op(h_l, h_r, gr, 0.2, feat, attn_drop=p)
    with pytest.raises(RuntimeError):
        cogdl_b200.fused_gat_op(h_l.cpu(), h_r.cpu(), gr, 0.2, feat.cpu(), attn_drop=0.5)


def test_reference_gat_through_install():
    """The reference GAT (attn_drop 0.5) through install(gat=True), in a child process (tests/gat_refpkg_check.py)."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.gat_refpkg_check"], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["untouched_without_flag"], "install() without gat=True must leave GATLayer.forward alone"
    assert res["rebound"] and res["patched"][-1] == "cogdl.layers.gat_layer.GATLayer.forward", res
    assert res["losses_finite"] and res["loss_decreases"], res
    assert res["reproducible"], res
    assert res["seed_changes_mask"], res
    assert res["eval_vs_unfused"] <= TOL, res
    assert res["uncovered_ran_original"] == ["cpu", "half", "p1"], res
    assert res["restored"], res

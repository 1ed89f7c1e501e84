"""Activation compression (actnn.cu) on the GPU against the numpy restatement (tests/actnn_ref.py): codes, packed
bytes, scales, dequantized values, masks and allocated bits bit-identical; the allocation against the reference greedy's
golden output at an arxiv-sized N; stochastic rounding seeded and unbiased; spmm(actnn=True); and the reference
ActGCN / GCNII / GraphSAGE through install(actnn=True) (tests/actnn_refpkg_check.py)."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests import actnn_ref as R

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
DEV = torch.device("cuda:0")


def K():
    from cogdl_b200.actnn import kernels

    return kernels


def bits_for(kind, N, rng):
    if kind == "mixed":
        return rng.integers(1, 9, N).astype(np.int32)
    return int(kind)


def to_dev_bits(bits):
    return torch.from_numpy(bits).to(DEV) if isinstance(bits, np.ndarray) else bits


SHAPES = [(0, 64), (1, 1), (1, 100), (37, 300), (64, 256), (129, 70)]


@pytest.mark.parametrize("gs", [64, 256])
@pytest.mark.parametrize("kind", ["1", "2", "4", "8", "mixed"])
@pytest.mark.parametrize("shape", SHAPES)
def test_pack_unpack_bit_identical(gs, kind, shape):
    import cogdl_b200

    N, D = shape
    rng = np.random.default_rng(N * 1000 + D + gs)
    x = (rng.standard_normal((N, D)) * rng.random((N, 1)) * 4).astype(np.float32)
    bits = bits_for(kind, N, rng)
    packed, scale, mn = K().pack(torch.from_numpy(x).to(DEV), to_dev_bits(bits), gs, False)
    kernel = cogdl_b200._cabi.last_kernel()
    assert kernel == (f"actnn_pack_mixed<{gs}>" if kind == "mixed" else f"actnn_pack<{gs}>")
    codes, rscale, rmn = R.quantize(x, bits, gs)
    assert np.array_equal(packed.cpu().numpy(), R.pack(codes, bits))
    assert np.array_equal(scale.float().cpu().numpy(), rscale)
    assert np.array_equal(mn.float().cpu().numpy(), rmn)
    out = K().unpack(packed, to_dev_bits(bits), scale, mn, N, D, gs)
    assert np.array_equal(out.cpu().numpy(), R.dequantize(codes, rscale, rmn, D, gs))
    if N:
        gmn, gmx = K().group_minmax(torch.from_numpy(x).to(DEV), gs)
        Dp = -(-D // gs) * gs
        xp = np.zeros((N, Dp), np.float32)
        xp[:, :D] = x
        assert np.array_equal(gmn.cpu().numpy(), xp.reshape(N, -1, gs).min(2))
        assert np.array_equal(gmx.cpu().numpy(), xp.reshape(N, -1, gs).max(2))


def test_unaligned_input_and_stochastic_rounding_bit_identical():
    rng = np.random.default_rng(1)
    buf = torch.from_numpy(rng.standard_normal(33 * 130 + 1).astype(np.float32)).to(DEV)
    x = buf[1:].view(33, 130)                      # 4-byte aligned only
    bits = rng.integers(1, 9, 33).astype(np.int32)
    for gs in (64, 256):
        packed, scale, mn = K().pack(x, to_dev_bits(bits), gs, True, seed=123)
        codes, rs, rm = R.quantize(x.cpu().numpy(), bits, gs, stochastic=True, seed=123)
        assert np.array_equal(packed.cpu().numpy(), R.pack(codes, bits))
        again = K().pack(x, to_dev_bits(bits), gs, True, seed=123)[0]
        assert torch.equal(packed, again)
        assert not torch.equal(packed, K().pack(x, to_dev_bits(bits), gs, True, seed=124)[0])


def test_stochastic_rounding_is_unbiased():
    rng = np.random.default_rng(2)
    x = torch.from_numpy(rng.standard_normal((256, 256)).astype(np.float32)).to(DEV)
    errs = []
    for s in range(256):
        p, sc, mn = K().pack(x, 2, 256, True, seed=1000 + s)
        errs.append(K().unpack(p, 2, sc, mn, 256, 256, 256) - x)
    one = errs[0].abs().mean().item()
    mean = torch.stack(errs).mean(0).abs().mean().item()
    assert mean <= one / 8, (mean, one)


@pytest.mark.parametrize("n", [0, 1, 31, 32, 33, 100000])
def test_relu_and_dropout_masks_bit_identical(n):
    rng = np.random.default_rng(n)
    x = rng.standard_normal(n).astype(np.float32)
    g = rng.standard_normal(n).astype(np.float32)
    xd, gd = torch.from_numpy(x).to(DEV), torch.from_numpy(g).to(DEV)
    y, m = K().relu_fwd(xd)
    ry, rm = R.relu(x)
    assert np.array_equal(y.cpu().numpy(), ry) and np.array_equal(m.cpu().numpy(), rm)
    assert np.array_equal(K().relu_bwd(gd, m).cpu().numpy(), np.where(x > 0, g, np.float32(0)))
    for p in (0.0, 0.1, 0.5, 0.9):
        y, m = K().dropout_fwd(xd, p, 77)
        ry, rm = R.dropout(x, p, 77)
        assert np.array_equal(y.cpu().numpy(), ry) and np.array_equal(m.cpu().numpy(), rm)
        rg = R.dropout(g, p, 77)[0]
        assert np.array_equal(K().dropout_bwd(gd, m, p).cpu().numpy(), rg)


def _gold():
    return np.load(os.path.join(ROOT, "tests", "golden", "actnn.npz"))


@pytest.mark.parametrize("name", ["random", "zeros", "dups", "frac", "allzero", "large", "arxiv"])
def test_bit_allocation_equals_reference_greedy(name):
    from tests.test_cpu_actnn_golden import alloc_case

    C, target, want = alloc_case(_gold(), name)
    got = K().allocate_bits(torch.from_numpy(C).to(DEV), target)
    assert np.array_equal(got.cpu().numpy(), want)


@pytest.mark.parametrize("b0", [8, 5, 2, 1])
def test_bit_allocation_other_initial_bits_and_targets(b0):
    rng = np.random.default_rng(b0)
    C = (rng.random(5000) * rng.choice([0, 1, 3], 5000)).astype(np.float32)
    for target in (0, 5000, 12345, b0 * 5000, 10 ** 9):
        got = K().allocate_bits(torch.from_numpy(C).to(DEV), target, b0).cpu().numpy()
        assert np.array_equal(got, R.alloc_topk(C, target, b0)), (b0, target)
    assert K().allocate_bits(torch.zeros(0, device=DEV), 0).numel() == 0


def test_bit_allocation_rejects_bad_C():
    from cogdl_b200._cabi import CogdlB200Error

    for bad in (float("nan"), float("inf"), -1.0):
        C = torch.ones(100, device=DEV)
        C[17] = bad
        with pytest.raises(CogdlB200Error, match="finite"):
            K().allocate_bits(C, 200)


def test_spmm_actnn_matches_plain_and_gives_weight_gradient():
    import cogdl_b200
    from cogdl_b200 import synth
    from cogdl_b200.actnn import config

    rp, col = synth.powerlaw_csr(2000, 20000, seed=3)
    w = synth.sym_norm_weights(rp, col)
    g = cogdl_b200.Graph(x=torch.randn(2000, 64), row_ptr=rp, col=col, edge_weight=w).to(DEV)
    x = torch.randn(2000, 64, device=DEV)
    assert torch.equal(cogdl_b200.spmm(g, x, actnn=True), cogdl_b200.spmm(g, x))
    st = g.structure()
    old = config.activation_compression_bits, config.stochastic
    config.activation_compression_bits, config.stochastic = [8], False
    try:
        grads = []
        for act in (False, True):
            wt = g.raw_edge_weight.detach().clone().requires_grad_(True)
            xt = x.clone().requires_grad_(True)
            cogdl_b200.csrspmm(st, None, xt, wt, False, actnn=act).square().sum().backward()
            grads.append((xt.grad, wt.grad))
    finally:
        config.activation_compression_bits, config.stochastic = old
    assert torch.equal(grads[0][0], grads[1][0])
    assert float((grads[0][1] - grads[1][1]).norm() / grads[0][1].norm()) < 1e-2


def test_reference_models_through_install():
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.actnn_refpkg_check"], cwd=ROOT, capture_output=True, text=True,
                       timeout=1800)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    print(json.dumps(res))
    assert res["stand_in"] and "actnn" in res["patched"], res
    for name in ("gcn", "gcnii", "sage"):
        assert res[f"{name}_forward_equal"], res
        assert res[f"{name}_grad8_rel"] <= 1e-2, res
        assert res[f"{name}_grad2_avg_rel"] * 4 <= res[f"{name}_grad2_one_rel"], res
    assert res["saved_ratio"] <= 1 / 8, res
    assert res["uninstalled"], res

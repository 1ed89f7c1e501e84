"""Sparse x sparse product (cogdl_b200/csrc/spgemm.cu), SpSpMMFunction, spspmm and coo_spmm against the sequential
restatement of tests/spgemm_oracle.py (itself checked against scipy by test_cpu_spgemm_oracle.py) and fp64 autograd."""
import json
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from tests.gpu_util import dev
from tests import graphs
from tests import spgemm_oracle as so

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def coo_of(rp, ci, seed, shuffle=True):
    """(row, col, val) numpy COO of a CSR, shuffled, with random fp32 values."""
    rng = np.random.default_rng(seed)
    row = np.repeat(np.arange(rp.size - 1), np.diff(rp))
    perm = rng.permutation(row.size) if shuffle else np.arange(row.size)
    val = rng.standard_normal(row.size).astype(np.float32)
    return row[perm].astype(np.int64), np.asarray(ci)[perm].astype(np.int64), val


def to_dev(row, col, val, dev):
    return (torch.from_numpy(np.stack([row, col])).to(dev), torch.from_numpy(val).to(dev))


def run_and_check(A, B, m, k, n, dev, coalesced=False):
    """spspmm on the device against the oracle on the coalesced inputs: the pattern exactly, the values bit for bit."""
    import cogdl_b200

    (ra, ca, va), (rb, cb, vb) = A, B
    ia, xa = to_dev(ra, ca, va, dev)
    ib, xb = to_dev(rb, cb, vb, dev)
    idx, val = cogdl_b200.spspmm(ia, xa, ib, xb, m, k, n, coalesced)
    pa, qa, wa = so.coalesce(ra, ca, va, m, k)
    pb, qb, wb = so.coalesce(rb, cb, vb, k, n)
    rp, col, want = so.spgemm(pa, qa, wa, pb, qb, wb, n)
    row = np.repeat(np.arange(m), np.diff(rp))
    got_idx = idx.cpu().numpy()
    assert got_idx.dtype == np.int64 and got_idx.shape == (2, col.size)
    assert np.array_equal(got_idx[0], row) and np.array_equal(got_idx[1], col)
    got = val.cpu().numpy()
    assert got.dtype == np.float32
    assert np.array_equal(got.view(np.int32), want.view(np.int32)), float(np.abs(got - want).max())
    return idx, val


def transpose(rp, ci, n_cols):
    row = np.repeat(np.arange(rp.size - 1), np.diff(rp))
    order = np.lexsort((row, ci))
    rpt = np.zeros(n_cols + 1, np.int64)
    np.cumsum(np.bincount(ci, minlength=n_cols), out=rpt[1:])
    return rpt, row[order]


@pytest.mark.parametrize("name", sorted(graphs.CASES))
def test_forward_bit_identical_every_graph(dev, name):
    rp, ci, n_cols = graphs.case(name)
    n = rp.size - 1
    A = coo_of(rp, ci, 1)
    rpt, cit = transpose(rp, ci, n_cols)
    At = coo_of(rpt, cit, 2)
    if n == n_cols:
        run_and_check(A, coo_of(rp, ci, 3), n, n, n, dev)                 # A . A
    run_and_check(A, At, n, n_cols, n, dev)                                 # A . A^T
    run_and_check(At, A, n_cols, n, n_cols, dev, coalesced=True)           # A^T . A


def test_duplicates_unsorted_and_rectangular(dev):
    rng = np.random.default_rng(5)
    m, k, n = 300, 170, 410
    ra, ca = rng.integers(0, m, 2500), rng.integers(0, k, 2500)
    ra, ca = np.concatenate([ra, ra[:600]]), np.concatenate([ca, ca[:600]])   # 600 duplicated entries
    rb, cb = rng.integers(0, k, 3000), rng.integers(0, n, 3000)
    va, vb = rng.standard_normal(ra.size).astype(np.float32), rng.standard_normal(rb.size).astype(np.float32)
    run_and_check((ra, ca, va), (rb, cb, vb), m, k, n, dev)
    run_and_check((ra, ca, va), (rb, cb, vb), m, k, n, dev, coalesced=True)


def test_dense_hub_row_reaches_the_bitmap_tier(dev):
    """One output row covering all of n = 120 000 columns (the bitmap bin), beside rows of the block bin."""
    k, n, width = 400, 120_000, 300
    rb = np.repeat(np.arange(k), width)
    cb = (np.arange(k)[:, None] * width + np.arange(width)[None, :]).ravel()
    rng = np.random.default_rng(6)
    ra = [np.zeros(k, np.int64)]                   # row 0: every row of B
    ca = [np.arange(k)]
    for i in range(1, 200):                        # the rest: 1 to 20 rows of B
        d = int(rng.integers(1, 21))
        ra.append(np.full(d, i))
        ca.append(rng.choice(k, d, replace=False))
    ra, ca = np.concatenate(ra), np.concatenate(ca)
    va, vb = rng.standard_normal(ra.size).astype(np.float32), rng.standard_normal(rb.size).astype(np.float32)
    idx, _ = run_and_check((ra, ca, va), (rb, cb, vb), 200, k, n, dev)
    assert int((idx[0] == 0).sum()) == n


def test_arxiv_shaped_square(dev):
    import cogdl_b200
    from cogdl_b200 import synth

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, self_loops=True)
    rp, col = rp.numpy(), col.numpy()
    A = coo_of(rp, col, 7, shuffle=False)
    idx, val = run_and_check(A, A, n, n, n, dev)
    assert cogdl_b200._cabi.last_kernel().startswith("cogdl_b200::spg_fill")
    assert idx.shape[1] > 5 * col.size


def dense_product_grads(A, B, m, k, n, G):
    """fp64 dense autograd of sum(G * (A B)) at the structural pattern: (d valueA, d valueB) per input entry."""
    (ra, ca, va), (rb, cb, vb) = A, B
    xa = torch.from_numpy(va).double().requires_grad_(True)
    xb = torch.from_numpy(vb).double().requires_grad_(True)
    Ad = torch.zeros(m, k, dtype=torch.float64).index_put((torch.from_numpy(ra), torch.from_numpy(ca)), xa, accumulate=True)
    Bd = torch.zeros(k, n, dtype=torch.float64).index_put((torch.from_numpy(rb), torch.from_numpy(cb)), xb, accumulate=True)
    C = Ad @ Bd
    (C * G).sum().backward()
    return C.detach(), xa.grad, xb.grad


def test_value_gradients_against_fp64(dev):
    import cogdl_b200

    rng = np.random.default_rng(8)
    m, k, n = 60, 45, 70
    ra, ca = rng.integers(0, m, 500), rng.integers(0, k, 500)
    ra, ca = np.concatenate([ra, ra[:80]]), np.concatenate([ca, ca[:80]])
    rb, cb = rng.integers(0, k, 400), rng.integers(0, n, 400)
    rb, cb = np.concatenate([rb, rb[:50]]), np.concatenate([cb, cb[:50]])
    A = (ra, ca, rng.standard_normal(ra.size).astype(np.float32))
    B = (rb, cb, rng.standard_normal(rb.size).astype(np.float32))
    ia, xa = to_dev(*A, dev)
    ib, xb = to_dev(*B, dev)
    xa.requires_grad_(True)
    xb.requires_grad_(True)
    idx, val = cogdl_b200.spspmm(ia, xa, ib, xb, m, k, n)
    G = torch.randn(m, n, dtype=torch.float64, generator=torch.Generator().manual_seed(3))
    gi = idx.cpu()
    (val * G[gi[0], gi[1]].float().to(dev)).sum().backward()
    C, da, db = dense_product_grads(A, B, m, k, n, G)
    assert torch.allclose(val.double().cpu(), C[gi[0], gi[1]], rtol=1e-5, atol=1e-5)
    for got, want in ((xa.grad, da), (xb.grad, db)):
        err = (got.double().cpu() - want).abs().max() / want.abs().max()
        assert float(err) <= 1e-5
    # merged duplicates: both copies of an entry get their slot's gradient
    assert torch.equal(xa.grad[:80], xa.grad[500:580])


def test_bitwise_reproducible(dev):
    import cogdl_b200

    rp, ci, _ = graphs.case("two_hubs")
    n = rp.size - 1
    A = coo_of(rp, ci, 9)
    outs = []
    for _ in range(2):
        ia, xa = to_dev(*A, dev)
        xa.requires_grad_(True)
        xb = xa.detach().clone().requires_grad_(True)
        idx, val = cogdl_b200.spspmm(ia, xa, ia, xb, n, n, n)
        val.backward(torch.linspace(-1, 1, val.numel(), device=dev))
        outs.append((idx, val.detach(), xa.grad, xb.grad))
    for a, b in zip(*outs):
        assert torch.equal(a, b)


def test_nnz_overflow_is_an_argument_error(dev):
    """A symmetric star with 50 000 leaves, squared: about 2.5e9 entries, more than int32 CSR holds."""
    import cogdl_b200
    from cogdl_b200 import _cabi

    L = 50_000
    leaves = torch.arange(1, L + 1, device=dev)
    hub = torch.zeros(L, dtype=torch.int64, device=dev)
    idx = torch.stack([torch.cat([hub, leaves]), torch.cat([leaves, hub])])
    val = torch.ones(2 * L, device=dev)
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(dev)
    with pytest.raises(_cabi.CogdlB200Error) as ei:
        cogdl_b200.spspmm(idx, val, idx, val, L + 1, L + 1, L + 1)
    assert ei.value.code == _cabi.EINVAL and "int32" in str(ei.value)
    assert torch.cuda.memory_allocated(dev) - before < 64 << 20      # nothing the size of C was allocated


def test_index_errors_cpu_input_and_kernel_names(dev):
    import cogdl_b200
    from cogdl_b200 import _cabi

    ia = torch.tensor([[0, 1], [1, 2]], device=dev)
    v = torch.ones(2, device=dev)
    n0 = _cabi.launch_count()
    with pytest.raises(ValueError, match="out of range"):
        cogdl_b200.spspmm(ia, v, ia, v, 2, 2, 3)            # column 2 of A outside k = 2
    with pytest.raises(ValueError, match="out of range"):
        cogdl_b200.coo_spmm(torch.tensor([[0, -1], [0, 0]], device=dev), v, 2, 2, torch.ones(2, 4, device=dev))
    assert _cabi.launch_count() == n0, "an index error is raised before any launch of this library"
    with pytest.raises(ValueError, match="out of range"):
        cogdl_b200.spspmm(ia, v, torch.tensor([[0, 5], [0, 0]], device=dev), v, 2, 3, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        cogdl_b200.spspmm(ia.cpu(), v.cpu(), ia.cpu(), v.cpu(), 3, 3, 3)
    with pytest.raises(RuntimeError, match="CUDA"):
        cogdl_b200.coo_spmm(ia.cpu(), v.cpu(), 3, 3, torch.ones(3, 2))
    idx, val = cogdl_b200.spspmm(ia, v, ia, v, 3, 3, 3)
    assert _cabi.last_kernel() == "cogdl_b200::spg_fill<warp=256,block=4096,bitmap>"
    # the C ABI's own checks: a B whose row count is not A's column count
    lib = _cabi.load()
    rp = torch.zeros(4, dtype=torch.int32, device=dev)
    from cogdl_b200.structure import _ptr, _stream

    nnz = _cabi.ctypes.c_int64(0)
    assert lib.cogdl_b200_spgemm_bwd_f32(_ptr(rp), _ptr(rp), None, 3, 3, _ptr(rp), _ptr(rp), _ptr(v), 3, 3, _ptr(rp),
                                         _ptr(rp), _ptr(v), None, None, None, _ptr(v), None, _stream(dev)) == _cabi.OK
    assert _cabi.last_kernel() == "cogdl_b200::spg_dA_kernel"
    rc = lib.cogdl_b200_spgemm_count(_ptr(rp), _ptr(rp), 3, 3, _ptr(rp), _ptr(rp), 2, 3, _ptr(rp), _cabi.ctypes.byref(nnz),
                                     _ptr(rp), 1 << 20, _stream(dev))
    assert rc == _cabi.EINVAL and "B has 2 rows" in _cabi.last_error()
    rc = lib.cogdl_b200_spgemm_count(_ptr(rp), None, 3, 3, _ptr(rp), _ptr(rp), 3, 3, _ptr(rp), _cabi.ctypes.byref(nnz),
                                     _ptr(rp), 1 << 20, _stream(dev))
    assert rc == _cabi.EINVAL and "null pointer" in _cabi.last_error()
    rc = lib.cogdl_b200_spgemm_count(_ptr(rp), _ptr(rp), -1, 3, _ptr(rp), _ptr(rp), 3, 3, _ptr(rp),
                                     _cabi.ctypes.byref(nnz), _ptr(rp), 1 << 20, _stream(dev))
    assert rc == _cabi.EINVAL and "negative size" in _cabi.last_error()


def test_coo_spmm_against_fp64(dev):
    import cogdl_b200

    rng = np.random.default_rng(10)
    m, n, F = 120, 90, 33
    row, col = rng.integers(0, m, 900), rng.integers(0, n, 900)
    row, col = np.concatenate([row, row[:100]]), np.concatenate([col, col[:100]])
    val = rng.standard_normal(row.size).astype(np.float32)
    index, v = to_dev(row, col, val, dev)
    v.requires_grad_(True)
    X = torch.randn(n, F, device=dev, requires_grad=True)
    out = cogdl_b200.coo_spmm(index, v, m, n, X)
    G = torch.randn(m, F, device=dev)
    (out * G).sum().backward()
    v64 = torch.from_numpy(val).double().requires_grad_(True)
    X64 = X.detach().double().cpu().requires_grad_(True)
    A = torch.zeros(m, n, dtype=torch.float64).index_put((torch.from_numpy(row), torch.from_numpy(col)), v64, accumulate=True)
    ref = A @ X64
    (ref * G.double().cpu()).sum().backward()
    for got, want in ((out, ref), (v.grad, v64.grad), (X.grad, X64.grad)):
        err = (got.detach().double().cpu() - want.detach()).abs().max() / want.detach().abs().max()
        assert float(err) <= 1e-5


def test_structure_cache_reuses_the_index(dev):
    import cogdl_b200
    from cogdl_b200 import structure

    rp, ci, _ = graphs.case("ragged")
    n = rp.size - 1
    ia, xa = to_dev(*coo_of(rp, ci, 11), dev)
    cogdl_b200.spspmm(ia, xa, ia, xa, n, n, n)
    before = dict(structure.coo_cache_stats)
    for _ in range(3):
        cogdl_b200.spspmm(ia, xa * 2, ia, xa, n, n, n)
        cogdl_b200.coo_spmm(ia, xa, n, n, torch.ones(n, 3, device=dev))
    assert structure.coo_cache_stats["miss"] == before["miss"]
    ia[0, 0] = ia[0, 0]                                   # an in-place write: the next call rebuilds
    cogdl_b200.spspmm(ia, xa, ia, xa, n, n, n)
    assert structure.coo_cache_stats["miss"] == before["miss"] + 1


def test_reference_gtn_srgcn_graph_unet_through_install():
    """The reference GTN, SRGCN and Graph U-Net through install(spspmm=True), in a child process
    (tests/spspmm_refpkg_check.py): logits against the reference's CPU run, gradients against fp64, uninstall."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.spspmm_refpkg_check"], cwd=ROOT, capture_output=True, text=True,
                       timeout=1200)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["import_failed_before_install"], res
    assert res["patched"][-1] == "torch_sparse", res
    assert res["gtn_logits_vs_cpu"] <= 1e-5, res
    assert res["gtn_grad_vs_fp64"] <= 1e-4, res
    assert res["gtn_conv_grad_nonzero"], res
    assert res["srgcn_logits_vs_cpu"] <= 1e-5, res
    assert res["srgcn_grad_vs_fp64"] <= 1e-4, res
    assert res["unet_ran"], res
    assert res["unet_aug_adj_error"], res
    assert res["restored"], res

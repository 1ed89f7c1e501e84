"""Graph-level readouts (cogdl_b200.operators.readout) and SortPool's selection kernel (cogdl_b200_sort_pool_select).

- Sum, mean, max and Set2Set over the membership of sorted and unsorted batches, empty graph ids in the middle and at
  the end, B = 1, one-node graphs, graph sizes on the hub-chunk boundaries under hub plans of 16 and 64 edges, and one
  graph of 2 * 10^6 nodes (the hub path), at F in {1, 3, 67, 128, 300}, inputs contiguous, strided and misaligned:
  * sum and mean within (L + 2) 2^-24 sum|terms| of fp64, L the longest accumulation chain of the row (its length, or
    a chunk plus the chunk count on a hub row); rows the plan does not split bit-identical to the oracle's CSR-order
    sum (the mean: times fl(1 / n_g)); max values and argmax exact; Set2Set within its bound; a second run bitwise
    equal, the hub graph included;
  * backward: the sum's dx bit-equal to dy[batch], the mean's within 2 ulps of dy / n_g, max exact, Set2Set's dx and
    dq within the bound.
- sort_pool against the stable fp64 restatement: the selected nodes exactly, the pooled rows and the gradient equal as
  values (the SpMM that moves the rows adds each to 0: -0 comes out as +0, NaN as the canonical NaN): k < n, k = n,
  k > n and n = 0; tied keys; +-Inf, NaN and -0 keys; a 10^5-node graph; an input past 2^31 elements
  (test_sort_pool_past_2_31_elements).
- No host synchronisation after the first call on a batch.
- The reference GIN, InfoGraph encoder, SortPool and pooling functions through install(gin=True, readout=True), in a
  child process (tests/readout_refpkg_check.py).
"""
import json
import math
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest
import torch

import oracle
from tests import readout_ref as R
from tests.gpu_util import T, bits, dev, misaligned, plan_structure  # noqa: F401

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
U = 2.0 ** -24
FS = (1, 3, 67, 128, 300)
HUB_N = 2_000_000


def batch_case(name):
    """(batch [N] int64, B, chunk) of a named batch; chunk is the hub plan's chunk (64 is the library's default)."""
    rng = np.random.default_rng(zlib.crc32(name.encode()))
    if name in ("sorted", "unsorted"):
        b = np.repeat(np.arange(20), rng.integers(1, 60, 20))
        return (b if name == "sorted" else rng.permutation(b)), 20, 64
    if name == "empty_mid_end":                 # ids 3, 4 and 9 have no nodes, 11 is past the last id
        b = np.repeat(np.array([0, 1, 2, 5, 6, 7, 8, 10]), rng.integers(1, 30, 8))
        return rng.permutation(b), 12, 64
    if name == "single":
        return np.zeros(77, np.int64), 1, 64
    if name == "one_node":
        return np.arange(30), 30, 64
    if name in ("chunk16", "chunk64"):
        c = int(name[5:])
        sizes = [s for m in (1, 2, 3) for s in (m * c - 1, m * c, m * c + 1)] + [1, 2]
        return np.repeat(np.arange(len(sizes)), sizes), len(sizes), c
    if name == "hub":
        return np.repeat(np.arange(4), [5, HUB_N, 1, 300]), 4, 64
    raise KeyError(name)


CASES = ("sorted", "unsorted", "empty_mid_end", "single", "one_node", "chunk16", "chunk64")


def membership(batch, B, chunk, dev):
    """The Membership the public entry points build (membership_for), with the hub plan at `chunk` edges."""
    from cogdl_b200.structure import Membership, membership_for

    bt = T(batch, dev)
    if chunk == 64:
        return membership_for(bt, B), bt
    order = np.argsort(batch, kind="stable")
    rp = np.concatenate([[0], np.cumsum(np.bincount(batch, minlength=B))]).astype(np.int32)
    st = plan_structure(rp, order.astype(np.int32), len(batch), dev, "default", chunk=chunk)
    st_t, perm = st.csc()
    n = torch.from_numpy(np.bincount(batch, minlength=B)).float().to(dev)
    inv = torch.where(n > 0, 1.0 / n.clamp_min(1.0), torch.zeros_like(n))
    return Membership(st, st_t, perm, inv, inv[bt].contiguous()), bt


def chain(n, chunk):
    """The longest accumulation chain of a row of n terms: n, or a chunk plus the chunk count on a hub row."""
    return n if n <= chunk else chunk + math.ceil(n / chunk)


def place(x, how):
    if how == "strided":
        w = torch.empty((x.shape[0], x.shape[1] + 5), dtype=x.dtype, device=x.device)
        w[:, 2:2 + x.shape[1]] = x
        return w[:, 2:2 + x.shape[1]]
    return misaligned(x) if how == "misaligned" else x


def check_sum_like(got, x_np, batch, B, chunk, mean):
    """got within (L + 2) u sum|terms| of fp64; unsplit rows bit-equal to the oracle's CSR-order sum (times fl(1/n))."""
    n = np.bincount(batch, minlength=B)
    ref = (R.mean_pool if mean else R.sum_pool)(x_np, batch, B)
    mag = R.sum_pool(np.abs(x_np), batch, B) / (np.maximum(n, 1)[:, None] if mean else 1)
    L = np.array([chain(int(v), chunk) + 2 + (2 if mean else 0) for v in n], np.float64)[:, None]
    g = got.detach().double().cpu().numpy()
    assert (np.abs(g - ref) <= L * U * mag + 1e-300).all(), float((np.abs(g - ref) / np.maximum(L * U * mag, 1e-30)).max())
    order = np.argsort(batch, kind="stable")
    rp = np.concatenate([[0], np.cumsum(n)])
    seq = oracle.spmm_csr(rp, order, None, x_np.astype(np.float32))
    if mean:
        seq = (np.float32(1.0) / np.maximum(n, 1).astype(np.float32))[:, None] * seq
        seq[n == 0] = 0
    unsplit = n <= chunk
    assert np.array_equal(got.detach().cpu().numpy()[unsplit].view(np.int32), seq[unsplit].view(np.int32))


def run_pool(mb, x, mode):
    from cogdl_b200.operators.readout import ReadoutFunction

    return ReadoutFunction.apply(x, mb, mode)


@pytest.mark.parametrize("how", ["contiguous", "strided", "misaligned"])
@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("name", CASES)
def test_sum_mean_max_against_fp64(dev, name, F, how):
    batch, B, chunk = batch_case(name)
    mb, _ = membership(batch, B, chunk, dev)
    rng = np.random.default_rng(F)
    x_np = rng.standard_normal((len(batch), F)).astype(np.float32)
    dy_np = rng.standard_normal((B, F)).astype(np.float32)
    for mode in ("sum", "mean", "max"):
        x = place(T(x_np, dev), how).requires_grad_(True)
        y = run_pool(mb, x, mode)
        dy = T(dy_np, dev)
        (dx,) = torch.autograd.grad(y, x, dy)
        y2 = run_pool(mb, place(T(x_np, dev), how), mode)
        assert torch.equal(bits(y), bits(y2)), f"{mode}: second run differs"
        if mode == "max":
            out, arg = R.max_pool(x_np, batch, B)
            assert np.array_equal(y.detach().cpu().numpy(), out.astype(np.float32))
            assert np.array_equal(dx.cpu().numpy(), R.max_pool_grad(dy_np, arg, len(batch)).astype(np.float32))
            continue
        check_sum_like(y, x_np, batch, B, chunk, mode == "mean")
        if mode == "sum":
            assert torch.equal(bits(dx), bits(dy[T(batch, dev)]))
        else:
            want = R.mean_pool_grad(dy_np, batch, B)
            assert (np.abs(dx.double().cpu().numpy() - want) <= 2.001 * U * np.abs(want)).all()


def test_public_entry_points_and_graph_readout(dev):
    import cogdl_b200

    batch, B, _ = batch_case("empty_mid_end")
    bt = T(batch, dev)
    xs = [torch.randn(len(batch), F, device=dev) for F in (3, 67, 1)]
    for mode, fn in (("sum", cogdl_b200.batch_sum_pooling), ("mean", cogdl_b200.batch_mean_pooling),
                     ("max", cogdl_b200.batch_max_pooling)):
        got = cogdl_b200.graph_readout(xs, bt, mode, num_graphs=B)
        want = torch.cat([fn(x, bt, num_graphs=B) for x in xs], dim=1)
        assert got.shape == (B, 71) and torch.equal(bits(got), bits(want))
        assert (got[[3, 4, 9, 11]] == 0).all()
    assert cogdl_b200.batch_sum_pooling(xs[0], bt).shape[0] == 11      # B = max(batch) + 1 without num_graphs
    with pytest.raises(ValueError, match="out of range"):
        cogdl_b200.batch_sum_pooling(xs[0], bt, num_graphs=5)
    with pytest.raises(TypeError):
        cogdl_b200.batch_sum_pooling(xs[0].double(), bt)


@pytest.mark.parametrize("mode", ["sum", "mean", "max"])
def test_hub_graph(dev, mode):
    batch, B, chunk = batch_case("hub")
    mb, bt = membership(batch, B, chunk, dev)
    assert mb.st.plan.n_chunks > 0
    for F in (3, 128):
        x_np = np.random.default_rng(F).standard_normal((len(batch), F)).astype(np.float32)
        x = T(x_np, dev).requires_grad_(True)
        y = run_pool(mb, x, mode)
        dy = torch.randn(B, F, device=dev)
        (dx,) = torch.autograd.grad(y, x, dy)
        y2 = run_pool(mb, T(x_np, dev), mode)
        assert torch.equal(bits(y), bits(y2)), "the hub graph's second run differs"
        if mode == "max":
            from cogdl_b200.operators._raw import scatter_max_fwd_raw

            xd = T(x_np, dev)
            want = torch.zeros(B, F, device=dev).index_reduce_(0, bt, xd, "amax", include_self=False)
            assert torch.equal(y.detach(), want)
            _, arg = scatter_max_fwd_raw(mb.st, xd)
            cols = torch.arange(F, device=dev).expand(B, F)
            assert torch.equal(xd[arg.long(), cols], want) and torch.equal(bt[arg.long()], torch.arange(B, device=dev)[:, None].expand(B, F))
            assert torch.equal(dx[arg.long(), cols], dy) and int(torch.count_nonzero(dx)) == int(torch.count_nonzero(dy))
        else:
            check_sum_like(y, x_np, batch, B, chunk, mode == "mean")
            if mode == "sum":
                assert torch.equal(bits(dx), bits(dy[bt]))


def set2set_tol(n, chunk):
    return 1e-5 + 8 * chain(int(n), chunk) * U


@pytest.mark.parametrize("F", FS)
@pytest.mark.parametrize("name", CASES + ("hub",))
def test_set2set_against_fp64(dev, name, F):
    from cogdl_b200.operators.readout import Set2SetAttentionFunction

    if name == "hub" and F not in (3, 128):
        pytest.skip("the hub graph runs at F = 3 and 128")
    batch, B, chunk = batch_case(name)
    mb, _ = membership(batch, B, chunk, dev)
    rng = np.random.default_rng(F + 7)
    x_np = (rng.standard_normal((len(batch), F)) / math.sqrt(F)).astype(np.float32)
    q_np = rng.standard_normal((B, F)).astype(np.float32)
    dr_np = rng.standard_normal((B, F)).astype(np.float32)
    x, q = T(x_np, dev).requires_grad_(True), T(q_np, dev).requires_grad_(True)
    r = Set2SetAttentionFunction.apply(x, q, mb)
    dx, dq = torch.autograd.grad(r, [x, q], T(dr_np, dev))
    r2 = Set2SetAttentionFunction.apply(T(x_np, dev), T(q_np, dev), mb)
    assert torch.equal(bits(r), bits(r2))
    n = np.bincount(batch, minlength=B)
    tol = set2set_tol(n.max(), chunk)
    ref, a = R.set2set(x_np, q_np, batch, B)
    mag = R.sum_pool(a[:, None] * np.abs(x_np), batch, B)
    assert (np.abs(r.detach().double().cpu().numpy() - ref) <= tol * np.maximum(mag, np.abs(ref).max(1, keepdims=True))).all()
    assert (r.detach().cpu()[torch.from_numpy(n == 0)] == 0).all()
    rdx, rdq = R.set2set_grad(x_np, q_np, batch, B, dr_np)
    for got, want in ((dx, rdx), (dq, rdq)):     # the softmax backward cancels: bounded by the tensor's largest value
        err = np.abs(got.double().cpu().numpy() - want).max()
        assert err <= tol * np.abs(want).max(), (err, np.abs(want).max())


def sort_pool_check(dev, h_np, batch, B, k):
    from cogdl_b200 import sort_pool

    from cogdl_b200.operators._raw import sort_pool_select_raw
    from cogdl_b200.structure import membership_for

    h = T(h_np, dev).requires_grad_(True)
    out = sort_pool(h, T(batch, dev), k, num_graphs=B)
    want, idx = R.sort_pool(h_np, batch, B, k)
    got_idx, _ = sort_pool_select_raw(membership_for(T(batch, dev), B).st, T(h_np[:, -1], dev), k)
    assert np.array_equal(got_idx.cpu().numpy(), idx)
    assert np.array_equal(out.detach().cpu().numpy(), want.astype(np.float32), equal_nan=True)
    dy = torch.randn(B, k, h_np.shape[1], device=dev)
    (dx,) = torch.autograd.grad(out, h, dy)
    assert np.array_equal(dx.cpu().numpy(), R.sort_pool_grad(dy.cpu().numpy(), idx, len(batch)).astype(np.float32))
    out2 = sort_pool(T(h_np, dev), T(batch, dev), k, num_graphs=B)
    assert torch.equal(bits(out), bits(out2))


@pytest.mark.parametrize("F", (1, 3, 67))
@pytest.mark.parametrize("k", (1, 7, 40))
def test_sort_pool_sizes_around_k(dev, F, k):
    sizes = [10, 7, 0, 3, 40, 41, 1]                       # k < n, k = n, n = 0, k > n (for k = 7)
    batch = np.random.default_rng(k).permutation(np.repeat(np.arange(7), sizes))
    h = np.random.default_rng(F).standard_normal((len(batch), F)).astype(np.float32)
    sort_pool_check(dev, h, batch, 8, k)                   # graph 7: an empty id at the end


@pytest.mark.parametrize("k", (1, 5, 64, 1024))
def test_sort_pool_ties_and_nonfinite_keys(dev, k):
    rng = np.random.default_rng(k)
    batch = np.repeat(np.arange(5), [3000, 200, 64, 5, 1])
    h = rng.standard_normal((len(batch), 4)).astype(np.float32)
    h[:, -1] = rng.integers(-2, 3, len(batch)).astype(np.float32)     # many ties
    specials = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, -np.nan], np.float32)
    pick = rng.choice(len(batch), 400, replace=False)
    h[pick, -1] = specials[rng.integers(0, len(specials), 400)]
    sort_pool_check(dev, h, batch, 5, k)


@pytest.mark.parametrize("k", (1, 30, 1024))
def test_sort_pool_large_graph(dev, k):
    batch = np.random.default_rng(1).permutation(np.repeat(np.arange(3), [100_000, 5, 3000]))
    h = np.random.default_rng(2).standard_normal((len(batch), 6)).astype(np.float32)
    h[::7, -1] = np.round(h[::7, -1], 1)                    # ties across the radix passes
    sort_pool_check(dev, h, batch, 3, k)


def test_sort_pool_rejects_k_past_the_maximum(dev):
    from cogdl_b200 import sort_pool
    from cogdl_b200.operators._raw import sort_pool_max_k

    assert sort_pool_max_k() == 1024
    h, b = torch.randn(10, 3, device=dev), torch.zeros(10, dtype=torch.int64, device=dev)
    for k in (0, 1025):
        with pytest.raises(ValueError, match="k ="):
            sort_pool(h, b, k)


def test_sort_pool_past_2_31_elements(dev):
    """h [N, F] with N * F > 2^31, two graphs, the selected rows of the second past element 2^31 (forward and
    backward)."""
    from cogdl_b200.operators._raw import scatter_max_bwd_raw, sort_pool_select_raw, spmm_raw
    from cogdl_b200.structure import membership_for

    F, N, k = 1025, 2**21 + 3, 16
    assert N * F > 2**31
    h = torch.empty((N, F), device=dev)
    h[:, :8].normal_()
    h[:, 8:].fill_(0.5)
    h[:, -1].normal_()
    top = torch.arange(N - 40, N, 2, device=dev)           # the largest keys: the last rows, past 2^31 elements
    h[top, -1] = 10.0 + torch.arange(top.numel(), device=dev, dtype=torch.float32)
    h[top, :8] = torch.arange(top.numel() * 8, device=dev, dtype=torch.float32).view(-1, 8)
    batch = (torch.arange(N, device=dev) >= N // 2).long()
    mb = membership_for(batch, 2)
    idx, sel = sort_pool_select_raw(mb.st, h[:, -1], k)
    out = spmm_raw(sel, None, h).view(2, k, F)
    for g in range(2):
        lo, hi = (0, N // 2) if g == 0 else (N // 2, N)
        want = torch.sort(h[lo:hi, -1], descending=True, stable=True).indices[:k] + lo
        assert torch.equal(idx[g].long(), want)
        assert torch.equal(out[g], h[want])
    assert int(idx[1].min()) * F > 2**31
    dy = torch.randn(2, k, F, device=dev)
    del h
    dx = scatter_max_bwd_raw(dy.view(2 * k, F), idx.view(-1, 1).expand(-1, F).contiguous(), N)
    flat = idx.view(-1).long()
    assert torch.equal(dx[flat], dy.view(-1, F))
    dx[flat] = 0
    assert int(torch.count_nonzero(dx)) == 0


def test_no_host_synchronisation(dev):
    import cogdl_b200

    batch, B, _ = batch_case("unsorted")
    bt = T(batch, dev)
    x = torch.randn(len(batch), 32, device=dev, requires_grad=True)
    q = torch.randn(B, 32, device=dev, requires_grad=True)
    for i in range(2):             # the first round builds the membership, its transpose and both hub plans
        torch.cuda.set_sync_debug_mode("error" if i else "default")
        try:
            outs = [cogdl_b200.batch_sum_pooling(x, bt), cogdl_b200.batch_mean_pooling(x, bt),
                    cogdl_b200.batch_max_pooling(x, bt), cogdl_b200.graph_readout([x, x[:, :5]], bt, "sum"),
                    cogdl_b200.set2set_attention(x, q, bt), cogdl_b200.sort_pool(x, bt, 30).flatten(1)]
            torch.autograd.grad(torch.cat(outs, 1).sum(), [x, q])
        finally:
            torch.cuda.set_sync_debug_mode("default")
    torch.cuda.synchronize()


def test_reference_models_through_install():
    """The reference's pooling functions, GIN, InfoGraph encoder and SortPool through install(gin=True, readout=True):
    within 1e-5 of the golden file and of the same models under install(gin=True), bit-identical across two runs,
    untouched without the flag and restored by uninstall_readout()."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.readout_refpkg_check"], cwd=ROOT, capture_output=True, text=True,
                       timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    assert res["untouched_without_flag"] and res["rebound"] and res["restored"], res
    assert res["bit_identical"] and all(res["bit_identical"].values()), res
    assert max(res["vs_golden"].values()) <= 1e-5, res
    assert max(res["vs_gin_only"].values()) <= 1e-5, res
    assert all(res["fallbacks"].values()), res
    assert res["set2set_rel"] <= 1e-5, res

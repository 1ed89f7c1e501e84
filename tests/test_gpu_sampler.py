"""Device neighbour sampler (SURVEY 8f-4) against the oracle's restatement of sample.cpp, bit for bit.

The oracle (oracle.sample_adj / oracle.subgraph) is pinned on the CPU side to the reference's own
sample.cpp compiled in place for every path that has no randomness (tests/test_cpu_oracle_and_host.py);
the random paths share the counter-based generator, so device and oracle must agree EXACTLY on every
output array, including the first-appearance node numbering."""
import numpy as np
import pytest
import torch

import oracle
from tests.gpu_util import dev

pytestmark = pytest.mark.gpu


def graph(n, e, seed, hub=None, empty=0.2):
    rng = np.random.default_rng(seed)
    p = rng.random(n) ** 3 + 1e-3
    p[rng.random(n) < empty] = 0
    p /= p.sum()
    deg = rng.multinomial(e, p)
    if hub:
        deg[hub[0]] = hub[1]
    indptr = np.zeros(n + 1, np.int64)
    indptr[1:] = np.cumsum(deg)
    indices = rng.integers(0, n, int(indptr[-1])).astype(np.int64)
    return indptr, indices


CASES = [(300, 2500, None), (5000, 60000, (17, 9000)), (50, 0, None), (20000, 400000, (3, 30000))]


@pytest.mark.parametrize("case", range(len(CASES)))
@pytest.mark.parametrize("size,replace", [(-1, False), (-1, True), (5, True), (5, False), (1, False), (25, False), (200, False), (3, True)])
def test_sample_adj_matches_oracle_exactly(dev, case, size, replace):
    from cogdl_b200.sampling import sample_adj

    n, e, hub = CASES[case]
    indptr, indices = graph(n, e, seed=case, hub=hub)
    rng = np.random.default_rng(100 + case)
    batch = rng.permutation(n)[: max(1, n // 7)].astype(np.int64)
    if hub:
        batch[0] = hub[0] if hub[0] not in batch[1:] else batch[0]
    for seed in (0, 12345678901234567):
        ref = oracle.sample_adj(indptr, indices, batch, size, replace, seed=seed)
        got = sample_adj(torch.from_numpy(indptr).to(dev), torch.from_numpy(indices).to(dev), torch.from_numpy(batch).to(dev),
                         size, replace, seed=seed)
        for name, a, b in zip(("indptr", "indices", "nodes", "edges"), got, ref):
            assert a.dtype == torch.int64 and a.is_cuda
            assert np.array_equal(a.cpu().numpy(), b), f"{name} differs (size={size}, replace={replace}, seed={seed})"
    # structural properties, independent of the oracle
    oi, oc, on, oe = [t.cpu().numpy() for t in got]
    assert np.array_equal(on[: batch.shape[0]], batch) and len(set(on.tolist())) == on.shape[0]
    assert np.array_equal(on[oc], indices[oe]), "out_indices relabels exactly the sources of the emitted edges"
    rows_of_edges = np.repeat(batch, np.diff(oi))
    assert np.all(oe >= indptr[rows_of_edges]) and np.all(oe < indptr[rows_of_edges + 1])
    if not replace and size >= 0:
        for i in range(batch.shape[0]):
            seg = oe[oi[i]:oi[i + 1]]
            assert len(set(seg.tolist())) == seg.shape[0] == min(size, indptr[batch[i] + 1] - indptr[batch[i]])


def test_assoc_scratch_is_left_clean_and_calls_are_reproducible(dev):
    from cogdl_b200 import sampling

    indptr, indices = graph(4000, 50000, seed=9)
    ip, ix = torch.from_numpy(indptr).to(dev), torch.from_numpy(indices).to(dev)
    batch = torch.arange(0, 4000, 9, device=dev)
    sampling.set_seed(77)
    a = sampling.sample_adj(ip, ix, batch, 10, False)
    b = sampling.sample_adj(ip, ix, batch, 10, False)        # next seed: a different sample
    assert not torch.equal(a[3], b[3])
    sampling.set_seed(77)
    c = sampling.sample_adj(ip, ix, batch, 10, False)
    assert all(torch.equal(x, y) for x, y in zip(a, c))
    scratch = sampling._assoc[(str(dev), 4000)]
    assert int((scratch != sampling.UNSEEN).sum()) == 0


@pytest.mark.parametrize("case", range(len(CASES)))
def test_subgraph_matches_oracle_exactly(dev, case):
    from cogdl_b200.sampling import subgraph

    n, e, hub = CASES[case]
    indptr, indices = graph(n, e, seed=case, hub=hub)
    rng = np.random.default_rng(200 + case)
    nodes = rng.permutation(n)[: max(1, n // 3)].astype(np.int64)
    ref = oracle.subgraph(indptr, indices, nodes)
    got = subgraph(torch.from_numpy(indptr).to(dev), torch.from_numpy(indices).to(dev), torch.from_numpy(nodes).to(dev))
    assert np.array_equal(got[0].cpu().numpy(), ref[0]) and np.array_equal(got[1].cpu().numpy(), ref[1])
    assert np.array_equal(got[3].cpu().numpy(), ref[2]) and np.array_equal(got[2].cpu().numpy(), np.arange(nodes.shape[0]))


def test_floyd_is_uniform_where_the_reference_loop_is_biased(dev):
    """Inclusion frequencies over many seeds: every edge of a degree-d row must be kept with probability
    k/d.  The reference's `rand() % j` loop (oracle floyd_variant=1) fails this badly -- shown here so the
    documented divergence is evidence, not opinion."""
    from cogdl_b200.sampling import sample_adj

    d, k, trials = 6, 2, 3000
    indptr = np.array([0, d], np.int64)
    indices = np.zeros(d, np.int64)
    ip, ix = torch.from_numpy(indptr).to(dev), torch.from_numpy(indices).to(dev)
    batch = torch.zeros(1, dtype=torch.int64, device=dev)
    cnt = np.zeros(d)
    for seed in range(trials):
        cnt[sample_adj(ip, ix, batch, k, False, seed=seed)[3].cpu().numpy()] += 1
    freq = cnt / trials
    assert np.abs(freq - k / d).max() < 0.04, freq
    cnt_ref = np.zeros(d)
    for seed in range(trials):
        cnt_ref[oracle.sample_adj(indptr, indices, np.zeros(1, np.int64), k, False, seed=seed, floyd_variant=1)[3]] += 1
    assert np.abs(cnt_ref / trials - k / d).max() > 0.1, "the reference variant is visibly non-uniform"


def test_reference_graph_sample_adj_through_install(dev):
    """cogdl.data.Graph.sample_adj (data.py:792-832) on a CUDA graph after install(): the reference's own
    method body runs, with sample_adj_c resolved to the device sampler."""
    from tests.refpkg import import_reference, reference_dir

    if reference_dir() is None:
        pytest.skip("reference package not present")
    import_reference()
    import cogdl_b200
    from cogdl.data import Graph

    cogdl_b200.install()
    indptr, indices = graph(3000, 40000, seed=5, empty=0.0)
    g = Graph(row_ptr=torch.from_numpy(indptr), col=torch.from_numpy(indices)).to(dev)
    batch = torch.arange(0, 3000, 11, device=dev)
    cogdl_b200.sampling.set_seed(5)
    nodes, sub = g.sample_adj(batch, 7, replace=False)
    ref = oracle.sample_adj(indptr, indices, batch.cpu().numpy(), 7, False, seed=5)
    assert np.array_equal(nodes.cpu().numpy(), ref[2])
    assert np.array_equal(sub.col_indices.cpu().numpy(), ref[1])
    assert np.array_equal(sub.row_indptr.cpu().numpy()[: batch.numel() + 1], ref[0])

"""GENConv edge-encoder kernels (cogdl_b200/csrc/genconv_edge.cu) and genconv_aggregate(edge_attr=, edge_weight=)
against the fp64 restatement of tests/genconv_ref.py with edge_term = attr @ W.T, against the edge-term kernels bit
for bit where the product is exact, and the reference DeeperGCN with an EdgeEncoder through install(genconv=True)."""
import json
import os
import subprocess
import sys

import pytest
import torch

from tests import graphs
from tests.genconv_edge_table import TABLE
from tests.genconv_ref import genconv_aggregate_fp64
from tests.test_gpu_genconv import err, structure

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SOFTMAX_AGGRS = ("softmax_sg", "softmax", "mean", "sum")


@pytest.fixture(scope="module")
def dev():
    import cogdl_b200  # noqa: F401

    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def operands(st, F, D, dev, seed=0):
    g = torch.Generator(device=dev).manual_seed(seed)
    x = torch.randn(st.n_cols, F, device=dev, generator=g)
    attr = torch.rand(st.nnz, D, device=dev, generator=g)
    w = torch.randn(F, D, device=dev, generator=g) / D ** 0.5
    return x, attr, w


def fp64(st, x, attr, w, aggr, beta=1.0):
    return genconv_aggregate_fp64(st.rowptr, st.colind, x, aggr, beta=beta, edge_term=attr.double() @ w.double().T)


@pytest.mark.parametrize("chunk", [None, 16])
@pytest.mark.parametrize("D", [1, 3, 8, 16])
@pytest.mark.parametrize("F", [7, 16, 64, 128, 256])
@pytest.mark.parametrize("name", list(graphs.CASES))
def test_forward_matches_fp64(dev, name, F, D, chunk):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev, chunk)
    x, attr, w = operands(st, F, D, dev, seed=F + D)
    for beta in (0.0, 0.5, 1.0, 4.0):
        got = genconv_aggregate(st, x, "softmax_sg", beta=beta, edge_attr=attr, edge_weight=w)
        assert got.shape == (st.n_rows, F)
        assert err(got, fp64(st, x, attr, w, "softmax_sg", beta)) <= 1e-5, f"beta={beta}"
    for aggr in ("softmax", "mean", "sum"):
        got = genconv_aggregate(st, x, aggr, edge_attr=attr, edge_weight=w)
        assert err(got, fp64(st, x, attr, w, aggr)) <= 1e-5, aggr


def q_fp64(st, x, attr, w, beta, eps=1e-7):
    """Q[i] = sum_e w_e m_e^2 in fp64 (the forward's d beta operand); 0 on degree-0 rows."""
    rp, ci = st.rowptr.long(), st.colind.long()
    n, F = st.n_rows, x.shape[1]
    row = torch.repeat_interleave(torch.arange(n, device=rp.device), rp[1:] - rp[:-1])
    m = torch.relu(x.double()[ci] + attr.double() @ w.double().T) + eps
    z = beta * m
    zmax = torch.full((n, F), -torch.inf, dtype=torch.float64, device=m.device).scatter_reduce(
        0, row[:, None].expand(-1, F), z, "amax")
    ex = torch.exp(z - zmax[row])
    zeros = torch.zeros(n, F, dtype=torch.float64, device=m.device)
    return zeros.index_add(0, row, ex * m * m) / zeros.index_add(0, row, ex).clamp_min(1e-300)


def _grads(fn, x, w, beta, r, dtype, need_x=True, need_w=True, need_b=True):
    xs = x.clone().to(dtype).requires_grad_(need_x)
    ws = w.clone().to(dtype).requires_grad_(need_w)
    bs = beta.clone().to(dtype).requires_grad_(need_b)
    out = fn(xs, ws, bs)
    (out * r.to(dtype)).sum().backward()
    return out.detach(), xs.grad, ws.grad, bs.grad


@pytest.mark.parametrize("aggr", SOFTMAX_AGGRS)
@pytest.mark.parametrize("name", ["ragged", "hub", "two_hubs", "rect"])
def test_gradients_match_fp64_autograd(dev, name, aggr):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev)
    F, D = 64, 8
    x, attr, w = operands(st, F, D, dev, seed=11)
    r = torch.randn(st.n_rows, F, device=dev, generator=torch.Generator(device=dev).manual_seed(12))
    beta = torch.full((1,), 1.5, device=dev)
    need_b = aggr == "softmax_sg"

    def mine(x_, w_, b_):
        return genconv_aggregate(st, x_, aggr, beta=b_, edge_attr=attr, edge_weight=w_)

    def exact(x_, w_, b_):
        return genconv_aggregate_fp64(st.rowptr, st.colind, x_, aggr, beta=b_, edge_term=attr.double() @ w_.T)

    want = _grads(exact, x, w, beta, r, torch.float64, need_b=need_b)
    got = _grads(mine, x, w, beta, r, torch.float32, need_b=need_b)
    assert err(got[1], want[1]) <= 1e-4
    assert err(got[2], want[2]) <= 1e-4
    if need_b:
        assert err(got[3], want[3]) <= 1e-4
    else:
        assert got[3] is None
    # only W needs grad: no dx; only x: no dW (and the frozen W costs no dW pass)
    only_w = _grads(mine, x, w, beta, r, torch.float32, need_x=False, need_b=False)
    assert only_w[1] is None and err(only_w[2], want[2]) <= 1e-4
    assert torch.equal(only_w[2], got[2])
    only_x = _grads(mine, x, w, beta, r, torch.float32, need_w=False, need_b=False)
    assert only_x[2] is None and torch.equal(only_x[1], got[1])


@pytest.mark.parametrize("aggr", SOFTMAX_AGGRS)
@pytest.mark.parametrize("F", [7, 128, 256])
@pytest.mark.parametrize("name", ["hub", "two_hubs", "rect"])
def test_bit_identical_to_edge_term_kernels(dev, name, F, aggr):
    """attr in {-2..2} and W in multiples of 1/8 make attr @ W.T exact in fp32 in any order: out and dx equal the
    edge-term kernels' bit for bit, dW is within 1e-5 of d_edge_term.T @ attr."""
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev, 16)
    D = 8
    g = torch.Generator(device=dev).manual_seed(F)
    x = torch.randn(st.n_cols, F, device=dev, generator=g)
    attr = torch.randint(-2, 3, (st.nnz, D), device=dev, generator=g).float()
    w = torch.randint(-8, 9, (F, D), device=dev, generator=g).float() / 8
    r = torch.randn(st.n_rows, F, device=dev, generator=g)
    beta = 0.7 if aggr == "softmax_sg" else None

    xa = x.clone().requires_grad_(True)
    wa = w.clone().requires_grad_(True)
    out_a = genconv_aggregate(st, xa, aggr, beta=beta, edge_attr=attr, edge_weight=wa)
    (out_a * r).sum().backward()
    xb = x.clone().requires_grad_(True)
    term = (attr @ w.T).requires_grad_(True)
    out_b = genconv_aggregate(st, xb, aggr, beta=beta, edge_term=term)
    (out_b * r).sum().backward()
    assert torch.equal(out_a, out_b)
    assert torch.equal(xa.grad, xb.grad)
    assert err(wa.grad, term.grad.T.double() @ attr.double()) <= 1e-5


@pytest.mark.parametrize("name", ["hub", "two_hubs"])
def test_forward_backward_bitwise_reproducible(dev, name):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure(name, dev, 16)
    x0, attr, w0 = operands(st, 128, 8, dev, seed=5)
    r = torch.randn(st.n_rows, 128, device=dev, generator=torch.Generator(device=dev).manual_seed(6))

    def once():
        x, w = x0.clone().requires_grad_(True), w0.clone().requires_grad_(True)
        b = torch.full((1,), 0.8, device=dev, requires_grad=True)
        out = genconv_aggregate(st, x, "softmax_sg", beta=b, edge_attr=attr, edge_weight=w)
        (out * r).sum().backward()
        return out.detach(), x.grad, w.grad, b.grad

    first, second = once(), once()
    assert all(torch.equal(u, v) for u, v in zip(first, second))


def _row_operands(c, dev):
    from cogdl_b200.structure import DEFAULT_CHUNK_EDGES

    st, *_ = structure(c.graph, dev, c.chunk or DEFAULT_CHUNK_EDGES)
    x, attr, w = operands(st, c.F, c.D, dev, seed=c.F * 17 + c.D)
    if not c.aligned:    # 4 bytes off 16-byte alignment: the scalar kernel
        x = torch.empty(st.n_cols * c.F + 1, device=dev)[1:].view(st.n_cols, c.F).copy_(x)
    return st, x, attr, w


@pytest.mark.parametrize("c", TABLE, ids=[c.id for c in TABLE])
def test_table_row(dev, c):
    """Every compiled instantiation: records its name, and matches fp64 (forward 1e-5, gradients 1e-4)."""
    from cogdl_b200 import _cabi
    from cogdl_b200.operators._raw import genconv_edge_bwd_raw, genconv_edge_fwd_raw

    st, x, attr, w = _row_operands(c, dev)
    beta = torch.full((1,), 1.3, device=dev)
    out, lse2, q = genconv_edge_fwd_raw(st, x, attr, w, beta, 1e-7, want_lse=True, want_q=c.want_q)
    if c.op == "fwd":
        if st.n_rows and c.F:
            assert _cabi.last_kernel() == c.kernel
        want = fp64(st, x, attr, w, "softmax_sg", beta)
        assert err(out, want) <= 1e-5
        if c.want_q:
            assert err(q, q_fp64(st, x, attr, w, float(beta))) <= 1e-5
        return
    r = torch.randn(st.n_rows, c.F, device=dev, generator=torch.Generator(device=dev).manual_seed(3))
    dx, dw = genconv_edge_bwd_raw(st, x, attr, w, beta, 1e-7, r, out, lse2, want_dx="dx" in c.want,
                                  want_dw="dw" in c.want)
    if st.n_cols and c.F:
        assert _cabi.last_kernel() == c.kernel
    x64, w64 = x.double().requires_grad_(True), w.double().requires_grad_(True)
    (fp64(st, x64, attr, w64, "softmax_sg", beta) * r.double()).sum().backward()
    if "dx" in c.want:
        assert err(dx, x64.grad) <= 1e-4
    else:
        assert dx is None
    if "dw" in c.want:
        assert err(dw, w64.grad) <= 1e-4
    else:
        assert dw is None


def test_no_edge_sized_tensor(dev):
    """Arxiv shape, F = 128, D = 8: beyond the three [N, F] tensors the operator has to hold (out, the saved lse2,
    then dx), forward + backward grow max_memory_allocated by less than a quarter of one [nnz, F] tensor; and the
    forward is within 1e-5 of fp64 evaluated on the GPU.  (At arxiv's mean degree of 7.9 one [N, F] tensor is an
    eighth of an [nnz, F] one, so the node-sized tensors are counted out rather than hidden in the bound; beta is a
    constant here, as the dense d beta reduction adds node-sized temporaries of its own.)"""
    from cogdl_b200 import genconv_aggregate, synth
    from cogdl_b200.structure import CSRStructure

    n, e = synth.SHAPES["arxiv"]
    rp, col = synth.powerlaw_csr(n, e, seed=0, device=dev, self_loops=True)
    st = CSRStructure.from_int64(rp, col)
    del rp, col
    F, D = 128, 8
    x, attr, w = operands(st, F, D, dev, seed=0)
    st.plan, st.csc()[0].plan                          # structure built before the measurement
    xg, wg = x.clone().requires_grad_(True), w.clone().requires_grad_(True)
    beta = torch.ones(1, device=dev)
    r = torch.randn(st.n_rows, F, device=dev)
    with torch.no_grad():
        genconv_aggregate(st, x, "softmax_sg", beta=1.0, edge_attr=attr, edge_weight=w)   # plan scratch sized
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    out = genconv_aggregate(st, xg, "softmax_sg", beta=beta, edge_attr=attr, edge_weight=wg)
    out.backward(r)
    torch.cuda.synchronize()
    growth = torch.cuda.max_memory_allocated() - base - 3 * st.n_rows * F * 4
    assert growth < st.nnz * F * 4 / 4, (growth, st.nnz * F * 4)
    assert xg.grad is not None and wg.grad is not None
    with torch.no_grad():
        got = genconv_aggregate(st, x, "softmax_sg", beta=1.0, edge_attr=attr, edge_weight=w)
    assert err(got, fp64(st, x, attr, w, "softmax_sg", 1.0)) <= 1e-5


def test_errors(dev):
    from cogdl_b200 import genconv_aggregate

    st, *_ = structure("tiny", dev)
    x, attr, w = operands(st, 8, 3, dev)
    with pytest.raises(ValueError):      # both an edge term and edge features
        genconv_aggregate(st, x, "softmax", edge_term=attr @ w.T, edge_attr=attr, edge_weight=w)
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr)
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_weight=w)
    with pytest.raises(ValueError):      # nnz mismatch
        genconv_aggregate(st, x, "softmax", edge_attr=attr[:-1], edge_weight=w)
    with pytest.raises(ValueError):      # W not [F, D]
        genconv_aggregate(st, x, "softmax", edge_attr=attr, edge_weight=w.T.contiguous())
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr[:, 0], edge_weight=w)
    wide = torch.rand(st.nnz, 17, device=dev)
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_attr=wide, edge_weight=torch.randn(8, 17, device=dev))
    with pytest.raises(ValueError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr.clone().requires_grad_(True), edge_weight=w)
    with pytest.raises(RuntimeError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr.cpu(), edge_weight=w)
    with pytest.raises(TypeError):
        genconv_aggregate(st, x, "softmax", edge_attr=attr.double(), edge_weight=w)
    for aggr in ("max", "powermean"):
        with pytest.raises(NotImplementedError):
            genconv_aggregate(st, x, aggr, edge_attr=attr, edge_weight=w)


def test_reference_deepergcn_with_edge_encoder_through_install():
    """Reference DeeperGCN (softmax_sg, learnable beta, edge_attr_size=[8]) and a lone GENConv with an EdgeEncoder
    through install(genconv=True), in a child process (tests/genconv_edge_refpkg_check.py)."""
    from tests.refpkg import reference_dir

    if reference_dir() is None:
        pytest.fail("the reference package must be built (oracle/_ref/pkg): run oracle/build_ref.py")
    r = subprocess.run([sys.executable, "-m", "tests.genconv_edge_refpkg_check"], cwd=ROOT, capture_output=True,
                       text=True, timeout=900)
    assert r.returncode == 0, r.stderr[-4000:]
    res = json.loads(r.stdout.strip().splitlines()[-1])
    for name in ("deepergcn", "genconv_edge"):
        m = res[name]
        assert m["logits_vs_ref_cpu"] <= 1e-4, (name, m)
        assert m["logits_vs_fp64"] <= 1e-4, (name, m)
        assert m["grads_present"], (name, m)
        assert m["edge_encoder_calls"] == 0, (name, m)
        assert "genconv_edge_" in m["last_kernel"], (name, m)
    assert max(res["genconv_edge"]["grad_errs"].values()) <= 1e-4, res["genconv_edge"]
    assert max(res["deepergcn"]["grad_errs_model_scale"].values()) <= 1e-3, res["deepergcn"]
    for case in ("bond_encoder", "attr_requires_grad"):
        assert res[case]["edge_term_kernel"], (case, res[case])

"""fp64 restatements of the reference GTN (cogdl/models/nn/gtn.py) and SRGCN (cogdl/models/nn/srgcn.py,
cogdl/utils/srgcn_utils.py) forward passes, and the fp64 sparse products they are written on -- test infrastructure.

`spspmm64` is the sparse x sparse product in fp64 with scipy: the pattern is structural (from |A| @ |B|), the values
and their gradients come from the fp64 products.  It doubles as the `torch_sparse` stand-in of the golden run
(tests/golden/make_golden_spspmm_models.py), which returns the values in the input's dtype.  The model shapes and the
seeded inputs shared by the golden run, its CPU test and the GPU child check live here too.
"""
import numpy as np
import scipy.sparse as sp
import torch
import torch.nn.functional as F

N_GTN, E_REL, F_GTN, HID_GTN, C_GTN = 9000, 9000, 8, 16, 4
N_CORA, E_CORA, F_CORA, C_CORA, NHEAD = 2708, 10556, 16, 7, 4


def gtn_inputs():
    """4 relations of 9 000 random edges over 9 000 nodes (unit values), and node features."""
    g = torch.Generator().manual_seed(41)
    adj = []
    for _ in range(4):
        row, col = torch.randint(0, N_GTN, (E_REL,), generator=g), torch.randint(0, N_GTN, (E_REL,), generator=g)
        adj.append((torch.stack([row, col]), torch.ones(E_REL)))
    return adj, torch.randn(N_GTN, F_GTN, generator=g)


def cora_inputs():
    """A symmetric Cora-shaped edge list (with repeated edges and self loops, as random graphs have) and features."""
    g = torch.Generator().manual_seed(42)
    row, col = torch.randint(0, N_CORA, (E_CORA // 2,), generator=g), torch.randint(0, N_CORA, (E_CORA // 2,), generator=g)
    return torch.stack([torch.cat([row, col]), torch.cat([col, row])]), torch.randn(N_CORA, F_CORA, generator=g)


def _csr(index, value, m, n):
    i = index.detach().cpu().numpy()
    return sp.coo_matrix((value.detach().cpu().double().numpy(), (i[0], i[1])), shape=(m, n)).tocsr()


class _SpSpMM64(torch.autograd.Function):
    @staticmethod
    def forward(ctx, indexA, valueA, indexB, valueB, m, k, n):
        A, B = _csr(indexA, valueA, m, k), _csr(indexB, valueB, k, n)
        ones = lambda M: sp.csr_matrix((np.ones(M.nnz), M.indices, M.indptr), shape=M.shape)  # noqa: E731
        P = (ones(_csr(indexA, torch.ones(indexA.shape[1]), m, k)) @ ones(_csr(indexB, torch.ones(indexB.shape[1]), k, n)))
        P = P.tocsr()
        P.sort_indices()
        r, c = np.repeat(np.arange(m), np.diff(P.indptr)), P.indices
        vals = np.asarray((A @ B).tocsr()[r, c]).ravel() if r.size else np.zeros(0)
        ctx.save_for_backward(indexA, valueA, indexB, valueB)
        ctx.dims, ctx.rc = (m, k, n), (r, c)
        return torch.from_numpy(np.stack([r, c]).astype(np.int64)), torch.from_numpy(vals).to(valueA.dtype)

    @staticmethod
    def backward(ctx, _gi, g):
        indexA, valueA, indexB, valueB = ctx.saved_tensors
        m, k, n = ctx.dims
        r, c = ctx.rc
        G = sp.csr_matrix((g.double().numpy(), (r, c)), shape=(m, n))
        A, B = _csr(indexA, valueA, m, k), _csr(indexB, valueB, k, n)
        ia, ib = indexA.numpy(), indexB.numpy()
        dA = np.asarray((G @ B.T).tocsr()[ia[0], ia[1]]).ravel()
        dB = np.asarray((A.T @ G).tocsr()[ib[0], ib[1]]).ravel()
        return None, torch.from_numpy(dA).to(valueA.dtype), None, torch.from_numpy(dB).to(valueB.dtype), None, None, None


def spspmm64(indexA, valueA, indexB, valueB, m, k, n, coalesced=False):
    """torch_sparse.spspmm's signature and result (row-major sorted index, values in valueA's dtype), in fp64."""
    return _SpSpMM64.apply(indexA, valueA, indexB, valueB, m, k, n)


def spmm64(index, value, m, n, matrix):
    """torch_sparse.spmm: the COO (duplicates summed) times a dense matrix, differentiable in value and matrix."""
    out = torch.zeros(m, matrix.shape[1], dtype=matrix.dtype)
    return out.index_add(0, index[0], value.to(matrix.dtype)[:, None] * matrix[index[1]])


# ----------------------------------------------------------------------------------------------------------- GTN
def _coalesce(row, col, value):
    """cogdl.utils.coalesce (cogdl/utils/graph_utils.py:194-217) as it is: the index is sorted, the values are not
    permuted, and with duplicates they are scatter-added by column."""
    order = np.lexsort((col.numpy(), row.numpy()))
    row, col = row[order], col[order]
    max_num = max(int(row.max()), int(col.max())) + 100
    idx = torch.cat([torch.full((1,), -1, dtype=torch.long), (row + 1) * max_num + col])
    mask = idx[1:] > idx[:-1]
    if mask.all():
        return row, col, value
    row = row[mask]
    value = torch.zeros(row.shape[0], dtype=value.dtype).scatter_add(0, col, value)
    return row, col[mask], value


def _gt_conv(weight, A):
    filt = torch.softmax(weight, dim=1)
    out = []
    for i in range(filt.shape[0]):
        index = torch.cat([e for e, _ in A], dim=1)
        value = torch.cat([v * filt[i][j] for j, (_, v) in enumerate(A)])
        row, col, value = _coalesce(index[0], index[1], value)
        out.append((torch.stack([row, col]), value))
    return out


def _gtn_normalization(H, N):
    out = []
    for edge, value in H:
        mask = edge[0] != edge[1]
        edge, value = edge[:, mask], value[mask]
        with torch.no_grad():
            deg = torch.zeros(N, dtype=value.dtype).scatter_add(0, edge[0], value.detach())
            inv = deg.pow(-1)
            inv[inv == float("inf")] = 0
        out.append((edge, inv[edge[1]] * value))
    return out


def _linear(p, name, x):
    return x @ p[name + ".weight"].t() + p[name + ".bias"]


def gtn_fp64(p, adj, x, num_layers=2):
    """Logits of GTN.forward (gtn.py:159-184) in fp64; p maps parameter names to fp64 leaves, adj is the list of
    (index [2, E], value [E]) relations."""
    N = x.shape[0]
    adj = [(e, v.double()) for e, v in adj]
    H = None
    for li in range(num_layers):
        pre = f"layers.{li}."
        if li == 0:
            A_, B_ = _gt_conv(p[pre + "conv1.weight"], adj), _gt_conv(p[pre + "conv2.weight"], adj)
        else:
            A_, B_ = _gtn_normalization(H, N), _gt_conv(p[pre + "conv1.weight"], adj)
        H = [spspmm64(a[0], a[1], b[0], b[1], N, N, N) for a, b in zip(A_, B_)]
    xs = []
    for edge, value in H:
        support = _linear(p, "gcn.linear", x)
        xs.append(F.relu(spmm64(edge, value, N, N, support)))
    h = F.relu(_linear(p, "linear1", torch.cat(xs, dim=1)))
    return _linear(p, "linear2", h)


# ----------------------------------------------------------------------------------------------------------- SRGCN
def _self_loops(ei, N):
    """add_remaining_self_loops (cogdl/utils/graph_utils.py:40-72): the non-loop edges, then (i, i) for every i."""
    mask = ei[0] != ei[1]
    loops = torch.arange(N)
    return torch.stack([torch.cat([ei[0][mask], loops]), torch.cat([ei[1][mask], loops])])


def _node_attention(p, pre, h, ind, val):
    """NodeAttention (srgcn_utils.py:17-37): val * deg^-1[row] times the diagonal sigmoid(p(h)), through spspmm."""
    N = h.shape[0]
    diag = torch.sigmoid(_linear(p, pre + "attention.p", h)).view(-1)
    deg = torch.bincount(ind[0], minlength=N).to(h.dtype)
    diag_ind = torch.arange(N).repeat(2, 1)
    return spspmm64(ind, deg.pow(-1)[ind[0]] * val, diag_ind, diag, N, N, N)[1]


def _row_norm(ind, val, N):
    rs = spmm64(ind, val, N, N, torch.ones(N, 1, dtype=val.dtype)).view(-1)
    return (1.0 / rs)[ind[0]] * val


def _adaptive(p, pre, x):
    h = torch.sigmoid(x @ p[pre + "fc"] + p[pre + "bf"])
    return torch.where(x < 0, torch.zeros_like(x), x) + h * torch.where(x > 0, torch.zeros_like(x), x)


def _square(ind, N):
    val = torch.ones(ind.shape[1], dtype=torch.float64)
    return spspmm64(ind, val, ind, val, N, N, N)


def srgcn_fp64(p, ei, x, nhead=NHEAD):
    """Logits of SRGCN.forward (srgcn.py:273-277) in fp64 for attention="node", normalization="row_uniform",
    activation="leaky_relu", nhop=2, subheads=1 and no dropout (eval)."""
    N = x.shape[0]
    ind, val = _square(_self_loops(ei, N), N)
    heads = []
    for a in range(nhead):
        pre = f"attention_{a}."
        h = x @ p[pre + "weight.0"]
        v = _row_norm(ind, _node_attention(p, pre, h, ind, val), N)
        out = spmm64(ind, v, N, N, h)
        out = torch.nan_to_num(out, nan=0.0, posinf=float("inf"), neginf=float("-inf")) + p[pre + "bias.0"]
        heads.append(F.leaky_relu(_adaptive(p, pre + "adaptive_enc.0.", out)))
    x2 = F.elu(torch.cat(heads, dim=1))
    h = x2 @ p["out_att.weight"]
    v = _node_attention(p, "out_att.", h, ind, val).exp()
    v = (1.0 / spmm64(ind, v, N, N, torch.ones(N, 1, dtype=v.dtype)).view(-1))[ind[0]] * v
    out = spmm64(ind, v, N, N, h)
    out = torch.nan_to_num(out, nan=0.0, posinf=float("inf"), neginf=float("-inf")) + p["out_att.bias"]
    return _adaptive(p, "out_att.adaptive_enc.", out)

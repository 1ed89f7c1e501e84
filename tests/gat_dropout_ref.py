"""Restatements of the GAT attention dropout: the keep rule of the kernels in numpy, and CogDL's GATLayer forward
(cogdl/layers/gat_layer.py:59-86, unfused branch: leakyrelu(h_l[row] + h_r[col]) -> edge_softmax -> dropout ->
mh_spmm) in fp64 torch with a given mask.  The GPU tests compare the fused kernels against these; the CPU tests pin
them to the library's draw function and to the reference layer's own output (tests/golden/gat_dropout.npz)."""
import numpy as np
import torch

_GOLDEN_GAMMA = np.uint64(0xD1342543DE82EF95)


def _mix64(z):
    z = z + np.uint64(0x9E3779B97F4A7C15)
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def draw(seed, i, k):
    """cogdl_b200_sample_draw(seed, i, k) over broadcast uint64 arrays (wrapping arithmetic)."""
    i, k = np.asarray(i, np.uint64), np.asarray(k, np.uint64)
    with np.errstate(over="ignore"):
        return _mix64(_mix64(np.uint64(seed) + i * _GOLDEN_GAMMA) + k)


def drop_below(p):
    """floor(p * 2^64): an (edge, head) whose draw is below it is dropped."""
    return int(p * 2.0 ** 64)


def keep_mask(seed, nnz, H, p):
    """bool [nnz, H]: CSR edge e, head h is kept iff draw(seed, e, h) >= floor(p * 2^64)."""
    e = np.arange(nnz, dtype=np.uint64)[:, None]
    h = np.arange(H, dtype=np.uint64)[None, :]
    return draw(seed, e, h) >= np.uint64(drop_below(p))


def _rows(rowptr):
    rowptr = torch.as_tensor(np.asarray(rowptr, np.int64))
    return torch.repeat_interleave(torch.arange(rowptr.numel() - 1), rowptr[1:] - rowptr[:-1])


def gat_attention_fp64(rowptr, colind, h_l, h_r, slope):
    """softmax over each row's edges of leakyrelu(h_l[row] + h_r[col]), [nnz, H] (h_l, h_r: [n, H] fp64 tensors)."""
    rows, cols = _rows(rowptr).to(h_l.device), torch.as_tensor(np.asarray(colind, np.int64)).to(h_l.device)
    n, H = h_l.shape
    e = torch.nn.functional.leaky_relu(h_l[rows] + h_r[cols], slope)
    m = torch.full((n, H), -torch.inf, dtype=e.dtype, device=e.device)
    m = m.scatter_reduce(0, rows[:, None].expand(-1, H), e.detach(), "amax")     # a shift: no gradient needed
    ex = torch.exp(e - m[rows])
    s = torch.zeros((n, H), dtype=e.dtype, device=e.device).index_add_(0, rows, ex)
    return ex / s[rows]


def gat_dropout_fp64(rowptr, colind, h_l, h_r, feat, slope, keep, p):
    """out [n, H, F] = sum over row i's edges of dropout(att)[e, h] * feat[col[e], h, :], dropout(att) = att * keep /
    (1 - p).  keep: bool [nnz, H] in CSR order."""
    rows, cols = _rows(rowptr).to(h_l.device), torch.as_tensor(np.asarray(colind, np.int64)).to(h_l.device)
    att = gat_attention_fp64(rowptr, colind, h_l, h_r, slope)
    keep = torch.as_tensor(np.asarray(keep)).to(device=att.device, dtype=att.dtype)
    a = att * keep / (1.0 - p)
    out = torch.zeros((h_l.shape[0],) + tuple(feat.shape[1:]), dtype=feat.dtype, device=feat.device)
    return out.index_add_(0, rows, a[:, :, None] * feat[cols])


def gat_layer_fp64(x, W, a_l, a_r, rowptr, colind, slope, keep, p):
    """GATLayer.forward (no residual, norm or activation) with the attention dropout given by keep, all in fp64."""
    nhead, out_feats = a_l.shape[1], a_l.shape[2]
    h = (x @ W).view(-1, nhead, out_feats)
    h_l, h_r = (a_l * h).sum(dim=-1), (a_r * h).sum(dim=-1)
    out = gat_dropout_fp64(rowptr, colind, h_l, h_r, h, slope, keep, p)
    return out.reshape(out.shape[0], -1)

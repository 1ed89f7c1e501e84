"""fp64 torch restatement of GENConv's aggregation (cogdl/layers/deepergcn_layer.py:64-95), shared by the CPU golden
test and the GPU parity tests.  Differentiable in x, the edge term and beta (plain autograd, exact in fp64)."""
import torch


def genconv_aggregate_fp64(rowptr, colind, x, aggr, beta=1.0, eps=1e-7, edge_term=None, p=1.0):
    """rowptr [n+1], colind [nnz] (CSR), x [n_cols, F], edge_term [nnz, F] in CSR order or None.  Any device; the
    arithmetic is fp64 whatever the input dtype.  Returns h [n, F]."""
    rowptr, colind = torch.as_tensor(rowptr).long(), torch.as_tensor(colind).long()
    n = rowptr.numel() - 1
    deg = rowptr[1:] - rowptr[:-1]
    row = torch.repeat_interleave(torch.arange(n, device=rowptr.device), deg)
    pre = x.double()[colind]
    if edge_term is not None:
        pre = pre + edge_term.double()
    m = torch.relu(pre) + eps
    F = m.shape[1]
    idx = row[:, None].expand(-1, F)
    zeros = torch.zeros(n, F, dtype=torch.float64, device=m.device)
    degf = deg.double()[:, None]
    if aggr in ("softmax_sg", "softmax"):
        b = beta if aggr == "softmax_sg" else 1.0
        b = b.double() if torch.is_tensor(b) else float(b)
        z = b * m
        zmax = torch.full((n, F), -torch.inf, dtype=torch.float64, device=m.device).scatter_reduce(
            0, idx, z.detach(), "amax")
        ex = torch.exp(z - zmax[row])
        w = ex / zeros.index_add(0, row, ex)[row]
        return zeros.index_add(0, row, w * m)
    if aggr in ("mean", "sum"):
        s = zeros.index_add(0, row, m)
        return s / degf.clamp_min(1) if aggr == "mean" else s
    if aggr == "max":
        return zeros.scatter_reduce(0, idx, m, "amax", include_self=False)
    if aggr == "powermean":
        mp = torch.clamp(m, 1e-7, 1.0) ** p
        return (zeros.index_add(0, row, mp) / degf.clamp_min(1)) ** (1.0 / p)
    raise ValueError(aggr)

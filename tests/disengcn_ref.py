"""fp64 torch restatement of DisenGCN's neighbourhood routing (cogdl/layers/disengcn_layer.py:40-91), shared by the
CPU golden test and the GPU parity tests.  Differentiable in q, c and h (plain autograd, exact in fp64)."""
import torch


def _rows(rowptr):
    rowptr = torch.as_tensor(rowptr).long()
    n = rowptr.numel() - 1
    return n, torch.repeat_interleave(torch.arange(n, device=rowptr.device), rowptr[1:] - rowptr[:-1])


def route_step_fp64(rowptr, colind, q, c, K, tau, with_norm=False):
    """One routing step over the CSR (rowptr, colind): per row i and channel k, out = u / |u| with
    u = sum_e softmax_e(q_i,k . c_j,k / tau) c_j,k + c_i,k.  q, c [n, K*d]; any device, fp64 arithmetic.
    with_norm: also return |u| [n, K]."""
    n, row = _rows(rowptr)
    col = torch.as_tensor(colind).long().to(row.device)
    q, c = q.double(), c.double()
    F = c.shape[1]
    d = F // K
    qk, ck = q.reshape(n, K, d), c.reshape(n, K, d)
    s = (qk[row] * ck[col]).sum(-1) / tau                                              # [E, K]
    smax = torch.full((n, K), -torch.inf, dtype=torch.float64, device=c.device).scatter_reduce(
        0, row[:, None].expand(-1, K), s.detach(), "amax")
    ex = torch.exp(s - smax[row])
    w = ex / torch.zeros(n, K, dtype=torch.float64, device=c.device).index_add(0, row, ex)[row]
    a = torch.zeros(n, K, d, dtype=torch.float64, device=c.device).index_add(0, row, w[..., None] * ck[col])
    u = a + ck
    r = u.pow(2).sum(-1, keepdim=True).sqrt()
    out = (u / r).reshape(n, F)
    return (out, r.squeeze(-1)) if with_norm else out


def normalize_channels_fp64(h, K):
    h = h.double()
    n, F = h.shape
    hk = h.reshape(n, K, F // K)
    return (hk / hk.pow(2).sum(-1, keepdim=True).sqrt()).reshape(n, F)


def disen_routing_fp64(rowptr, colind, h, K, iterations, tau, with_norm=False):
    """DisenGCNLayer.forward after h = act(x W + b): normalise per channel, then `iterations` (>= 1 with
    with_norm) routing steps.  with_norm: also return the last step's |u| [n, K]."""
    c = normalize_channels_fp64(h, K)
    q, r = c, None
    for _ in range(iterations):
        q, r = route_step_fp64(rowptr, colind, q, c, K, tau, with_norm=True)
    return (q, r) if with_norm else q

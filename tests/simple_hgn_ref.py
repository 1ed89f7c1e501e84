"""fp64 restatement of Simple-HGN's layer (myGATConv, CogDL examples/simple_hgn/conv.py) and its attention, with the
attention dropout given as a keep mask (tests/gat_dropout_ref.keep_mask builds the kernels' mask).  The backward is
torch autograd of these fp64 expressions.  Also a stand-in module with myGATConv's parameters and attributes, so
cogdl_b200.install_simple_hgn can be exercised without the example file; its forward is the example's op sequence in
the module's dtype."""
import math

import numpy as np
import torch

from tests.gat_dropout_ref import _rows


def hgn_attention_fp64(rowptr, colind, etype, h_l, h_r, h_e, slope, keep=None, p=0.0, res_attn=None, alpha=0.0):
    """(a, m) [nnz, H]: a = softmax over each row's edges of leakyrelu(h_l[row] + h_r[col] + h_e[etype]); m = (1 -
    alpha) * a * keep / (1 - p) + alpha * res_attn (no blend without res_attn, no dropout without keep)."""
    dev = h_l.device
    rows = _rows(rowptr).to(dev)
    cols = torch.as_tensor(np.asarray(colind, np.int64)).to(dev)
    et = torch.as_tensor(np.asarray(etype, np.int64)).to(dev)
    n, H = h_l.shape[0], h_l.shape[1]
    z = torch.nn.functional.leaky_relu(h_l[rows] + h_r[cols] + h_e[et], slope)
    mx = torch.full((n, H), -torch.inf, dtype=z.dtype, device=dev)
    mx = mx.scatter_reduce(0, rows[:, None].expand(-1, H), z.detach(), "amax")
    ex = torch.exp(z - mx[rows])
    s = torch.zeros((n, H), dtype=z.dtype, device=dev).index_add_(0, rows, ex)
    a = ex / s[rows]
    m = a
    if keep is not None:
        m = m * torch.as_tensor(np.asarray(keep)).to(device=dev, dtype=a.dtype) / (1.0 - p)
    if res_attn is not None:
        m = m * (1.0 - alpha) + res_attn * alpha
    return a, m


def aggregate_fp64(rowptr, colind, m, h):
    """out [n, H, F] = sum over row i's edges of m[e, h] * h[col[e], h, :]."""
    dev = h.device
    rows = _rows(rowptr).to(dev)
    cols = torch.as_tensor(np.asarray(colind, np.int64)).to(dev)
    out = torch.zeros((rowptr.shape[0] - 1,) + tuple(h.shape[1:]), dtype=h.dtype, device=dev)
    return out.index_add_(0, rows, m[:, :, None] * h[cols])


def conv_fp64(prm, rowptr, colind, etype, x, nhead, slope, alpha=0.0, res_attn=None, keep=None, p=0.0, act=None):
    """myGATConv.forward without feat_drop, on a CSR (rowptr, colind) with per-slot types: prm holds W, W_e, edge_emb,
    a_l, a_r, a_e and, with residual=True, residual.weight / residual.bias.  Returns (out, m)."""
    F_out = prm["W"].shape[1] // nhead
    h = (x @ prm["W"]).view(-1, nhead, F_out)
    e = (prm["edge_emb"] @ prm["W_e"]).view(-1, nhead, prm["edge_emb"].shape[1])
    h_l, h_r, h_e = (prm["a_l"] * h).sum(-1), (prm["a_r"] * h).sum(-1), (prm["a_e"] * e).sum(-1)
    _, m = hgn_attention_fp64(rowptr, colind, etype, h_l, h_r, h_e, slope, keep, p, res_attn, alpha)
    out = aggregate_fp64(rowptr, colind, m, h).reshape(h.shape[0], -1)
    if "residual.weight" in prm:
        out = out + x @ prm["residual.weight"].t() + prm["residual.bias"]
    if act is not None:
        out = act(out)
    return out, m


class HgnConvStandIn(torch.nn.Module):
    """myGATConv's parameters, attributes and forward signature (edge_feats, num_etypes, in_features, out_features,
    nhead; attn_drop, negative_slope, residual, activation, alpha), with the example's op sequence as its forward:
    gathers, LeakyReLU, a per-row softmax, dropout, the residual blend and a per-edge aggregation, in eager torch."""

    def __init__(self, edge_feats, num_etypes, in_features, out_features, nhead, attn_drop=0.5, negative_slope=0.2,
                 residual=False, activation=None, alpha=0.0):
        super().__init__()
        self.edge_feats, self.in_features, self.out_features, self.nhead = edge_feats, in_features, out_features, nhead
        self.edge_emb = torch.nn.Parameter(torch.zeros(num_etypes, edge_feats))
        self.W = torch.nn.Parameter(torch.zeros(in_features, out_features * nhead))
        self.W_e = torch.nn.Parameter(torch.zeros(edge_feats, edge_feats * nhead))
        self.a_l = torch.nn.Parameter(torch.zeros(1, nhead, out_features))
        self.a_r = torch.nn.Parameter(torch.zeros(1, nhead, out_features))
        self.a_e = torch.nn.Parameter(torch.zeros(1, nhead, edge_feats))
        self.feat_drop = torch.nn.Dropout(0.0)
        self.dropout = torch.nn.Dropout(attn_drop)
        self.leakyrelu = torch.nn.LeakyReLU(negative_slope)
        self.act = activation
        self.residual = torch.nn.Linear(in_features, out_features * nhead) if residual else None
        self.alpha = alpha
        for t in (self.a_l, self.a_r, self.a_e, self.W, self.W_e, self.edge_emb):
            b = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
            torch.nn.init.uniform_(t, -b, b)

    def forward(self, graph, x, res_attn=None):
        x = self.feat_drop(x)
        h = torch.matmul(x, self.W).view(-1, self.nhead, self.out_features)
        h[torch.isnan(h)] = 0.0
        e = torch.matmul(self.edge_emb, self.W_e).view(-1, self.nhead, self.edge_feats)
        row, col = graph.edge_index
        z = self.leakyrelu((self.a_l * h).sum(-1)[row] + (self.a_r * h).sum(-1)[col] +
                           (self.a_e * e).sum(-1)[graph.edge_type])
        n, H = h.shape[0], self.nhead
        mx = torch.full((n, H), -torch.inf, dtype=z.dtype, device=z.device)
        mx = mx.scatter_reduce(0, row[:, None].expand(-1, H), z.detach(), "amax")
        ex = torch.exp(z - mx[row])
        a = ex / torch.zeros((n, H), dtype=z.dtype, device=z.device).index_add_(0, row, ex)[row]
        a = self.dropout(a)
        if res_attn is not None:
            a = a * (1 - self.alpha) + res_attn * self.alpha
        out = torch.zeros_like(h).index_add_(0, row, a[:, :, None] * h[col]).view(n, -1)
        if self.residual is not None:
            out = out + self.residual(x)
        if self.act is not None:
            out = self.act(out)
        return out, a.detach()

"""The three caller layers named by the north star, on top of this package's spmm_utils mirror:
GCNLayer (cogdl/layers/gcn_layer.py:9-64), GATLayer (cogdl/layers/gat_layer.py:17-86) and
SAGELayer with Mean/Sum/Max aggregators (cogdl/layers/sage_layer.py:8-87).  Same constructor
arguments and forward(graph, x) semantics; dense GEMMs stay in cuBLAS (unchanged, SURVEY 8a15),
every sparse step goes through the sm_90a kernels.
"""
import math

import torch
import torch.nn as nn
import torch.nn.functional as F

from .utils.spmm_utils import spmm, EdgeSoftmax, MultiHeadSpMM, fused_gat_op, check_fused_gat
from .operators.scatter_max import ScatterMaxFunction
from .structure import csr_order, graph_operands


def _activation(name):
    if name is None:
        return None
    table = {"relu": nn.ReLU(), "elu": nn.ELU(), "gelu": nn.GELU(), "tanh": nn.Tanh(), "sigmoid": nn.Sigmoid(),
             "prelu": nn.PReLU(), "identity": nn.Identity()}
    if callable(name) and not isinstance(name, str):
        return name
    return table[name]


def _norm(name, channels):
    if name is None:
        return None
    if name == "batchnorm":
        return nn.BatchNorm1d(channels)
    if name == "layernorm":
        return nn.LayerNorm(channels)
    raise NotImplementedError(name)


class GCNLayer(nn.Module):
    """fused=True (opt-in): (A.X).W^T + (A.1) b^T with the dense transform and ReLU in the epilogue of the
    aggregation kernel (wgmma, cogdl_b200/csrc/fused_gcn.cu) instead of the reference order A.(X.W^T + b);
    taken when in_features == 128, out_features <= 128 and there is no norm layer between them."""

    def __init__(self, in_features, out_features, dropout=0.0, activation=None, residual=False, norm=None, bias=True,
                 fused=False):
        super().__init__()
        self.in_features, self.out_features = in_features, out_features
        self.fused, self._act_name = bool(fused), activation
        self.linear = nn.Linear(in_features, out_features, bias=bias)
        self.dropout = nn.Dropout(dropout) if dropout > 0 else None
        self.residual = nn.Linear(in_features, out_features) if residual else None
        self.act = _activation(activation)
        self.norm = _norm(norm, out_features)
        stdv = 1.0 / math.sqrt(out_features)
        nn.init.uniform_(self.linear.weight, -stdv, stdv)

    def forward(self, graph, x):
        from .operators import fused_gcn

        if (self.fused and self.norm is None and x.is_cuda and x.dtype == torch.float32
                and fused_gcn.supported(self.in_features, self.out_features)
                and (ops := graph_operands(graph)).out_norm is None and ops.in_norm is None):
            relu = self._act_name == "relu"
            out = fused_gcn.fused_gcn_layer(graph, x, self.linear.weight, self.linear.bias, relu=relu)
            if self.act is not None and not relu:
                out = self.act(out)
        else:
            out = spmm(graph, self.linear(x))      # dense first, then aggregate (gcn_layer.py:52-53)
            if self.norm is not None:
                out = self.norm(out)
            if self.act is not None:
                out = self.act(out)
        if self.residual is not None:
            out = out + self.residual(x)
        if self.dropout is not None:
            out = self.dropout(out)
        return out


class GATLayer(nn.Module):
    def __init__(self, in_feats, out_feats, nhead=1, alpha=0.2, attn_drop=0.5, activation=None, residual=False,
                 norm=None, fused=None):
        super().__init__()
        self.in_features, self.out_features, self.nhead, self.alpha = in_feats, out_feats, nhead, alpha
        self.W = nn.Parameter(torch.empty(in_feats, out_feats * nhead))
        self.a_l = nn.Parameter(torch.empty(1, nhead, out_feats))
        self.a_r = nn.Parameter(torch.empty(1, nhead, out_feats))
        self.edge_softmax = EdgeSoftmax()
        self.mhspmm = MultiHeadSpMM()
        self.dropout = nn.Dropout(attn_drop)
        self.leakyrelu = nn.LeakyReLU(alpha)
        self.act = _activation(activation)
        self.norm = _norm(norm, out_feats * nhead)
        self.residual = nn.Linear(in_feats, out_feats * nhead) if residual else None
        # None: the reference's rule (gat_layer.py:68); True/False forces it.  With True the attention dropout runs in
        # the fused kernels when training.
        self.fused = fused
        for t in (self.a_l, self.a_r, self.W):
            stdv = math.sqrt(6.0 / (t.size(-2) + t.size(-1)))
            t.data.uniform_(-stdv, stdv)

    def forward(self, graph, x):
        h = torch.matmul(x, self.W).view(-1, self.nhead, self.out_features)
        h = torch.nan_to_num(h, nan=0.0, posinf=float("inf"), neginf=float("-inf"))
        h_l = (self.a_l * h).sum(dim=-1)
        h_r = (self.a_r * h).sum(dim=-1)
        use_fused = self.fused
        if use_fused is None:
            use_fused = (self.dropout.p == 0.0 or not self.training) and check_fused_gat()
        p = self.dropout.p if self.training else 0.0
        if use_fused and p < 1.0:      # p = 1 drops everything: nn.Dropout on the unfused path
            out = fused_gat_op(h_l, h_r, graph, self.alpha, h, attn_drop=p)
            out = out.view(out.shape[0], -1)
        else:
            csr_order(graph)                             # edge_index in the order edge_softmax reads the logits in
            row, col = graph.edge_index
            e = self.leakyrelu(h_l[row] + h_r[col])      # [E, H]
            a = self.edge_softmax(graph, e)
            a = self.dropout(a)
            out = self.mhspmm(graph, a, h)
        if self.residual is not None:
            out = out + self.residual(x)
        if self.norm is not None:
            out = self.norm(out)
        if self.act is not None:
            out = self.act(out)
        return out


class MeanAggregator:
    def __call__(self, graph, x):
        graph.row_norm()
        return spmm(graph, x)


class SumAggregator:
    def __call__(self, graph, x):
        return spmm(graph, x)


class MaxAggregator:
    def __call__(self, graph, x):
        return ScatterMaxFunction.apply(graph.structure(), None, x)


class SAGELayer(nn.Module):
    """fused=True (opt-in): the aggregation and the neighbour half of `fc` in one kernel (cogdl_b200/csrc/fused_gcn.cu,
    wgmma epilogue), the self half and bias as one GEMM before it; the aggregated features are never written out.
    Taken for CUDA fp32 x with in_feats == 128, out_feats <= 128, x.shape[0] == the graph's rows, no out_norm on
    the graph and edge weights without grad (mean / sum); otherwise the unfused path runs."""

    def __init__(self, in_feats, out_feats, normalize=False, aggr="mean", dropout=0.0, norm=None, activation=None,
                 residual=False, fused=False):
        super().__init__()
        self.in_feats, self.out_feats = in_feats, out_feats
        self.fused, self._aggr_name, self._act_name = bool(fused), aggr, activation
        self.fc = nn.Linear(2 * in_feats, out_feats)
        self.normalize = normalize
        self.dropout = nn.Dropout(dropout) if dropout > 0 else None
        self.aggr = {"mean": MeanAggregator, "sum": SumAggregator, "max": MaxAggregator}[aggr]()
        self.act = _activation(activation)
        self.norm = _norm(norm, out_feats)
        self.residual = nn.Linear(in_feats, out_feats) if residual else None

    def _fused_applies(self, graph, x):
        from .operators import fused_sage

        if not (self.fused and x.is_cuda and x.dtype == torch.float32 and getattr(graph, "grb_adj", None) is None
                and fused_sage.supported(self.in_feats, self.out_feats) and x.shape[0] == graph.row_indptr.shape[0] - 1):
            return False
        if self._aggr_name == "mean":
            graph.row_norm()             # as MeanAggregator, before the norms are looked at
        ops = graph_operands(graph)
        return ops.out_norm is None and (self._aggr_name == "max" or not ops.val.requires_grad)

    def forward(self, graph, x):
        relu = False
        if self._fused_applies(graph, x):
            from .operators import fused_sage

            relu = self._act_name == "relu" and not self.normalize and self.norm is None
            out = fused_sage.fused_sage_layer(graph, x, self.fc.weight, self.fc.bias, self._aggr_name, relu=relu)
        else:
            out = self.aggr(graph, x)
            out = self.fc(torch.cat([x, out], dim=-1))
        if self.normalize:
            out = F.normalize(out, p=2.0, dim=-1)
        if self.norm is not None:
            out = self.norm(out)
        if self.act is not None and not relu:
            out = self.act(out)
        if self.residual is not None:
            out = out + self.residual(x)
        if self.dropout is not None:
            out = self.dropout(out)
        return out


# ---- the 2-layer models of the benchmark configs (cogdl/models/nn/{gcn,gat,graphsage}.py) ----
class GCN(nn.Module):
    def __init__(self, in_feats, hidden_size, out_feats, num_layers=2, dropout=0.5, activation="relu"):
        super().__init__()
        dims = [in_feats] + [hidden_size] * (num_layers - 1) + [out_feats]
        self.layers = nn.ModuleList(
            GCNLayer(dims[i], dims[i + 1], dropout=dropout if i != num_layers - 1 else 0,
                     activation=activation if i != num_layers - 1 else None) for i in range(num_layers))

    def forward(self, graph):
        graph.sym_norm()
        h = graph.x
        for layer in self.layers:
            h = layer(graph, h)
        return h


class GAT(nn.Module):
    def __init__(self, in_feats, hidden_size, out_feats, nhead=8, last_nhead=1, attn_drop=0.0, alpha=0.2, fused=None):
        super().__init__()
        self.l1 = GATLayer(in_feats, hidden_size, nhead=nhead, alpha=alpha, attn_drop=attn_drop, activation="elu", fused=fused)
        self.l2 = GATLayer(hidden_size * nhead, out_feats, nhead=last_nhead, alpha=alpha, attn_drop=attn_drop, fused=fused)

    def forward(self, graph):
        return self.l2(graph, self.l1(graph, graph.x))


class SAGE(nn.Module):
    def __init__(self, in_feats, hidden_size, out_feats, aggr="max", dropout=0.0, fused=False):
        super().__init__()
        self.l1 = SAGELayer(in_feats, hidden_size, aggr=aggr, dropout=dropout, activation="relu", fused=fused)
        self.l2 = SAGELayer(hidden_size, out_feats, aggr=aggr, fused=fused)

    def forward(self, graph):
        return self.l2(graph, self.l1(graph, graph.x))

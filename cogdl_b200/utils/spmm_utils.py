"""Dispatch layer -- same public names, signatures and semantics as cogdl/utils/spmm_utils.py:

    spmm(graph, x, actnn=False, fast_spmm=None, fast_spmm_cpu=None)            :85
    edge_softmax(graph, edge_val, csr_edge_softmax=None)                       :172
    mh_spmm(graph, attention, h, csrmhspmm=None, fast_spmm=None)               :201
    fused_gat_op(attn_row, attn_col, graph, negative_slope, in_feat, fused_gat_func=None)   :251
      (plus attn_drop=0.0, seed=None: attention dropout inside the fused kernels)
    modules SpMM / EdgeSoftmax / MultiHeadSpMM / FusedGATOp, registry CONFIGS  :4-14

Differences (deliberate):
  * one backend only -- the sm_90a kernels.  There is no `spmm_scatter` / `spmm_cpu` /
    `edge_softmax_val` fallback: a CPU tensor raises instead of silently taking a slow path;
  * the int32 CSR, hub plan and transpose come from `graph.structure()` (cached on the
    Adjacency) instead of `row_ptr.int(), col_indices.int()` on every call (:106);
  * `out_norm` / `in_norm` are applied around the kernel exactly as the reference does (:99-109).
`fast_spmm=` / `csr_edge_softmax=` / `csrmhspmm=` overrides are honoured (the reference's A/B
injection point); the `grb_adj` short-circuit (:86-91) is kept.
"""
import torch

from ..operators import csrspmm, csr_edge_softmax, csrmhspmm, fused_gat_func
from ..operators.spmm import SPMMFunction
from ..operators.edge_softmax import EdgeSoftmaxFunction
from ..operators.mhspmm import MHSPMMFunction
from ..operators.fused_gat import FusedGATFunction
from ..structure import csr_order, graph_operands

CONFIGS = {
    "fast_spmm": csrspmm,
    "csrmhspmm": csrmhspmm,
    "csr_edge_softmax": csr_edge_softmax,
    "fused_gat_func": fused_gat_func,
    "fast_spmm_cpu": None,     # no CPU path in this package
    "spmm_flag": True,
    "mh_spmm_flag": True,
    "fused_gat_flag": True,
    "spmm_cpu_flag": True,
}


def initialize_spmm():
    return None


def initialize_edge_softmax():
    return None


def initialize_fused_gat():
    return None


def check_fused_gat():
    return CONFIGS["fused_gat_func"] is not None


def spmm(graph, x, actnn=False, fast_spmm=None, fast_spmm_cpu=None):
    if getattr(graph, "grb_adj", None) is not None:
        if graph.grb_adj.is_sparse:
            return torch.sparse.mm(graph.grb_adj, x)
        return torch.mm(graph.grb_adj, x)
    if not x.is_cuda:
        raise RuntimeError("cogdl_b200.spmm: CPU tensors are not supported (no CPU fallback); move the graph and "
                           "features to an H100 device")
    custom = fast_spmm is not None and fast_spmm is not csrspmm
    if custom:
        rowptr, colind, val = csr_order(graph)
        out_norm, in_norm, sym = graph.out_norm, graph.in_norm, graph.is_symmetric()
    else:
        st, val, out_norm, in_norm, sym = graph_operands(graph)
    if out_norm is not None:
        x = out_norm.to(x.device) * x
    if x.dtype == torch.half:
        val = val.half()
    if custom:
        x = fast_spmm(rowptr.int(), colind.int(), x, val, sym, actnn=actnn)
    else:
        x = SPMMFunction.apply(st, None, x, val, sym, actnn)
    if in_norm is not None:
        x = in_norm.to(x.device) * x
    return x


class SpMM(torch.nn.Module):
    def __init__(self, actnn=False):
        super().__init__()
        self.actnn = actnn
        self.fast_spmm = CONFIGS["fast_spmm"]

    def forward(self, graph, x):
        return spmm(graph, x, self.actnn, self.fast_spmm)


def edge_softmax(graph, edge_val, csr_edge_softmax=None):
    """Softmax of edge_val [E] or [E, H] over each row's edges.  As in the reference, edge_val is taken in the graph's
    CSR order: a graph still held as COO is put in CSR order by this call, and its edge_index is CSR-ordered after it,
    so values formed from graph.edge_index before the call are read in an order they were not formed in."""
    if not edge_val.is_cuda:
        raise RuntimeError("cogdl_b200.edge_softmax: CPU tensors are not supported (no CPU fallback)")
    flat = edge_val.dim() == 1
    if flat:
        edge_val = edge_val.view(-1, 1)
    if csr_edge_softmax is not None and csr_edge_softmax is not CONFIGS["csr_edge_softmax"]:
        val = csr_edge_softmax(graph.row_indptr.int(), edge_val)
    else:
        val = EdgeSoftmaxFunction.apply(graph_operands(graph).st, edge_val)
    return val.view(-1) if flat else val


class EdgeSoftmax(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.csr_edge_softmax = CONFIGS["csr_edge_softmax"]

    def forward(self, graph, edge_val):
        return edge_softmax(graph, edge_val, self.csr_edge_softmax)


def mh_spmm(graph, attention, h, csrmhspmm=None, fast_spmm=None):
    """out[i, h] = sum over row i's edges p of attention[p, h] * h[col[p], h], flattened to [N, H * F].  attention
    [E, H] is taken in the graph's CSR order (as edge_softmax takes its values), for every H: a graph still held as COO
    is put in CSR order first, so the single-head path's edge weight is not reordered again inside local_graph()."""
    if not h.is_cuda:
        raise RuntimeError("cogdl_b200.mh_spmm: CPU tensors are not supported (no CPU fallback)")
    nhead = h.shape[1]
    if nhead > 1:
        if csrmhspmm is not None and csrmhspmm is not CONFIGS["csrmhspmm"]:
            h_prime = csrmhspmm(graph.row_indptr.int(), graph.col_indices.int(), h, attention)
        else:
            h_prime = MHSPMMFunction.apply(graph_operands(graph).st, None, h, attention)
        return h_prime.view(h_prime.shape[0], -1)
    # single head: SpMM with the attention as edge weight inside local_graph() (reference :210-214;
    # set_weight flips the symmetric flag, so the backward takes the transpose branch).
    graph_operands(graph)
    edge_weight = attention.view(-1)
    with graph.local_graph():
        graph.edge_weight = edge_weight
        return spmm(graph, h.squeeze(1), fast_spmm=fast_spmm)


class MultiHeadSpMM(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.spmm = CONFIGS["fast_spmm"]
        self.csrmhspmm = CONFIGS["csrmhspmm"]

    def forward(self, graph, attention, h):
        return mh_spmm(graph, attention, h, csrmhspmm=self.csrmhspmm, fast_spmm=self.spmm)


def fused_gat_op(attn_row, attn_col, graph, negative_slope, in_feat, fused_gat_func=None, attn_drop=0.0, seed=None):
    """attn_drop (0 <= attn_drop < 1): dropout on the attention, drawn inside the kernels; apply it when training
    only.  seed: the mask's 64-bit seed (None: drawn from torch's CPU generator, a fresh mask per call)."""
    if fused_gat_func is not None and fused_gat_func is not CONFIGS["fused_gat_func"]:
        if attn_drop:
            raise ValueError("attention dropout needs this package's fused GAT operator, not a custom fused_gat_func")
        rp, ci = graph.row_indptr.int(), graph.col_indices.int()
        return fused_gat_func(attn_row, attn_col, rp, ci, rp, ci, negative_slope, in_feat)
    return FusedGATFunction.apply(attn_row, attn_col, graph_operands(graph).st, None, None, None, negative_slope,
                                  in_feat, attn_drop, seed)


class FusedGATOp(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.fused_gat_func = CONFIGS["fused_gat_func"]

    def forward(self, attn_row, attn_col, graph, negative_slope, in_feat):
        return fused_gat_op(attn_row, attn_col, graph, negative_slope, in_feat, fused_gat_func=self.fused_gat_func)

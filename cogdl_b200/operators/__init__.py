"""Operator-level API, same names and argument meaning as `cogdl.operators.*`:

    csrspmm(rowptr, colind, x, csr_data, sym=False, actnn=False)   cogdl/operators/spmm.py:24
    csr_edge_softmax(rowptr, h)                                    cogdl/operators/edge_softmax.py:17
    csrmhspmm(rowptr, colind, feat, attention)                     cogdl/operators/mhspmm.py:34
    scatter_max(rowptr, colind, feat)                              cogdl/operators/scatter_max.py:17
    fused_gat_func(attn_row, attn_col, row_ptr, col_ind, col_ptr, row_ind, negative_slope, in_feat)
                                                                   cogdl/operators/fused_gat.py:40

Unlike the reference modules these never evaluate to None (no silent fallback): importing them
without the built CUDA library raises.
"""
from .spmm import csrspmm, SPMMFunction  # noqa: F401
from .edge_softmax import csr_edge_softmax, EdgeSoftmaxFunction  # noqa: F401
from .mhspmm import csrmhspmm, MHSPMMFunction  # noqa: F401
from .scatter_max import scatter_max, ScatterMaxFunction  # noqa: F401
from .fused_gat import fused_gat_func, FusedGATFunction  # noqa: F401
from .softmax_aggr import genconv_aggregate, GenconvEdgeFunction, SoftmaxAggrFunction  # noqa: F401
from .disen_routing import disen_routing, DisenRouteFunction  # noqa: F401
from .comp_aggr import compgcn_aggregate, CompAggrFunction  # noqa: F401
from .spspmm import spspmm, coo_spmm, SpSpMMFunction  # noqa: F401
from .spmm_residual import spmm_residual, SpmmResidualFunction  # noqa: F401
from .label_prop import label_propagate  # noqa: F401
from .gin import gin_aggregate, GinAggregateFunction  # noqa: F401
from .grand import random_propagate  # noqa: F401
from .rgcn import rgcn_aggregate, rgcn_conv, RgcnAggregateFunction, RgcnConvFunction  # noqa: F401
from .simple_hgn import hgn_attention, HgnAttentionFunction  # noqa: F401
from .readout import (  # noqa: F401
    batch_sum_pooling, batch_mean_pooling, batch_max_pooling, graph_readout, set2set_attention, sort_pool,
    ReadoutFunction, Set2SetAttentionFunction, SortPoolFunction,
)

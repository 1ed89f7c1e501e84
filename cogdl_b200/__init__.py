"""cogdl_b200 -- H100 (sm_90a) native implementation of CogDL's sparse message-passing hot path:
CSR SpMM (GE-SpMM), edge-softmax, multi-head SpMM / SDDMM and scatter_max, behind CogDL's own call
signatures.  Hand-written CUDA in cogdl_b200/csrc reached through the C ABI of
include/cogdl_b200.h; PyTorch only provides device memory, streams and torch.distributed.

There is no CPU or PyTorch fallback: importing this package loads libcogdl_b200.so and fails
loudly when it has not been built.
"""
from . import _cabi

_cabi.load()  # fail at import time, not at first use

from .structure import CSRStructure, HubPlan, structure_for  # noqa: E402,F401
from .data import Graph, Adjacency  # noqa: E402,F401
from .utils.spmm_utils import (  # noqa: E402,F401
    spmm, edge_softmax, mh_spmm, fused_gat_op, SpMM, EdgeSoftmax, MultiHeadSpMM, FusedGATOp, CONFIGS,
)
from .operators import csrspmm, csr_edge_softmax, csrmhspmm, scatter_max, fused_gat_func  # noqa: E402,F401
from .operators import genconv_aggregate, disen_routing, compgcn_aggregate, spspmm, coo_spmm  # noqa: E402,F401
from .operators import spmm_residual, label_propagate, gin_aggregate, random_propagate  # noqa: E402,F401
from .operators import rgcn_aggregate, rgcn_conv, hgn_attention  # noqa: E402,F401
from .operators import (  # noqa: E402,F401
    batch_sum_pooling, batch_mean_pooling, batch_max_pooling, graph_readout, set2set_attention, sort_pool,
)
from .structure import membership_for  # noqa: E402,F401
from .install import (  # noqa: E402,F401
    install, uninstall, uninstall_actnn, uninstall_appnp, uninstall_compgcn, uninstall_correct_smooth, uninstall_disengcn,
    uninstall_gat, uninstall_gcnii, uninstall_genconv, uninstall_gin, uninstall_grand, uninstall_readout, uninstall_rgcn,
    uninstall_spspmm, install_simple_hgn, uninstall_simple_hgn,
)
from . import sampling  # noqa: E402,F401

__version__ = "0.1.0"

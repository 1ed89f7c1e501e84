"""ctypes binding of libcogdl_b200.so (C ABI declared in include/cogdl_b200.h).

There is no fallback of any kind here: if the shared library is missing the import fails loudly,
and every entry point raises when the CUDA call fails.  PyTorch is only used by callers for
device memory and streams; this module passes raw pointers.
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "lib", "libcogdl_b200.so")
MAX_PANELS = 8   # COGDL_B200_MAX_PANELS: a hub plan holds MAX_PANELS arrival counters per chunk
COMP_OPS = {"mult": 0, "sub": 1, "copy": 2}   # COGDL_B200_COMP_MULT / _SUB / _COPY of cogdl_b200_comp_aggr_f32

OK, EINVAL, ECUDA, EDEVICE, ESCRATCH = 0, -1, -2, -3, -4


class CogdlB200Error(RuntimeError):
    def __init__(self, code, text):
        super().__init__(f"libcogdl_b200 error {code}: {text}")
        self.code = code


class HubPlanStruct(ctypes.Structure):
    """Mirror of cogdl_b200_hub_plan_t."""

    _fields_ = [
        ("chunk_edges", ctypes.c_int32),
        ("n_hub_rows", ctypes.c_int32),
        ("n_chunks", ctypes.c_int32),
        ("n_empty_rows", ctypes.c_int32),
        ("hub_rows", ctypes.c_void_p),
        ("chunks", ctypes.c_void_p),
        ("counters", ctypes.c_void_p),
        ("partials", ctypes.c_void_p),
        ("partials_bytes", ctypes.c_int64),
        ("seg_cost", ctypes.c_int32),
        ("n_segs", ctypes.c_int32),
        ("segs", ctypes.c_void_p),
        ("edge_row", ctypes.c_void_p),
        ("hub_degrees_host", ctypes.c_void_p),
    ]


_vp, _i64, _i32, _f32 = ctypes.c_void_p, ctypes.c_int64, ctypes.c_int32, ctypes.c_float
_plan_p = ctypes.POINTER(HubPlanStruct)

# name -> (restype, argtypes); must list every symbol declared in include/cogdl_b200.h
SIGNATURES = {
    "cogdl_b200_abi_version": (ctypes.c_int, []),
    "cogdl_b200_last_error": (ctypes.c_char_p, []),
    "cogdl_b200_check_device": (ctypes.c_int, []),
    "cogdl_b200_launch_count": (_i64, []),
    "cogdl_b200_last_kernel": (ctypes.c_char_p, []),
    "cogdl_b200_hub_plan_layout": (ctypes.c_int, [ctypes.POINTER(ctypes.c_int64), ctypes.c_int]),
    "cogdl_b200_hub_plan_count": (ctypes.c_int, [_vp, _i64, _i32, _i32, _vp, _vp]),
    "cogdl_b200_hub_plan_fill": (ctypes.c_int, [_vp, _i64, _i32, _i32, _vp, _vp, _vp, _vp, _vp]),
    "cogdl_b200_edge_rows": (ctypes.c_int, [_vp, _i64, _i64, _vp, _vp]),
    "cogdl_b200_spmm_scratch_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_spmm_csr_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_spmm_csr_f32_ex": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _i64, _i64, _i32, _plan_p, _vp]),
    "cogdl_b200_spmm_residual_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _f32, _f32, _vp, _vp, _i64, _i64, _i32,
                                                    _plan_p, _vp]),
    "cogdl_b200_label_prop_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _f32, _f32, _vp, _vp, _i32, _f32, _f32, _vp,
                                                 _i64, _i64, _i32, _plan_p, _vp]),
    "cogdl_b200_spmm_residual_dcoef_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _f32, _vp, _vp, _vp, _i64, _i64,
                                                          _i32, _plan_p, _vp]),
    "cogdl_b200_spmm_accum_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _vp, _i32, _f32, _vp, _i64, _i64, _i32,
                                                 _plan_p, _vp]),
    "cogdl_b200_spmm_csr_f16": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_spmm_csr_f32_2src": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_spmm_csr_f32_peers": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _vp, _i32, _i32, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_sddmm_csr_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_csr2csc_workspace_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_csr2csc": (ctypes.c_int, [_vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _i64, _vp]),
    "cogdl_b200_gather_rows_f32": (ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _vp]),
    "cogdl_b200_edge_softmax_scratch_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_gat_attn_bwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _f32, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_edge_colsum_scratch_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_edge_colsum_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_edge_softmax_fwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_edge_softmax_bwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_mhspmm_scratch_bytes": (_i64, [_i64, _i64, _i64]),
    "cogdl_b200_mhspmm_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_mhsddmm_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_scatter_max_scratch_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_scatter_max_fwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_scatter_max_bwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp]),
    "cogdl_b200_sort_pool_max_k": (_i64, []),
    "cogdl_b200_sort_pool_select": (ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _vp, _vp, _vp, _vp, _vp]),
    "cogdl_b200_gat_fwd_scratch_bytes": (_i64, [_i64, _i64, _i64]),
    "cogdl_b200_gat_fwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _f32, _vp, _vp, _i64, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_gat_fwd_dropout_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _f32, ctypes.c_uint64, ctypes.c_uint64, _f32,
                                                      _vp, _vp, _i64, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_mhspmm_dropout_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _f32, _vp, _i64, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_gat_attn_bwd_dropout_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _f32, _f32, _vp, _vp, _i64, _i64,
                                                           _plan_p, _vp]),
    "cogdl_b200_gcn_fused_supported": (ctypes.c_int, [_i64, _i64]),
    "cogdl_b200_gcn_fused_scratch_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_gcn_fused_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _plan_p, _vp]),
    "cogdl_b200_sage_fused_scratch_bytes": (_i64, [_i64, _i64, _i32]),
    "cogdl_b200_sage_fused_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i32, _i32,
                                                 _plan_p, _vp]),
    "cogdl_b200_softmax_aggr_scratch_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_softmax_aggr_fwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _f32, _vp, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_softmax_aggr_bwd_scratch_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_softmax_aggr_bwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _f32, _vp, _vp, _vp, _vp, _vp, _i64, _i64,
                                                       _plan_p, _vp]),
    "cogdl_b200_genconv_edge_fwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _f32, _vp, _vp, _vp, _i64, _i64,
                                                       _plan_p, _vp]),
    "cogdl_b200_genconv_edge_dw_scratch_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_genconv_edge_bwd_scratch_bytes": (_i64, [_i64, _i64, _i32]),
    "cogdl_b200_genconv_edge_bwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _vp, _f32, _vp, _vp, _vp, _vp, _vp,
                                                       _vp, _i64, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_disen_route_scratch_bytes": (_i64, [_i64, _i64, _i64]),
    "cogdl_b200_disen_route_fwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _f32,
                                                      _plan_p, _vp]),
    "cogdl_b200_disen_route_bwd_f32": (ctypes.c_int, [_vp, _vp, _plan_p, _vp, _vp, _plan_p, _vp, _vp, _vp, _vp, _vp, _vp,
                                                      _vp, _vp, _vp, _vp, _i64, _i64, _i64, _i64, _f32, _vp]),
    "cogdl_b200_comp_aggr_scratch_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_comp_aggr_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i64, _vp, _i64, _i64, _i32, _plan_p,
                                                _vp]),
    "cogdl_b200_rgcn_aggr_scratch_bytes": (_i64, [_i64, _i64, _i64]),
    "cogdl_b200_rgcn_aggr_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _i64, _vp, _i32, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_rgcn_edge_dot_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_hgn_max_table": (_i64, []),
    "cogdl_b200_hgn_attn_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _i64, _f32, ctypes.c_uint64, ctypes.c_uint64,
                                               _f32, _vp, _f32, _vp, _vp, _i64, _i64, _plan_p, _vp]),
    "cogdl_b200_hgn_attn_bwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _i64, _f32, _f32, _vp, _vp, _i64,
                                                   _i64, _plan_p, _vp]),
    "cogdl_b200_spgemm_scratch_bytes":(_i64, [_i64, _i64, _i64]),
    "cogdl_b200_spgemm_count": (ctypes.c_int, [_vp, _vp, _i64, _i64, _vp, _vp, _i64, _i64, _vp, ctypes.POINTER(_i64), _vp,
                                               _i64, _vp]),
    "cogdl_b200_spgemm_fill_f32": (ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp,
                                                  _i64, _vp]),
    "cogdl_b200_spgemm_bwd_f32": (ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _i64, _i64, _vp, _vp, _vp, _vp,
                                                 _vp, _vp, _vp, _vp, _vp]),
    "cogdl_b200_coo2csr_workspace_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_coo2csr_index": (ctypes.c_int, [_vp, _i64, _i64, _vp, _vp, _vp, _i64, _vp]),
    "cogdl_b200_narrow_i64_i32": (ctypes.c_int, [_vp, _vp, _i64, _vp]),
    "cogdl_b200_sample_draw": (ctypes.c_uint64, [ctypes.c_uint64, _i64, _i64]),
    "cogdl_b200_sample_workspace_bytes": (_i64, [_i64, _i64]),
    "cogdl_b200_sample_adj_count": (ctypes.c_int, [_vp, _vp, _i64, _i64, _i32, _vp, _vp, _i64, _vp]),
    "cogdl_b200_sample_adj_fill": (ctypes.c_int, [_vp, _vp, _vp, _i64, _i64, _i64, _i32, ctypes.c_uint64, _vp, _i64, _vp,
                                                  _vp, _vp, _vp, _vp, _vp, _i64, _vp]),
    "cogdl_b200_subgraph_count": (ctypes.c_int, [_vp, _vp, _vp, _i64, _vp, _vp, _vp, _i64, _vp]),
    "cogdl_b200_subgraph_fill": (ctypes.c_int, [_vp, _vp, _vp, _i64, _vp, _vp, _vp, _vp, _vp]),
    "cogdl_b200_actnn_minmax_f32": (ctypes.c_int, [_vp, _i64, _i64, _i32, _vp, _vp, _vp]),
    "cogdl_b200_actnn_pack_f32": (ctypes.c_int, [_vp, _i64, _i64, _i32, _vp, _i32, _vp, _i32, ctypes.c_uint64, _vp, _vp,
                                                 _vp, _vp]),
    "cogdl_b200_actnn_unpack_f32": (ctypes.c_int, [_vp, _i64, _i64, _i32, _vp, _i32, _vp, _vp, _vp, _vp, _vp]),
    "cogdl_b200_actnn_relu_fwd_f32": (ctypes.c_int, [_vp, _i64, _vp, _vp, _vp]),
    "cogdl_b200_actnn_relu_bwd_f32": (ctypes.c_int, [_vp, _vp, _i64, _vp, _vp]),
    "cogdl_b200_actnn_dropout_fwd_f32": (ctypes.c_int, [_vp, _i64, _f32, ctypes.c_uint64, ctypes.c_uint64, _vp, _vp,
                                                        _vp]),
    "cogdl_b200_actnn_dropout_bwd_f32": (ctypes.c_int, [_vp, _vp, _i64, _f32, _vp, _vp]),
    "cogdl_b200_actnn_bits_scratch_bytes": (_i64, [_i64]),
    "cogdl_b200_actnn_bits": (ctypes.c_int, [_vp, _i64, _i32, _i64, _vp, _vp, _i64, _vp]),
}

_lib = None


def load():
    """Load libcogdl_b200.so.  Raises ImportError if it has not been built."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise ImportError(
                f"{LIB_PATH} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "or `make -C cogdl_b200/csrc` (nvcc, sm_90a). cogdl_b200 has no CPU / PyTorch fallback."
            )
        lib = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)  # AttributeError here = header/library mismatch: fail loudly
            fn.restype = res
            fn.argtypes = args
        if lib.cogdl_b200_abi_version() != 6:
            raise ImportError("libcogdl_b200.so ABI version mismatch")
        # the ctypes mirror of cogdl_b200_hub_plan_t must have the library's layout, field for field
        want = [ctypes.sizeof(HubPlanStruct)] + [getattr(HubPlanStruct, n).offset for n, _ in HubPlanStruct._fields_]
        got = (ctypes.c_int64 * 32)()
        k = lib.cogdl_b200_hub_plan_layout(got, 32)
        if list(got[:k]) != want:
            raise ImportError(f"cogdl_b200_hub_plan_t layout mismatch: library {list(got[:k])}, ctypes mirror {want}")
        _lib = lib
    return _lib


def last_error():
    return load().cogdl_b200_last_error().decode("utf-8", "replace")


def check(rc):
    if rc != OK:
        raise CogdlB200Error(rc, last_error())


def call(name, *args):
    """Call an int-status entry point and raise on failure."""
    check(getattr(load(), name)(*args))


def launch_count():
    return int(load().cogdl_b200_launch_count())


def last_kernel():
    return load().cogdl_b200_last_kernel().decode("utf-8", "replace")

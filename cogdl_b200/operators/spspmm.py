"""torch_sparse's spspmm (sparse x sparse) and spmm (COO sparse x dense) on this package's sm_90a kernels.

CogDL's GTN, SRGCN and Graph U-Net import `from torch_sparse import spspmm[, spmm]` at module level
(cogdl/models/nn/gtn.py:7, srgcn.py:6, cogdl/utils/srgcn_utils.py:7, graph_unet.py:9); install(spspmm=True) binds these
two functions under those names.  Both take torch_sparse's signatures and return values:

    spspmm(indexA, valueA, indexB, valueB, m, k, n, coalesced=False) -> (index [2, nnz] int64, value [nnz] fp32)
    coo_spmm(index, value, m, n, matrix)                               -> [m, F]

The product C = A.B runs in cogdl_b200/csrc/spgemm.cu (count -> one host read -> fill), and its value gradients
in the same file.  COO inputs may be in any order and hold duplicates: they are sorted by (row, col) on the device and
duplicates are summed in input order, once per index tensor (the structure is cached on its storage and version).
`coalesced` is accepted for torch_sparse's signature and changes nothing: the input is always sorted and merged.
"""
import torch

from .. import _cabi
from ..structure import _ptr, _stream, coo_structure_for, require_cuda
from .spmm import SPMMFunction


def _spgemm_forward(ca, cb, va, vb):
    """(rowptrC int32 [m+1], colC int32 [nnz], valC fp32 [nnz]) of C = A.B on the merged CSRs of ca and cb."""
    a, b = ca.csr, cb.csr
    dev = a.device
    lib = _cabi.load()
    with torch.cuda.device(dev):
        scratch = torch.empty(int(lib.cogdl_b200_spgemm_scratch_bytes(a.n_rows, a.n_cols, b.n_cols)), dtype=torch.uint8,
                              device=dev)
        rowptr = torch.empty(a.n_rows + 1, dtype=torch.int32, device=dev)
        nnz = _cabi.ctypes.c_int64(0)
        _cabi.call("cogdl_b200_spgemm_count", _ptr(a.rowptr), _ptr(a.colind), a.n_rows, a.n_cols, _ptr(b.rowptr),
                   _ptr(b.colind), b.n_rows, b.n_cols, _ptr(rowptr), _cabi.ctypes.byref(nnz), _ptr(scratch),
                   scratch.numel(), _stream(dev))
        col = torch.empty(nnz.value, dtype=torch.int32, device=dev)
        val = torch.empty(nnz.value, dtype=torch.float32, device=dev)
        _cabi.call("cogdl_b200_spgemm_fill_f32", _ptr(a.rowptr), _ptr(a.colind), _ptr(va), a.n_rows, a.n_cols,
                   _ptr(b.rowptr), _ptr(b.colind), _ptr(vb), b.n_rows, b.n_cols, _ptr(rowptr), _ptr(col), _ptr(val),
                   _ptr(scratch), scratch.numel(), _stream(dev))
    return rowptr, col, val


class SpSpMMFunction(torch.autograd.Function):
    """Values of C = A.B for the CooStructures ca (m x k) and cb (k x n), with gradients for both input value
    tensors: dA[(i,k)] = sum_j B[k,j] dC[i,j], dB[(k,j)] = sum_i A[i,k] dC[i,j], handed to every merged input
    entry.  Returns (rowptrC, colC, valC); only valC is differentiable."""

    @staticmethod
    def forward(ctx, ca, cb, value_a, value_b):
        va, vb = ca.merge(value_a), cb.merge(value_b)
        rowptr, col, val = _spgemm_forward(ca, cb, va, vb)
        ctx.ca, ctx.cb = ca, cb
        ctx.save_for_backward(va, vb, rowptr, col)
        ctx.mark_non_differentiable(rowptr, col)
        return rowptr, col, val

    @staticmethod
    def backward(ctx, _g_rowptr, _g_col, g):
        va, vb, rowptr, col = ctx.saved_tensors
        ca, cb = ctx.ca, ctx.cb
        a, b = ca.csr, cb.csr
        want_a, want_b = ctx.needs_input_grad[2], ctx.needs_input_grad[3]
        if not (want_a or want_b):
            return None, None, None, None
        dev = a.device
        g = g.contiguous().float()
        with torch.cuda.device(dev):
            da = torch.empty(a.nnz, dtype=torch.float32, device=dev) if want_a else None
            db = torch.empty(b.nnz, dtype=torch.float32, device=dev) if want_b else None
            at, perm = a.csc() if want_b else (None, None)
            _cabi.call("cogdl_b200_spgemm_bwd_f32", _ptr(a.rowptr), _ptr(a.colind), _ptr(va), a.n_rows, a.n_cols,
                       _ptr(b.rowptr), _ptr(b.colind), _ptr(vb), b.n_rows, b.n_cols, _ptr(rowptr), _ptr(col), _ptr(g),
                       _ptr(at.rowptr) if want_b else None, _ptr(at.colind) if want_b else None, _ptr(perm),
                       _ptr(da), _ptr(db), _stream(dev))
        return (None, None, ca.spread(da) if want_a else None, cb.spread(db) if want_b else None)


def _check_values(index, value, name):
    if value.dim() != 1 or value.numel() != index.shape[1]:
        raise ValueError(f"{name} must be [E={index.shape[1]}], got {tuple(value.shape)}")
    if not value.is_floating_point():
        raise TypeError(f"{name} must be floating point, got {value.dtype}")


def spspmm(indexA, valueA, indexB, valueB, m, k, n, coalesced=False):
    """torch_sparse.spspmm: C = A.B with A (indexA, valueA) m x k and B (indexB, valueB) k x n in COO form (any order,
    duplicates summed).  Returns (index [2, nnz] int64 in row-major sorted order, value [nnz] fp32); (i, j) is in C when
    some product A[i,k] B[k,j] exists, even if the values sum to 0.  Gradients reach valueA and valueB.  CUDA tensors
    only; an index outside the matrix raises ValueError."""
    del coalesced
    require_cuda(indexA, valueA, indexB, valueB)
    _check_values(indexA, valueA, "valueA")
    _check_values(indexB, valueB, "valueB")
    ca, cb = coo_structure_for(indexA, m, k), coo_structure_for(indexB, k, n)
    rowptr, col, val = SpSpMMFunction.apply(ca, cb, valueA, valueB)
    counts = (rowptr[1:] - rowptr[:-1]).long()
    row = torch.repeat_interleave(torch.arange(int(m), device=col.device), counts, output_size=col.numel())
    return torch.stack([row, col.long()]), val


def coo_spmm(index, value, m, n, matrix):
    """torch_sparse.spmm: out [m, F] = A @ matrix with A (index, value) an m x n COO (any order, duplicates summed),
    matrix [n, F] fp32.  Runs the CSR SpMM on the stable COO -> CSR of the index (cached on the index tensor), with
    gradients for value (SDDMM) and matrix (SpMM over the cached transpose)."""
    require_cuda(index, value, matrix)
    _check_values(index, value, "value")
    if matrix.dim() != 2 or matrix.shape[0] != int(n):
        raise ValueError(f"matrix must be [{int(n)}, F], got {tuple(matrix.shape)}")
    if matrix.dtype != torch.float32:
        raise TypeError(f"matrix must be float32, got {matrix.dtype}")
    st, reindex = coo_structure_for(index, m, n).coo_csr()
    return SPMMFunction.apply(st, None, matrix, value.float()[reindex], False)

"""Thin tensor-level wrappers over the C ABI: allocate outputs with torch, pass raw pointers and
the current stream.  No autograd here (see the sibling modules)."""
import torch

from .. import _cabi
from ..structure import CSRStructure, _ptr, _stream, require_cuda


def _f32c(t, name):
    if t.dtype != torch.float32:
        raise TypeError(f"{name} must be float32, got {t.dtype}")
    return t.contiguous()


def _scratch(family, st: CSRStructure, *shape):
    """Bytes of plan scratch an entry of `family` needs on st's hub plan, as the library's
    cogdl_b200_<family>_scratch_bytes(n_chunks, *shape) gives it; 0 when st has no plan."""
    if st.chunk_edges <= 0:
        return 0
    return int(getattr(_cabi.load(), f"cogdl_b200_{family}_scratch_bytes")(st.plan.n_chunks, *shape))


def _launch(symbol, st: CSRStructure, partial_bytes, *args):
    """symbol(*args, plan, stream) on st's device: plan is st's hub plan with partial_bytes of scratch, which stays
    alive until the call returns; stream is the device's current stream."""
    with torch.cuda.device(st.device):
        plan, keep = st.plan_struct(partial_bytes)
        _cabi.call(symbol, *args, plan, _stream(st.device))


def _spmm_out(st: CSRStructure, val, x, out=None):
    """What every SpMM wrapper shares: checks val against the nnz and x for being 2-D and allocates Y [n_rows, F] in
    x's dtype (unless given `out`).  Returns y."""
    if x.dim() != 2:
        raise ValueError("x must be [n_src, F]")
    if val is not None and val.numel() != st.nnz:
        raise ValueError(f"edge values have {val.numel()} entries, CSR has {st.nnz}")
    return torch.empty((st.n_rows, x.shape[1]), dtype=x.dtype, device=x.device) if out is None else out


def _epilogue_args(st: CSRStructure, val, x, z, row_scale):
    """The operands of an SpMM-epilogue entry (residual, label propagation), checked and made fp32 contiguous:
    (device, val [nnz], x [n_src, F], z [n_rows, F], row_scale [n_rows]); val, z and row_scale may be None."""
    dev = require_cuda(x, z, val, row_scale)
    x = _f32c(x, "x")
    if x.dim() != 2:
        raise ValueError("x must be [n_src, F]")
    z = None if z is None else _f32c(z, "z")
    row_scale = None if row_scale is None else _f32c(row_scale, "row_scale").view(-1)
    val = None if val is None else _f32c(val, "edge values").view(-1)
    if z is not None and z.shape != (st.n_rows, x.shape[1]):
        raise ValueError(f"z must be [{st.n_rows}, {x.shape[1]}], got {tuple(z.shape)}")
    if row_scale is not None and row_scale.numel() != st.n_rows:
        raise ValueError(f"row_scale has {row_scale.numel()} entries, the CSR has {st.n_rows} rows")
    return dev, val, x, z, row_scale


def _spmm_epilogue_raw(symbol, st: CSRStructure, val, x, z, a, b, row_scale, extra=(), panels=0, out=None):
    """One launch of an SpMM-epilogue entry: symbol(rowptr, colind, val, x, n_src, z, a, b, row_scale, *extra, y,
    n_rows, F, panels, plan, stream), with the operands of _epilogue_args.  Returns y (`out` when given)."""
    _, val, x, z, row_scale = _epilogue_args(st, val, x, z, row_scale)
    y = _spmm_out(st, val, x, out)
    _launch(symbol, st, _scratch("spmm", st, x.shape[1]), _ptr(st.rowptr), _ptr(st.colind), _ptr(val), _ptr(x),
            x.shape[0], _ptr(z), float(a), float(b), _ptr(row_scale), *extra, _ptr(y), st.n_rows, x.shape[1], int(panels))
    return y


def spmm_raw(st: CSRStructure, val, x, panels=0):
    """Y = A @ X with A = (st, val).  x: [n_src, F] fp32 or fp16; val: [nnz] or None.
    panels: column panels of X for the fp32 kernel (0 = chosen from X's size against the L2; the output
    does not depend on it)."""
    require_cuda(x, val)
    x = x.contiguous()
    val = None if val is None else val.contiguous().view(-1)
    y = _spmm_out(st, val, x)
    need = _scratch("spmm", st, x.shape[1])
    if x.dtype == torch.float32:
        if val is not None and val.dtype != torch.float32:
            val = val.float()
        _launch("cogdl_b200_spmm_csr_f32_ex", st, need, _ptr(st.rowptr), _ptr(st.colind), _ptr(val), _ptr(x),
                x.shape[0], _ptr(y), st.n_rows, x.shape[1], int(panels))
    elif x.dtype == torch.float16:
        if val is not None and val.dtype != torch.float16:
            val = val.half()
        _launch("cogdl_b200_spmm_csr_f16", st, need, _ptr(st.rowptr), _ptr(st.colind), _ptr(val), _ptr(x), _ptr(y),
                st.n_rows, x.shape[1])
    else:
        raise TypeError(f"spmm supports float32 / float16 features, got {x.dtype}")
    return y


def spmm_2src_raw(st: CSRStructure, val, x0, x1):
    """Partitioned SpMM: columns < x0.shape[0] read x0, the others read x1 (halo rows)."""
    require_cuda(x0, x1, val)
    x0, x1 = _f32c(x0, "x0"), _f32c(x1, "x1")
    if x1.shape[1] != x0.shape[1]:
        raise ValueError("x0 / x1 feature widths differ")
    val = None if val is None else _f32c(val, "val").view(-1)
    y = _spmm_out(st, val, x0)
    x1p = x1 if x1.numel() > 0 else x0
    _launch("cogdl_b200_spmm_csr_f32_2src", st, _scratch("spmm", st, x0.shape[1]), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(val), _ptr(x0), x0.shape[0], _ptr(x1p), _ptr(y), st.n_rows, x0.shape[1])
    return y


def spmm_residual_raw(st: CSRStructure, val, x, z, a, b, row_scale=None, panels=0):
    """Y = a * (row_scale[:, None] * (A @ x)) + b * z with A = (st, val); z and row_scale may be None.  x [n_src, F]
    fp32, z [n_rows, F] fp32, row_scale [n_rows] fp32, val [nnz] fp32 or None.  a and b are rounded to fp32.
    panels: column panels of x, as for spmm_raw (0 = chosen by the library)."""
    return _spmm_epilogue_raw("cogdl_b200_spmm_residual_f32", st, val, x, z, a, b, row_scale, panels=panels)


def spmm_adjoint_raw(st: CSRStructure, val, g, sym, a=None):
    """A^T @ g, times a when a is given, for A = (st, val): the feature gradient of every SpMM-based operator.  Runs
    over A itself when sym (A is symmetric), else over the cached transpose with the edge values permuted to it.
    Without a it is spmm_raw (fp32 or fp16 g); with a it is spmm_residual_raw with b = 0 (fp32)."""
    if not sym:
        st, perm = st.csc()
        val = None if val is None else gather_rows_raw(perm, val.detach().float())
    if a is None:
        return spmm_raw(st, val, g)
    return spmm_residual_raw(st, val, g, None, a, 0.0)


def sddmm_raw(st: CSRStructure, d1, d2):
    dev = require_cuda(d1, d2)
    d1, d2 = _f32c(d1, "d1"), _f32c(d2, "d2")
    out = torch.empty(st.nnz, dtype=torch.float32, device=dev)
    _launch("cogdl_b200_sddmm_csr_f32", st, 0, _ptr(st.rowptr), _ptr(st.colind), _ptr(d1), _ptr(d2), _ptr(out),
            st.n_rows, d1.shape[1])
    return out


def gather_rows_raw(perm, x):
    dev = require_cuda(perm, x)
    x = _f32c(x, "x")
    H = 1 if x.dim() == 1 else x.shape[1]
    with torch.cuda.device(dev):
        out = torch.empty((perm.numel(),) + tuple(x.shape[1:]), dtype=torch.float32, device=dev)
        _cabi.call("cogdl_b200_gather_rows_f32", _ptr(perm), _ptr(x), _ptr(out), perm.numel(), H, _stream(dev))
    return out


def edge_softmax_fwd_raw(st: CSRStructure, e):
    require_cuda(e)
    e = _f32c(e, "edge values")
    if e.dim() != 2 or e.shape[0] != st.nnz:
        raise ValueError(f"edge values must be [nnz={st.nnz}, H], got {tuple(e.shape)}")
    out = torch.empty_like(e)
    _launch("cogdl_b200_edge_softmax_fwd_f32", st, _scratch("edge_softmax", st, e.shape[1]), _ptr(st.rowptr), _ptr(e),
            _ptr(out), st.n_rows, e.shape[1])
    return out


def edge_softmax_bwd_raw(st: CSRStructure, y, g):
    require_cuda(y, g)
    y, g = _f32c(y, "y"), _f32c(g, "g")
    out = torch.empty_like(y)
    _launch("cogdl_b200_edge_softmax_bwd_f32", st, _scratch("edge_softmax", st, y.shape[1]), _ptr(st.rowptr), _ptr(y),
            _ptr(g), _ptr(out), st.n_rows, y.shape[1])
    return out


def mhspmm_raw(st: CSRStructure, att, feat, perm=None, drop_scale=None):
    """out[i,h,:] = sum_p att[P(p),h] * feat[col[p],h,:];  feat [n_src,H,F], att [nnz,H].
    drop_scale: att is the signed attention of gat_fwd_raw(drop=...): sign-bit entries count as 0, the others as
    att * drop_scale."""
    dev = require_cuda(att, feat, perm)
    att, feat = _f32c(att, "attention"), _f32c(feat, "feat")
    if feat.dim() != 3:
        raise ValueError("feat must be [N, H, F]")
    H, F = feat.shape[1], feat.shape[2]
    if att.shape != (st.nnz, H):
        raise ValueError(f"attention must be [nnz={st.nnz}, H={H}], got {tuple(att.shape)}")
    out = torch.empty((st.n_rows, H, F), dtype=torch.float32, device=dev)
    need = _scratch("mhspmm", st, H, F)
    if drop_scale is None:
        _launch("cogdl_b200_mhspmm_f32", st, need, _ptr(st.rowptr), _ptr(st.colind), _ptr(perm), _ptr(att), _ptr(feat),
                _ptr(out), st.n_rows, H, F)
    else:
        _launch("cogdl_b200_mhspmm_dropout_f32", st, need, _ptr(st.rowptr), _ptr(st.colind), _ptr(perm), _ptr(att),
                _ptr(feat), float(drop_scale), _ptr(out), st.n_rows, H, F)
    return out


def mhsddmm_raw(st: CSRStructure, grad, feat):
    dev = require_cuda(grad, feat)
    grad, feat = _f32c(grad, "grad"), _f32c(feat, "feat")
    H, F = feat.shape[1], feat.shape[2]
    out = torch.empty((st.nnz, H), dtype=torch.float32, device=dev)
    _launch("cogdl_b200_mhsddmm_f32", st, 0, _ptr(st.rowptr), _ptr(st.colind), _ptr(grad), _ptr(feat), _ptr(out),
            st.n_rows, H, F)
    return out


def scatter_max_fwd_raw(st: CSRStructure, x):
    dev = require_cuda(x)
    x = _f32c(x, "feat")
    F = x.shape[1]
    out = torch.empty((st.n_rows, F), dtype=torch.float32, device=dev)
    arg = torch.empty((st.n_rows, F), dtype=torch.int32, device=dev)
    _launch("cogdl_b200_scatter_max_fwd_f32", st, _scratch("scatter_max", st, F), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(x), _ptr(out), _ptr(arg), st.n_rows, F)
    return out, arg


def scatter_max_bwd_raw(grad, argmax, n_src):
    dev = require_cuda(grad, argmax)
    grad = _f32c(grad, "grad")
    n, F = grad.shape
    with torch.cuda.device(dev):
        gx = torch.empty((n_src, F), dtype=torch.float32, device=dev)
        _cabi.call("cogdl_b200_scatter_max_bwd_f32", _ptr(grad), _ptr(argmax), _ptr(gx), n, n_src, F, _stream(dev))
    return gx


def sort_pool_max_k():
    """The largest k of the SortPool readout (COGDL_B200_SORT_POOL_MAX_K)."""
    return int(_cabi.load().cogdl_b200_sort_pool_max_k())


def sort_pool_select_raw(st: CSRStructure, keys, k):
    """SortPool's per-graph top-k over the membership CSR st (row g: graph g's nodes) by keys [st.n_cols] fp32 (read as
    their bit patterns): (idx [st.n_rows, k] int32, the selection CSR of st.n_rows * k rows and st.n_cols columns, run
    without a hub plan); see cogdl_b200_sort_pool_select."""
    dev = require_cuda(keys)
    k = int(k)
    if not 1 <= k <= sort_pool_max_k():
        raise ValueError(f"k = {k}; the SortPool readout takes 1 to {sort_pool_max_k()}")
    if keys.dtype != torch.float32 or keys.numel() != st.n_cols:
        raise ValueError(f"keys must be float32 [{st.n_cols}], got {keys.dtype} {tuple(keys.shape)}")
    bits = keys.contiguous().view(torch.int32)
    B = st.n_rows
    m = (st.rowptr[1:] - st.rowptr[:-1]).clamp(max=k)
    off = (torch.cumsum(m, 0) - m).to(torch.int32)
    idx = torch.empty((B, k), dtype=torch.int32, device=dev)
    sel_rowptr = torch.empty(B * k + 1, dtype=torch.int32, device=dev)
    sel_colind = torch.empty(min(B * k, st.n_cols), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _cabi.call("cogdl_b200_sort_pool_select", _ptr(st.rowptr), _ptr(st.colind), _ptr(bits), st.n_cols, B, k,
                   _ptr(off), _ptr(idx), _ptr(sel_rowptr), _ptr(sel_colind), _stream(dev))
    return idx, CSRStructure(sel_rowptr, sel_colind, n_cols=st.n_cols, chunk_edges=0)


def attn_dropout_args(p):
    """(drop_below, scale) of attention dropout with probability p, 0 <= p < 1: an (edge, head) is kept iff
    draw(seed, edge, head) >= drop_below = floor(p * 2^64), a kept attention is multiplied by scale = 1 / (1 - p)."""
    p = float(p)
    if not 0.0 <= p < 1.0:
        raise ValueError(f"attention dropout must be in [0, 1), got {p}")
    return int(p * 2.0 ** 64), 1.0 / (1.0 - p)


def gat_fwd_raw(st: CSRStructure, h_l, h_r, feat, slope, want_att, drop=None):
    """(out [n_rows,H,F], att [nnz,H]).  drop = (seed, drop_below, scale): attention dropout, and att is returned
    signed (sign bit set on the dropped entries; see cogdl_b200_gat_fwd_dropout_f32)."""
    dev = require_cuda(h_l, h_r, feat)
    h_l, h_r, feat = _f32c(h_l, "attn_row"), _f32c(h_r, "attn_col"), _f32c(feat, "in_feat")
    H, F = feat.shape[1], feat.shape[2]
    out = torch.empty((st.n_rows, H, F), dtype=torch.float32, device=dev)
    att = torch.empty((st.nnz, H), dtype=torch.float32, device=dev)   # output for training, scratch otherwise
    need = _scratch("gat_fwd", st, H, F)
    if drop is None:
        _launch("cogdl_b200_gat_fwd_f32", st, need, _ptr(st.rowptr), _ptr(st.colind), _ptr(h_l), _ptr(h_r), _ptr(feat),
                float(slope), _ptr(out), _ptr(att), st.n_rows, H, F)
    else:
        seed, drop_below, scale = drop
        _launch("cogdl_b200_gat_fwd_dropout_f32", st, need, _ptr(st.rowptr), _ptr(st.colind), _ptr(h_l), _ptr(h_r),
                _ptr(feat), float(slope), int(seed), int(drop_below), float(scale), _ptr(out), _ptr(att), st.n_rows, H,
                F)
    return out, att


def gat_attn_bwd_raw(st: CSRStructure, att, d_att, h_l, h_r, slope, drop_scale=None):
    """(d_edge [nnz,H], g_row [n_rows,H]): softmax backward * LeakyReLU' and its row sums in one pass.
    drop_scale: att is the signed attention of gat_fwd_raw(drop=...) and d_att the gradient after the dropout."""
    dev = require_cuda(att, d_att, h_l, h_r)
    att, d_att, h_l, h_r = _f32c(att, "att"), _f32c(d_att, "d_att"), _f32c(h_l, "attn_row"), _f32c(h_r, "attn_col")
    H = att.shape[1]
    d_edge = torch.empty_like(att)
    g_row = torch.empty((st.n_rows, H), dtype=torch.float32, device=dev)
    need = _scratch("edge_softmax", st, H)
    if drop_scale is None:
        _launch("cogdl_b200_gat_attn_bwd_f32", st, need, _ptr(st.rowptr), _ptr(st.colind), _ptr(att), _ptr(d_att),
                _ptr(h_l), _ptr(h_r), float(slope), _ptr(d_edge), _ptr(g_row), st.n_rows, H)
    else:
        _launch("cogdl_b200_gat_attn_bwd_dropout_f32", st, need, _ptr(st.rowptr), _ptr(st.colind), _ptr(att),
                _ptr(d_att), _ptr(h_l), _ptr(h_r), float(slope), float(drop_scale), _ptr(d_edge), _ptr(g_row),
                st.n_rows, H)
    return d_edge, g_row


def _sa_scratch(st, F):
    """Plan scratch of the softmax aggregation's forward, which the GENConv edge encoder's forward shares."""
    return _scratch("softmax_aggr", st, F)


def _sa_check(st, x, beta, edge_term, n_x_rows):
    """Shared argument checks of the softmax aggregation: [n_x_rows, F] fp32 x, [nnz, F] fp32 edge term, a
    one-element fp32 beta on x's device."""
    require_cuda(x, beta, edge_term)
    x = _f32c(x, "x")
    if x.dim() != 2 or x.shape[0] != n_x_rows:
        raise ValueError(f"x must be [{n_x_rows}, F], got {tuple(x.shape)}")
    beta = _f32c(beta, "beta").reshape(-1)
    if beta.numel() != 1:
        raise ValueError(f"beta must hold one value, got {beta.numel()}")
    if edge_term is not None:
        edge_term = _f32c(edge_term, "edge term")
        if edge_term.shape != (st.nnz, x.shape[1]):
            raise ValueError(f"edge term must be [nnz={st.nnz}, F={x.shape[1]}], got {tuple(edge_term.shape)}")
    return x, beta, edge_term


def softmax_aggr_fwd_raw(st: CSRStructure, x, beta, eps, edge_term=None, want_lse=False, want_q=False):
    """GENConv softmax aggregation: out[i] = sum_e softmax_e(beta m_e) m_e, m_e = relu(x[col_e] + edge_term[e]) + eps.
    x [n_cols, F], beta a one-element CUDA tensor (read on the device), edge_term [nnz, F] in CSR order or None.
    Returns (out, lse2, q): lse2 (base-2 log-sum-exp of the logits, for the backward) and q (sum_e w_e m_e^2, for
    d beta) are [n_rows, F] when asked for, else None."""
    dev = require_cuda(x)
    x, beta, edge_term = _sa_check(st, x, beta, edge_term, st.n_cols)
    F = x.shape[1]
    out = torch.empty((st.n_rows, F), dtype=torch.float32, device=dev)
    lse2 = torch.empty_like(out) if want_lse else None
    q = torch.empty_like(out) if want_q else None
    _launch("cogdl_b200_softmax_aggr_fwd_f32", st, _sa_scratch(st, F), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(x), _ptr(edge_term), _ptr(beta), float(eps), _ptr(out), _ptr(lse2), _ptr(q), st.n_rows, F)
    return out, lse2, q


def softmax_aggr_bwd_raw(st: CSRStructure, x, beta, eps, g, out, lse2, edge_term=None, want_edge_grad=True):
    """(dx [n_cols, F], d_edge_term [nnz, F] or None) of softmax_aggr_fwd_raw, over the cached transpose of st."""
    dev = require_cuda(x, g, out, lse2)
    x, beta, edge_term = _sa_check(st, x, beta, edge_term, st.n_cols)
    F = x.shape[1]
    g, out, lse2 = _f32c(g, "grad"), _f32c(out, "out"), _f32c(lse2, "lse2")
    for name, t in (("grad", g), ("out", out), ("lse2", lse2)):
        if t.shape != (st.n_rows, F):
            raise ValueError(f"{name} must be [{st.n_rows}, {F}], got {tuple(t.shape)}")
    st_t, perm = st.csc()
    dx = torch.empty_like(x)
    da = torch.empty_like(edge_term) if edge_term is not None and want_edge_grad else None
    _launch("cogdl_b200_softmax_aggr_bwd_f32", st_t, _scratch("softmax_aggr_bwd", st_t, F), _ptr(st_t.rowptr),
            _ptr(st_t.colind), _ptr(perm), _ptr(x), _ptr(edge_term), _ptr(beta), float(eps), _ptr(g), _ptr(out),
            _ptr(lse2), _ptr(dx), _ptr(da), st_t.n_rows, F)
    return dx, da


GENCONV_EDGE_MAX_D = 16   # widest edge feature of cogdl_b200/csrc/genconv_edge.cu


def _ge_check(st, x, attr, w):
    """Shared argument checks of the edge-encoder aggregation: attr [nnz, D] and w [F, D] fp32 on x's device,
    1 <= D <= 16.  Returns (attr, w) contiguous."""
    require_cuda(attr, w)
    attr, w = _f32c(attr, "edge_attr"), _f32c(w, "edge encoder weight")
    if attr.dim() != 2 or attr.shape[0] != st.nnz:
        raise ValueError(f"edge_attr must be [nnz={st.nnz}, D], got {tuple(attr.shape)}")
    D = attr.shape[1]
    if not 1 <= D <= GENCONV_EDGE_MAX_D:
        raise ValueError(f"edge_attr has D = {D} features; the fused edge encoder takes 1 to {GENCONV_EDGE_MAX_D}")
    if w.shape != (x.shape[1], D):
        raise ValueError(f"edge encoder weight must be [F={x.shape[1]}, D={D}], got {tuple(w.shape)}")
    return attr, w


def genconv_edge_fwd_raw(st: CSRStructure, x, attr, w, beta, eps, want_lse=False, want_q=False):
    """softmax_aggr_fwd_raw with the edge term attr @ w.T formed inside the kernel (no [nnz, F] tensor): attr
    [nnz, D] in CSR order, w [F, D] (nn.Linear layout), 1 <= D <= 16.  Returns (out, lse2, q) as softmax_aggr_fwd_raw."""
    dev = require_cuda(x)
    x, beta, _ = _sa_check(st, x, beta, None, st.n_cols)
    attr, w = _ge_check(st, x, attr, w)
    F = x.shape[1]
    out = torch.empty((st.n_rows, F), dtype=torch.float32, device=dev)
    lse2 = torch.empty_like(out) if want_lse else None
    q = torch.empty_like(out) if want_q else None
    _launch("cogdl_b200_genconv_edge_fwd_f32", st, _sa_scratch(st, F), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(x), _ptr(attr), _ptr(w), attr.shape[1], _ptr(beta), float(eps), _ptr(out), _ptr(lse2), _ptr(q),
            st.n_rows, F)
    return out, lse2, q


def genconv_edge_bwd_raw(st: CSRStructure, x, attr, w, beta, eps, g, out, lse2, want_dx=True, want_dw=True):
    """(dx [n_cols, F] or None, dw [F, D] or None) of genconv_edge_fwd_raw, over the cached transpose of st.  dw is
    summed in a fixed order without float atomics (bit-identical run to run)."""
    dev = require_cuda(x, g, out, lse2)
    x, beta, _ = _sa_check(st, x, beta, None, st.n_cols)
    attr, w = _ge_check(st, x, attr, w)
    F, D = x.shape[1], attr.shape[1]
    g, out, lse2 = _f32c(g, "grad"), _f32c(out, "out"), _f32c(lse2, "lse2")
    for name, t in (("grad", g), ("out", out), ("lse2", lse2)):
        if t.shape != (st.n_rows, F):
            raise ValueError(f"{name} must be [{st.n_rows}, {F}], got {tuple(t.shape)}")
    if not (want_dx or want_dw):
        return None, None
    st_t, perm = st.csc()
    dx = torch.empty_like(x) if want_dx else None
    dw = torch.empty((F, D), dtype=torch.float32, device=dev) if want_dw else None
    n_scr = int(_cabi.load().cogdl_b200_genconv_edge_dw_scratch_bytes(F, D)) if want_dw else 0
    scratch = torch.empty(n_scr // 4, dtype=torch.float32, device=dev) if want_dw else None
    _launch("cogdl_b200_genconv_edge_bwd_f32", st_t, _scratch("genconv_edge_bwd", st_t, F, int(bool(want_dx))),
            _ptr(st_t.rowptr), _ptr(st_t.colind), _ptr(perm), _ptr(x), _ptr(attr), _ptr(w), D, _ptr(beta), float(eps),
            _ptr(g), _ptr(out), _ptr(lse2), _ptr(dx), _ptr(dw), _ptr(scratch), n_scr, st_t.n_rows, F)
    return dx, dw


def _dr_check(st, K, **feats):
    """[n, F] fp32 contiguous features of one routing step, all on one device."""
    require_cuda(*feats.values())
    out = []
    for name, t in feats.items():
        t = _f32c(t, name)
        if t.dim() != 2 or t.shape[0] != st.n_rows:
            raise ValueError(f"{name} must be [{st.n_rows}, F], got {tuple(t.shape)}")
        out.append(t)
    F = out[0].shape[1]
    if any(t.shape[1] != F for t in out):
        raise ValueError("the routing features must have the same width")
    if K < 1 or F % K:
        raise ValueError(f"F={F} is not a multiple of K={K}")
    return out, F


def disen_route_fwd_raw(st: CSRStructure, q, c, K, tau, want_saved=False):
    """One DisenGCN routing step: out[i,k] = u / |u|, u = sum_e softmax_e(q[i,k] . c[j,k] / tau) c[j,k] + c[i,k]
    over row i's edges, per channel k of d = F/K columns.  Returns (out [n, F], lse2 [n, K], r [n, K]); lse2 (base-2
    log-sum-exp of the logits) and r (|u|) are for the backward and None unless want_saved."""
    dev = require_cuda(q, c)
    (q, c), F = _dr_check(st, K, q=q, c=c)
    n = st.n_rows
    out = torch.empty((n, F), dtype=torch.float32, device=dev)
    lse2 = torch.empty((n, K), dtype=torch.float32, device=dev) if want_saved else None
    r = torch.empty_like(lse2) if want_saved else None
    _launch("cogdl_b200_disen_route_fwd_f32", st, _scratch("disen_route", st, F, K), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(q), _ptr(c), _ptr(out), _ptr(lse2), _ptr(r), n, st.n_cols, F, K, float(tau))
    return out, lse2, r


def disen_route_bwd_raw(st: CSRStructure, q, c, K, tau, g, out, lse2, r):
    """(dq, dc) [n, F] of disen_route_fwd_raw given g = dL/dout: a row pass over st and a column pass over its
    cached transpose.  Scratch g_u [n, F] and D [n, K]; nothing edge-sized."""
    dev = require_cuda(q, c, g, out, lse2, r)
    (q, c, g, out), F = _dr_check(st, K, q=q, c=c, grad=g, out=out)
    lse2, r = _f32c(lse2, "lse2"), _f32c(r, "r")
    n = st.n_rows
    for name, t in (("lse2", lse2), ("r", r)):
        if t.shape != (n, K):
            raise ValueError(f"{name} must be [{n}, {K}], got {tuple(t.shape)}")
    st_t, _ = st.csc()
    with torch.cuda.device(dev):
        dq, dc, gu = torch.empty_like(q), torch.empty_like(q), torch.empty_like(q)
        D = torch.empty_like(lse2)
        plan, keep = st.plan_struct(_scratch("disen_route", st, F, K))
        plan_t, keep_t = st_t.plan_struct(_scratch("disen_route", st_t, F, K))
        _cabi.call("cogdl_b200_disen_route_bwd_f32", _ptr(st.rowptr), _ptr(st.colind), plan, _ptr(st_t.rowptr),
                   _ptr(st_t.colind), plan_t, _ptr(q), _ptr(c), _ptr(g), _ptr(out), _ptr(lse2), _ptr(r), _ptr(gu),
                   _ptr(D), _ptr(dq), _ptr(dc), n, st.n_cols, F, K, float(tau), _stream(dev))
        del keep, keep_t
    return dq, dc


def edge_colsum_raw(st_t: CSRStructure, perm, e):
    """out[j,h] = sum of e[p,h] over the edges p whose column is j (st_t = cached transpose, perm its permutation)."""
    dev = require_cuda(perm, e)
    e = _f32c(e, "edge values")
    H = e.shape[1]
    out = torch.empty((st_t.n_rows, H), dtype=torch.float32, device=dev)
    _launch("cogdl_b200_edge_colsum_f32", st_t, _scratch("edge_colsum", st_t, H), _ptr(st_t.rowptr), _ptr(perm), _ptr(e),
            _ptr(out), st_t.n_rows, H)
    return out


def comp_aggr_raw(st: CSRStructure, idx2, w, a, b, op):
    """CompGCN composition aggregation: y[i] = sum over row i's slots q of w[q] * phi(a[colind[q]], b[idx2[q]]), with
    phi = a * b ("mult"), a - b ("sub") or a ("copy": idx2 and b unused).  a [*, F] and b [*, F] fp32; w [nnz] fp32;
    idx2 [nnz] int32.  Returns y [st.n_rows, F]; rows without slots are zero."""
    dev = require_cuda(a, b, w, idx2)
    if op not in _cabi.COMP_OPS:
        raise ValueError(f"unknown composition op {op!r} (one of {sorted(_cabi.COMP_OPS)})")
    two = op != "copy"
    a = _f32c(a, "a")
    b = _f32c(b, "b") if two else None
    if a.dim() != 2 or (two and (b.dim() != 2 or b.shape[1] != a.shape[1])):
        raise ValueError(f"a and b must be [*, F] of one width, got {tuple(a.shape)} and "
                         f"{None if b is None else tuple(b.shape)}")
    F = a.shape[1]
    if F <= 0:
        raise ValueError("F must be positive")
    w = _f32c(w, "w").view(-1)
    if w.numel() != st.nnz or (two and idx2.numel() != st.nnz):
        raise ValueError(f"per-slot arrays must have {st.nnz} entries")
    if two and idx2.dtype != torch.int32:
        raise TypeError(f"idx2 must be int32, got {idx2.dtype}")
    if st.nnz == 0:
        return torch.zeros((st.n_rows, F), dtype=torch.float32, device=dev)
    y = torch.empty((st.n_rows, F), dtype=torch.float32, device=dev)
    _launch("cogdl_b200_comp_aggr_f32", st, _scratch("comp_aggr", st, F), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(idx2.contiguous() if two else None), _ptr(w), _ptr(a), a.shape[0], _ptr(b), b.shape[0] if two else 0,
            _ptr(y), st.n_rows, F, _cabi.COMP_OPS[op])
    return y


def spmm_residual_dcoef_raw(st: CSRStructure, val, x, z, a, b_dev, row_scale=None, panels=0):
    """Y = a * (row_scale[:, None] * (A @ x)) + b * z with b = b_dev[0], a one-element fp32 tensor on x's device that
    the kernel reads (no host synchronisation); otherwise as spmm_residual_raw.  z may be None (b_dev is then unused)."""
    _, val, x, z, row_scale = _epilogue_args(st, val, x, z, row_scale)
    require_cuda(x, b_dev)
    b_dev = _f32c(b_dev, "b_dev").view(-1)
    if b_dev.numel() != 1:
        raise ValueError(f"b_dev must hold one value, got {b_dev.numel()}")
    y = _spmm_out(st, val, x)
    _launch("cogdl_b200_spmm_residual_dcoef_f32", st, _scratch("spmm", st, x.shape[1]), _ptr(st.rowptr),
            _ptr(st.colind), _ptr(val), _ptr(x), x.shape[0], _ptr(z), float(a), _ptr(b_dev), _ptr(row_scale), _ptr(y),
            st.n_rows, x.shape[1], int(panels))
    return y


def spmm_accum_raw(st: CSRStructure, val, x, acc, acc_in=None, row_scale=None, last=False, scale=1.0, xn=None,
                   panels=0):
    """One hop of GRAND's propagation: xn = row_scale[:, None] * (A @ x) (not stored when last) and, in place,
    acc = acc_in + xn (acc_in None: acc itself), then acc * scale when last.  x [n_src, F], acc and acc_in [n_rows, F],
    row_scale [n_rows], all fp32; scale is rounded to fp32.  xn: a preallocated [n_rows, F] fp32 output, allocated when
    None and not last.  Returns xn (None when last)."""
    _, val, x, acc_in, row_scale = _epilogue_args(st, val, x, acc_in, row_scale)
    require_cuda(x, acc, xn)
    for name, t in (("acc", acc), ("xn", xn)):
        if t is not None and (t.dtype != torch.float32 or not t.is_contiguous() or t.shape != (st.n_rows, x.shape[1])):
            raise ValueError(f"{name} must be a contiguous float32 [{st.n_rows}, {x.shape[1]}] tensor")
    out = _spmm_out(st, val, x, acc if last else xn)   # acc: nothing to allocate on the last hop
    _launch("cogdl_b200_spmm_accum_f32", st, _scratch("spmm", st, x.shape[1]), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(val), _ptr(x), x.shape[0], _ptr(row_scale), _ptr(acc_in), _ptr(acc), int(bool(last)), float(scale),
            _ptr(None if last else out), st.n_rows, x.shape[1], int(panels))
    return None if last else out


def rgcn_aggr_raw(st: CSRStructure, etype, w, coef, x, per_basis=False):
    """R-GCN fan-out aggregation: y[i, b] = sum over row i's slots q of fl(w[q] * coef[etype[q], b]) * x[colind[q]]
    (per_basis: x is [*, B, F] and basis b gathers x[colind[q], b]).  etype [nnz] int32 with every type in
    [0, coef.shape[0]) (the caller's to guarantee), w [nnz] fp32, coef [T, B] fp32, x [*, F] fp32.  Returns y
    [st.n_rows, B, F]; rows without slots are zero."""
    dev = require_cuda(x, w, coef, etype)
    x, w, coef = _f32c(x, "x"), _f32c(w, "w").view(-1), _f32c(coef, "coef")
    if coef.dim() != 2:
        raise ValueError(f"coef must be [T, B], got {tuple(coef.shape)}")
    B = coef.shape[1]
    if per_basis and (x.dim() != 3 or x.shape[1] != B):
        raise ValueError(f"x must be [*, {B}, F] for the per-basis form, got {tuple(x.shape)}")
    if not per_basis and x.dim() != 2:
        raise ValueError(f"x must be [*, F], got {tuple(x.shape)}")
    F = x.shape[-1]
    if F <= 0 or B <= 0:
        raise ValueError("F and B must be positive")
    if w.numel() != st.nnz or etype.numel() != st.nnz:
        raise ValueError(f"per-slot arrays must have {st.nnz} entries")
    if etype.dtype != torch.int32:
        raise TypeError(f"etype must be int32, got {etype.dtype}")
    if st.nnz == 0:
        return torch.zeros((st.n_rows, B, F), dtype=torch.float32, device=dev)
    y = torch.empty((st.n_rows, B, F), dtype=torch.float32, device=dev)
    _launch("cogdl_b200_rgcn_aggr_f32", st, _scratch("rgcn_aggr", st, B, F), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(etype.contiguous()), _ptr(w), _ptr(coef), B, _ptr(x), int(bool(per_basis)), _ptr(y), st.n_rows, F)
    return y


def rgcn_edge_dot_raw(st: CSRStructure, w, g, x):
    """p[q, b] = fl(w[q] * <g[row_q, b], x[colind[q]]>) for every slot q: g [st.n_rows, B, F], x [*, F], w [nnz], all
    fp32.  Returns p [nnz, B] in slot order."""
    dev = require_cuda(w, g, x)
    w, g, x = _f32c(w, "w").view(-1), _f32c(g, "g"), _f32c(x, "x")
    if g.dim() != 3 or g.shape[0] != st.n_rows or x.dim() != 2 or x.shape[1] != g.shape[2]:
        raise ValueError(f"g must be [{st.n_rows}, B, F] and x [*, F], got {tuple(g.shape)} and {tuple(x.shape)}")
    if w.numel() != st.nnz:
        raise ValueError(f"w must have {st.nnz} entries")
    B, F = g.shape[1], g.shape[2]
    p = torch.empty((st.nnz, B), dtype=torch.float32, device=dev)
    if st.nnz == 0:
        return p
    _launch("cogdl_b200_rgcn_edge_dot_f32", st, 0, _ptr(st.rowptr), _ptr(st.colind), _ptr(w), _ptr(g), _ptr(x), _ptr(p),
            st.n_rows, B, F)
    return p


def hgn_max_table():
    """The largest T * H of a Simple-HGN type table (h_e is staged in shared memory by the kernels)."""
    return int(_cabi.load().cogdl_b200_hgn_max_table())


def _hgn_table(st, etype, h_e, H):
    """The type operands of the Simple-HGN kernels, checked: etype [nnz] int32, h_e [T, H] fp32 with T * H within the
    kernels' table.  Types in [0, T) are the caller's to guarantee (RgcnStructure checks them)."""
    h_e = _f32c(h_e, "h_e")
    if h_e.dim() != 2 or h_e.shape[1] != H:
        raise ValueError(f"h_e must be [T, H={H}], got {tuple(h_e.shape)}")
    if h_e.shape[0] * H > hgn_max_table() or h_e.shape[0] < 1:
        raise ValueError(f"h_e is [T={h_e.shape[0]}, H={H}]; the fused attention takes T * H from 1 to {hgn_max_table()}")
    if etype.dtype != torch.int32 or etype.numel() != st.nnz:
        raise ValueError(f"etype must be int32 [nnz={st.nnz}], got {etype.dtype} {tuple(etype.shape)}")
    return etype.contiguous(), h_e


def hgn_attn_raw(st: CSRStructure, etype, h_l, h_r, h_e, slope, want_att, drop=None, res_attn=None, alpha=0.0):
    """Simple-HGN attention stage: (mix [nnz, H], att [nnz, H] or None).  a = softmax_row(leakyrelu(h_l[row] + h_r[col]
    + h_e[etype])); att is a with the sign bit set on the dropped entries (when want_att); mix = (1 - alpha) * (dropped
    ? 0 : a * scale) + alpha * res_attn (res_attn None: no blend).  drop = (seed, drop_below, scale) as for
    gat_fwd_raw, None for no dropout."""
    dev = require_cuda(h_l, h_r, h_e, etype, res_attn)
    h_l, h_r = _f32c(h_l, "h_l"), _f32c(h_r, "h_r")
    H = h_l.shape[1]
    etype, h_e = _hgn_table(st, etype, h_e, H)
    if res_attn is not None:
        res_attn = _f32c(res_attn, "res_attn")
        if res_attn.shape != (st.nnz, H):
            raise ValueError(f"res_attn must be [nnz={st.nnz}, H={H}], got {tuple(res_attn.shape)}")
    seed, drop_below, scale = (0, 0, 1.0) if drop is None else drop
    mix = torch.empty((st.nnz, H), dtype=torch.float32, device=dev)
    att = torch.empty_like(mix) if want_att else None
    _launch("cogdl_b200_hgn_attn_f32", st, _scratch("edge_softmax", st, H), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(etype), _ptr(h_l), _ptr(h_r), _ptr(h_e), h_e.shape[0], float(slope), int(seed), int(drop_below),
            float(scale), _ptr(res_attn), float(alpha), _ptr(att), _ptr(mix), st.n_rows, H)
    return mix, att


def hgn_attn_bwd_raw(st: CSRStructure, etype, att, d_mix, h_l, h_r, h_e, slope, grad_scale):
    """(d_edge [nnz, H], g_row [n_rows, H]) of hgn_attn_raw: the softmax backward on |att| with g = kept ? d_mix *
    grad_scale : 0, times the typed LeakyReLU', and its row sums, in one pass."""
    dev = require_cuda(att, d_mix, h_l, h_r, h_e, etype)
    att, d_mix, h_l, h_r = _f32c(att, "att"), _f32c(d_mix, "d_mix"), _f32c(h_l, "h_l"), _f32c(h_r, "h_r")
    H = att.shape[1]
    etype, h_e = _hgn_table(st, etype, h_e, H)
    d_edge = torch.empty_like(att)
    g_row = torch.empty((st.n_rows, H), dtype=torch.float32, device=dev)
    _launch("cogdl_b200_hgn_attn_bwd_f32", st, _scratch("edge_softmax", st, H), _ptr(st.rowptr), _ptr(st.colind),
            _ptr(etype), _ptr(att), _ptr(d_mix), _ptr(h_l), _ptr(h_r), _ptr(h_e), h_e.shape[0], float(slope),
            float(grad_scale), _ptr(d_edge), _ptr(g_row), st.n_rows, H)
    return d_edge, g_row

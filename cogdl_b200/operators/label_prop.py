"""label_propagate -- the propagation loop of Correct & Smooth, one SpMM launch per step.

The reference (cogdl/models/nn/correct_smooth.py, outcome_correlation) runs, nprop times,

    result = alpha * spmm(g, result)
    result += (1 - alpha) * labels          (or `+= labels` without the alpha term)
    result = post_step(result)              torch.clamp(result, lower, upper), or result[nid] = labels[nid]

Here each step is one cogdl_b200_label_prop_f32 launch: the in_norm, both scalings, the addition, the clamp and the
reset of the pinned rows run in the SpMM's store, with the same fp32 roundings in the same order, so the result is
bit-identical to that loop run with this package's spmm.  The steps ping-pong between two buffers, with no host
synchronisation between them."""
import torch

from .. import _cabi
from ..structure import _ptr, _stream, graph_operands, require_cuda, unsupported_operands
from ._raw import _epilogue_args, _scratch, _spmm_epilogue_raw, _spmm_out


def label_prop_raw(st, val, x, z, a, b, row_scale=None, pin=None, clamp=None, panels=0, out=None):
    """One step: Y = pin ? z : clamp(a * (row_scale * (A @ x)) + b * z, *clamp), with A = (st, val).  x [n_src, F]
    fp32; z [n_rows, F] fp32 or None; row_scale [n_rows] fp32 or None; pin [n_rows] uint8 or None (needs z); clamp
    (lo, hi) or None; val [nnz] fp32 or None.  a, b, lo and hi are rounded to fp32.  out: a preallocated [n_rows, F]
    fp32 Y (must not overlap x, z or row_scale)."""
    require_cuda(x, pin)
    if pin is not None and (pin.dtype != torch.uint8 or pin.numel() != st.n_rows):
        raise ValueError(f"pin must be [{st.n_rows}] uint8")
    lo, hi = (0.0, 0.0) if clamp is None else (float(clamp[0]), float(clamp[1]))
    return _spmm_epilogue_raw("cogdl_b200_label_prop_f32", st, val, x, z, a, b, row_scale,
                              (_ptr(pin), int(clamp is not None), lo, hi), panels, out)


def pin_mask(n, pinned, device):
    """The [n] uint8 mask of label_prop_raw with a 1 at every index of `pinned` (an int64 node index or a bool mask,
    as `x[nid]` takes it), built on the device."""
    pin = torch.zeros(n, dtype=torch.uint8, device=device)
    pin[pinned.to(device)] = 1
    return pin


def label_propagate(graph, labels, alpha, nprop, lower=None, upper=None, pinned=None, alpha_term=True):
    """outcome_correlation(graph, labels, alpha, nprop, post_step, alpha_term) for fp32 CUDA labels [N, C], with
    post_step torch.clamp(x, lower, upper) when both bounds are given, and the reset x[pinned] = labels[pinned] when
    `pinned` (a node index) is.  The graph is taken as cogdl_b200.spmm takes it: the cached int32 CSR and hub plan,
    out_norm applied to x first and in_norm to the SpMM's rows (here inside the kernel).  Forward only.  The result is
    bit-identical to the reference loop run with this package's spmm; nprop = 0 returns labels.clone()."""
    err = unsupported_operands(graph, labels, entry="label_propagate", what="labels")
    if err is not None:
        raise err
    if (lower is None) != (upper is None):
        raise ValueError("label_propagate clamps to [lower, upper]: give both bounds or neither")
    if lower is not None and pinned is not None:
        raise ValueError("label_propagate: one post step at a time, the clamp or the pinned rows")
    st, val, out_norm, r, _ = graph_operands(graph)
    if torch.is_grad_enabled() and (labels.requires_grad or (val is not None and val.requires_grad)):
        raise RuntimeError("label_propagate is forward only: call it under torch.no_grad() or on inputs that do not "
                           "require grad")
    nprop = int(nprop)
    if nprop < 0:
        raise ValueError(f"nprop must be >= 0, got {nprop}")
    if nprop == 0:
        return labels.clone()
    if labels.shape[0] != st.n_rows or st.n_cols != st.n_rows:
        raise ValueError(f"labels must be [{st.n_rows}, C] on a square graph, got {tuple(labels.shape)}")
    dev, val, labels, _, r = _epilogue_args(st, val, labels, None, None if r is None else r.to(labels.device))
    out_norm = None if out_norm is None else out_norm.to(dev)
    pin = None if pinned is None else pin_mask(st.n_rows, pinned, dev)
    lo, hi = (0.0, 0.0) if lower is None else (float(lower), float(upper))
    a, b = float(alpha), float((1 - alpha) if alpha_term else 1.0)
    n, F = labels.shape
    step = _cabi.load().cogdl_b200_label_prop_f32
    with torch.cuda.device(dev):
        y = _spmm_out(st, val, labels)
        plan, keep = st.plan_struct(_scratch("spmm", st, F))
        bufs = (y, torch.empty_like(y))
        stream = _stream(dev)
        x = labels
        for k in range(nprop):
            if out_norm is not None:
                x = out_norm * x
            y = bufs[k & 1]
            _cabi.check(step(_ptr(st.rowptr), _ptr(st.colind), _ptr(val), _ptr(x), n, _ptr(labels), a, b, _ptr(r),
                             _ptr(pin), int(lower is not None), lo, hi, _ptr(y), n, F, 0, plan, stream))
            x = y
        del keep
    return x

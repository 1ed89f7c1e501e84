"""Helpers the test modules share: the device fixture, operand placement, bit views, error metrics, plan forms and the
hub plan's arrival-counter check.  A module takes the fixture with `from tests.gpu_util import dev`."""
import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def dev():
    """cuda:0 after the library has loaded and accepted the device; TF32 matmuls off (torch's default), so an fp32
    reference computed with torch on the device is fp32."""
    assert torch.cuda.is_available()
    import cogdl_b200

    assert cogdl_b200._cabi.load().cogdl_b200_check_device() == 0, cogdl_b200._cabi.last_error()
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


def T(a, dev):
    """a on the device: a numpy array (or anything np.ascontiguousarray takes) as a contiguous copy of its dtype, a
    tensor moved as it is."""
    if isinstance(a, torch.Tensor):
        return a.to(dev)
    return torch.from_numpy(np.ascontiguousarray(a)).to(dev)


def misaligned(t):
    """A contiguous copy of t whose data starts one element past the allocation (not 16-byte aligned)."""
    buf = torch.empty(t.numel() + 1, dtype=t.dtype, device=t.device)
    out = buf[1:].view(t.shape)
    out.copy_(t)
    return out


def bits(t):
    """The bits of a 4-byte tensor as int32, for bitwise comparisons that see -0.0 and NaN payloads."""
    return t.contiguous().view(torch.int32)


def _fp64(a):
    return a.detach().double().cpu().numpy() if isinstance(a, torch.Tensor) else np.asarray(a, np.float64)


def rel(got, want):
    """max |got - want| / max |want| in fp64, torch or numpy operands; 0 for an empty want."""
    got, want = _fp64(got), _fp64(want)
    if want.size == 0:
        return 0.0
    return float(np.abs(got - want).max() / max(np.abs(want).max(), 1e-30))


def row_err(got, ref, bound=None):
    """max |got - ref| / max(|ref|, the row's max |ref|, |bound|) in fp64; a 1-D ref (a bias gradient) is one row.
    bound: a tensor of ref's shape, e.g. the same sum over |terms|: a sum of terms that cancels is known in fp32 only
    to a few ulps of the sum of the magnitudes, whatever the order of summation."""
    got, ref = got.detach().double().cpu(), ref.detach().double().cpu()
    if ref.numel() == 0:
        return 0.0
    if ref.dim() == 1:
        ref, got = ref[None, :], got[None, :]
    scale = torch.maximum(ref.abs(), ref.abs().amax(dim=1, keepdim=True))
    if bound is not None:
        scale = torch.maximum(scale, bound.detach().double().cpu().abs())
    return float(((got - ref).abs() / scale.clamp_min(1e-30)).max())


def plan_structure(rp, ci, n_cols, dev, plan="default", chunk=256, seg_cost=None):
    """The CSRStructure of an int32 CSR under a plan form: "none" (no hub plan), "chunks" (hub chunks of `chunk`
    edges, no row segments) or "default" (hub chunks and the segments of seg_cost, the library's when None)."""
    from cogdl_b200.structure import CSRStructure

    chunk, seg_cost = {"none": (0, None), "chunks": (chunk, 0), "default": (chunk, seg_cost)}[plan]
    return CSRStructure(T(rp, dev), T(ci, dev), n_cols=n_cols, chunk_edges=chunk, seg_cost=seg_cost)


def check_counters(st, what):
    """A call on a structure with hub chunks leaves the plan's arrival counters back at zero."""
    if st.chunk_edges > 0 and st.plan.n_chunks > 0:
        assert int(st.plan.counters.abs().sum()) == 0, f"{what}: arrival counters not back at zero"

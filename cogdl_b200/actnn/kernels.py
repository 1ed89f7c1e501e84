"""Tensor-level wrappers of the actnn.cu entry points (include/cogdl_b200.h, "Activation-compressed training").
No autograd and no config here: outputs are allocated with torch, pointers and the current stream go to the C ABI."""
import numpy as np
import torch

from .. import _cabi
from ..structure import _ptr, _stream, require_cuda


def draw_seed():
    """A 64-bit seed from torch's CPU default generator (follows torch.manual_seed, no device synchronisation)."""
    lo, hi = torch.randint(0, 2 ** 32, (2,), dtype=torch.int64).tolist()
    return (hi << 32) | lo


def _f32_2d(x):
    require_cuda(x)
    if x.dtype != torch.float32:
        raise TypeError(f"actnn kernels take float32 activations, got {x.dtype}")
    return x.reshape(x.shape[0], int(np.prod(x.shape[1:]))).contiguous()


def padded_width(D, group_size):
    return -(-D // group_size) * group_size


def row_offsets(bits, Dp):
    """Exclusive prefix sum of bits * Dp / 8 (int64 byte offsets of the mixed-width rows) and the total bytes."""
    ends = torch.cumsum(bits.to(torch.int64), 0) * (Dp // 8)
    total = int(ends[-1].item()) if ends.numel() else 0
    return ends - bits.to(torch.int64) * (Dp // 8), total


def group_minmax(x, group_size):
    """(mn, mx) [N, G] fp32 of the zero-padded groups of x.view(N, -1)."""
    x = _f32_2d(x)
    N, D = x.shape
    G = padded_width(D, group_size) // group_size
    mn = torch.empty((N, G), dtype=torch.float32, device=x.device)
    mx = torch.empty_like(mn)
    with torch.cuda.device(x.device):
        _cabi.call("cogdl_b200_actnn_minmax_f32", _ptr(x), N, D, int(group_size), _ptr(mn), _ptr(mx),
                   _stream(x.device))
    return mn, mx


def _widths(bits, N, dev):
    """(bits tensor or None, uniform width) as the C ABI takes them."""
    if isinstance(bits, torch.Tensor):
        if bits.numel() != N or bits.device != dev:
            raise ValueError("bits must be an int32 tensor of N entries on the input's device")
        return bits.to(torch.int32).contiguous(), 0
    return None, int(bits)


def pack(x, bits, group_size, stochastic, seed=0):
    """Quantize x.view(N, -1) by groups and pack it: (packed uint8, scale bf16 [N, G], mn bf16 [N, G]).
    bits: an int (1, 2, 4, 8) or an int32 [N] tensor (1..8 per row)."""
    x = _f32_2d(x)
    N, D = x.shape
    Dp = padded_width(D, group_size)
    bt, ub = _widths(bits, N, x.device)
    if bt is None:
        offs, total = None, N * Dp * ub // 8
    else:
        if N and (int(bt.min()) < 1 or int(bt.max()) > 8):
            raise ValueError("per-row bit widths must be in 1..8")
        offs, total = row_offsets(bt, Dp)
    packed = torch.empty(total, dtype=torch.uint8, device=x.device)
    scale = torch.empty((N, Dp // group_size), dtype=torch.bfloat16, device=x.device)
    mn = torch.empty_like(scale)
    with torch.cuda.device(x.device):
        _cabi.call("cogdl_b200_actnn_pack_f32", _ptr(x), N, D, int(group_size), _ptr(bt), ub, _ptr(offs),
                   1 if stochastic else 0, int(seed) & (2 ** 64 - 1), _ptr(packed), _ptr(scale), _ptr(mn),
                   _stream(x.device))
    return packed, scale, mn


def unpack(packed, bits, scale, mn, N, D, group_size):
    """[N, D] fp32 from pack()'s output."""
    require_cuda(packed, scale, mn)
    Dp = padded_width(D, group_size)
    bt, ub = _widths(bits, N, packed.device)
    offs = None if bt is None else row_offsets(bt, Dp)[0]
    out = torch.empty((N, D), dtype=torch.float32, device=packed.device)
    with torch.cuda.device(packed.device):
        _cabi.call("cogdl_b200_actnn_unpack_f32", _ptr(packed), N, D, int(group_size), _ptr(bt), ub, _ptr(offs),
                   _ptr(scale.contiguous()), _ptr(mn.contiguous()), _ptr(out), _stream(packed.device))
    return out


def _mask_words(n, dev):
    return torch.empty((n + 31) // 32, dtype=torch.int32, device=dev)


def relu_fwd(x):
    """(relu(x), 1-bit mask of x > 0)."""
    require_cuda(x)
    if x.dtype != torch.float32:
        raise TypeError(f"QReLU takes float32 input, got {x.dtype}")
    x = x.contiguous()
    y, mask = torch.empty_like(x), _mask_words(x.numel(), x.device)
    with torch.cuda.device(x.device):
        _cabi.call("cogdl_b200_actnn_relu_fwd_f32", _ptr(x), x.numel(), _ptr(y), _ptr(mask), _stream(x.device))
    return y, mask


def relu_bwd(g, mask):
    g = g.contiguous()
    gx = torch.empty_like(g)
    with torch.cuda.device(g.device):
        _cabi.call("cogdl_b200_actnn_relu_bwd_f32", _ptr(g), _ptr(mask), g.numel(), _ptr(gx), _stream(g.device))
    return gx


def dropout_threshold(p):
    """drop_below = floor(p * 2^64) of the fp32 probability the kernels use (the reference passes p as a float)."""
    return int(float(np.float32(p)) * 2.0 ** 64)


def dropout_fwd(x, p, seed):
    """(x * keep / (1 - p), 1-bit keep mask); element i is kept iff draw(seed, i, 0) >= dropout_threshold(p)."""
    require_cuda(x)
    if x.dtype != torch.float32:
        raise TypeError(f"QDropout takes float32 input, got {x.dtype}")
    x = x.contiguous()
    y, mask = torch.empty_like(x), _mask_words(x.numel(), x.device)
    with torch.cuda.device(x.device):
        _cabi.call("cogdl_b200_actnn_dropout_fwd_f32", _ptr(x), x.numel(), float(p), int(seed) & (2 ** 64 - 1),
                   dropout_threshold(p), _ptr(y), _ptr(mask), _stream(x.device))
    return y, mask


def dropout_bwd(g, mask, p):
    g = g.contiguous()
    gx = torch.empty_like(g)
    with torch.cuda.device(g.device):
        _cabi.call("cogdl_b200_actnn_dropout_bwd_f32", _ptr(g), _ptr(mask), g.numel(), float(p), _ptr(gx),
                   _stream(g.device))
    return gx


def allocate_bits(C, target, initial_bits=8):
    """Per-row bit widths [N] int32 on C's device: the reference greedy calc_precision(b = initial_bits, C, w = 1,
    target) (calc_precision.cc:9-50), bit for bit, as a device top-K selection."""
    require_cuda(C)
    C = C.reshape(-1).to(torch.float32).contiguous()
    N = C.numel()
    bits = torch.empty(N, dtype=torch.int32, device=C.device)
    scratch = torch.empty(int(_cabi.load().cogdl_b200_actnn_bits_scratch_bytes(N)), dtype=torch.uint8,
                          device=C.device)
    with torch.cuda.device(C.device):
        _cabi.call("cogdl_b200_actnn_bits", _ptr(C), N, int(initial_bits), int(target), _ptr(bits), _ptr(scratch),
                   scratch.numel(), _stream(C.device))
    return bits

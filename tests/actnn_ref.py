"""numpy restatement of the actnn kernels (cogdl_b200/csrc/actnn.cu): quantize + pack, unpack + dequantize, the 1-bit
ReLU / dropout masks, the counter-based stochastic rounding and the top-K bit allocation, plus a heapq restatement of
the reference greedy (calc_precision.cc:9-50).  Every result is exact: fp32 steps are rounded one at a time."""
import heapq

import numpy as np

M64 = (1 << 64) - 1


def mix64(z):
    z = (z + np.uint64(0x9E3779B97F4A7C15))
    z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
    z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def draw(seed, i, k):
    """rng.cuh draw(seed, i, k), vectorised over i (uint64 wrap-around arithmetic)."""
    with np.errstate(over="ignore"):
        i = np.asarray(i, dtype=np.int64).astype(np.uint64)
        return mix64(mix64(np.uint64(seed) + i * np.uint64(0xD1342543DE82EF95)) + np.uint64(k))


def hashed_C(seed, n):
    """float32 [n]: (draw(seed, i, 0) >> 48) / 1024, multiples of 1/1024 in [0, 64) with many duplicates; a pure
    function of (seed, n), so fixtures store the seed instead of the values."""
    return ((draw(seed, np.arange(n), 0) >> np.uint64(48)).astype(np.float32) / np.float32(1024)).astype(np.float32)


def bf16(x):
    """fp32 -> bf16 (round to nearest even) -> fp32."""
    u = np.asarray(x, dtype=np.float32).view(np.uint32).astype(np.uint64)
    r = ((u + 0x7FFF + ((u >> 16) & 1)) >> 16) << 16
    return r.astype(np.uint32).view(np.float32)


def quantize(x, bits, group_size, stochastic=False, seed=0):
    """(codes int32 [N, Dp], scale fp32 [N, G] (bf16 values), mn fp32 [N, G] (bf16 values)).  bits: int or [N]."""
    x = np.asarray(x, dtype=np.float32)
    N, D = x.shape
    Dp = -(-D // group_size) * group_size
    xp = np.zeros((N, Dp), dtype=np.float32)
    xp[:, :D] = x
    groups = xp.reshape(N, Dp // group_size, group_size)
    if N == 0:
        z = np.zeros((0, Dp // group_size), np.float32)
        return np.zeros((0, Dp), np.int32), z, z
    mn, mx = groups.min(axis=2), groups.max(axis=2)
    b = np.broadcast_to(np.asarray(bits, dtype=np.int64), (N,))
    B = ((1 << b) - 1).astype(np.float32)[:, None]
    mnp = (mn - np.float32(1e-6)).astype(np.float32)
    mxp = (mx + np.float32(1e-6)).astype(np.float32)
    scale = (B / (mxp - mnp)).astype(np.float32)
    v = ((groups - mnp[:, :, None]).astype(np.float32) * scale[:, :, None]).astype(np.float32)
    if stochastic:
        u = (draw(seed, np.arange(N * Dp), 0) >> np.uint64(40)).astype(np.float32) * np.float32(2.0 ** -24)
        v = (v + (u - np.float32(0.5)).reshape(N, -1, group_size)).astype(np.float32)
    v = np.minimum(np.maximum(v, np.float32(0)), B[:, :, None])
    codes = np.rint(v).astype(np.int32).reshape(N, Dp)
    return codes, bf16(scale), bf16(mn)


def dequantize(codes, scale, mn, D, group_size):
    N, Dp = codes.shape
    c = codes.reshape(N, Dp // group_size, group_size).astype(np.float32)
    y = (c / scale[:, :, None]).astype(np.float32) + mn[:, :, None]
    return y.astype(np.float32).reshape(N, Dp)[:, :D]


def pack(codes, bits):
    """The packed bytes: row n is a bitstream of its codes at bits[n] bits each, LSB first, rows back to back."""
    N, Dp = codes.shape
    b = np.broadcast_to(np.asarray(bits, dtype=np.int64), (N,))
    rows = []
    for n in range(N):
        shifts = np.arange(b[n])
        bitstream = ((codes[n][:, None] >> shifts[None, :]) & 1).astype(np.uint8).reshape(-1)
        rows.append(np.packbits(bitstream, bitorder="little"))
    return np.concatenate(rows) if rows else np.zeros(0, dtype=np.uint8)


def unpack(packed, bits, N, Dp):
    b = np.broadcast_to(np.asarray(bits, dtype=np.int64), (N,))
    codes = np.zeros((N, Dp), dtype=np.int32)
    off = 0
    for n in range(N):
        nbytes = Dp * b[n] // 8
        bitstream = np.unpackbits(packed[off:off + nbytes], bitorder="little").reshape(Dp, b[n]).astype(np.int32)
        codes[n] = (bitstream << np.arange(b[n])[None, :]).sum(axis=1)
        off += nbytes
    return codes


def mask_words(bits):
    """Bool [n] -> int32 words, bit i % 32 of word i / 32 = element i."""
    bits = np.asarray(bits, dtype=bool)
    pad = np.zeros(-(-bits.size // 32) * 32, dtype=bool)
    pad[:bits.size] = bits
    return np.packbits(pad, bitorder="little").view(np.int32)


def relu(x):
    x = np.asarray(x, dtype=np.float32).reshape(-1)
    keep = x > 0
    return np.where(keep, x, np.float32(0)), mask_words(keep)


def dropout_keep(n, p, seed):
    drop_below = int(float(np.float32(p)) * 2.0 ** 64)
    return draw(seed, np.arange(n), 0) >= np.uint64(min(drop_below, M64))


def dropout(x, p, seed):
    x = np.asarray(x, dtype=np.float32).reshape(-1)
    keep = dropout_keep(x.size, p, seed)
    scaled = (x.astype(np.float64) / (1.0 - float(np.float32(p)))).astype(np.float32)
    return np.where(keep, scaled, np.float32(0)), mask_words(keep)


def _coef(b):
    b = np.asarray(b, dtype=np.int64)
    return 1.0 / ((1 << b) - 1) ** 2 - 1.0 / ((1 << (b - 1)) - 1) ** 2


def alloc_topk(C, target, b0=8):
    """Top-K restatement: K = b0 * N - target keys (float32(C_i * coef(b)), i, b) taken in descending order."""
    C = np.asarray(C, dtype=np.float32).astype(np.float64)
    N = C.size
    K = int(min(max(b0 * N - target, 0), (b0 - 1) * N))
    bb = np.tile(np.arange(b0, 1, -1), N)
    ii = np.repeat(np.arange(N), b0 - 1)
    key = (C[ii] * _coef(bb)).astype(np.float32).astype(np.float64) + 0.0   # -0.0 -> +0.0
    order = np.lexsort((-bb, -ii, -key))
    return (b0 - np.bincount(ii[order[:K]], minlength=N)).astype(np.int32)


def alloc_greedy(C, target, b0=8):
    """The reference greedy with w = 1, a heap of (float key, row) popped largest first."""
    C = np.asarray(C, dtype=np.float32)
    b = np.full(C.size, b0, dtype=np.int64)

    def key(i):
        return float(np.float32(float(C[i]) * _coef(b[i])))

    heap = [(-key(i), -i) for i in range(C.size)]
    heapq.heapify(heap)
    b_sum = b0 * C.size
    while b_sum > target and heap:   # the reference asserts a non-empty queue; every row at 1 bit ends it here
        _, ni = heapq.heappop(heap)
        b[-ni] -= 1
        b_sum -= 1
        if b[-ni] > 1:
            heapq.heappush(heap, (-key(-ni), ni))
    return b.astype(np.int32)

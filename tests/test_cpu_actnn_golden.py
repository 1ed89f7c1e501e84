"""The numpy restatement of the actnn kernels (tests/actnn_ref.py) against the reference's own actnn code
(tests/golden/actnn.npz, written by tests/golden/make_golden_actnn.py): bit allocation against calc_precision.cc,
codes and dequantized values against actnn's torch path.  Also: the top-K allocation equals a heapq restatement of the
greedy, pack / unpack round-trip, the counter-based rounding noise, the masks, and the host allocate_perlayer
greedy of cogdl_b200.actnn against the heap."""
import os

import numpy as np
import pytest
import torch

from tests import actnn_ref as R

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "actnn.npz")
ALLOC_CASES = ("random", "zeros", "dups", "frac", "allzero", "large", "arxiv")
Q_CASES = ("u2_g256", "u4_g64", "u8_g64", "u1_g256", "mixed_g64", "mixed_g256")


@pytest.fixture(scope="module")
def gold():
    return np.load(GOLD)


def alloc_case(gold, name):
    if f"alloc_{name}_C" in gold:
        C = gold[f"alloc_{name}_C"]
    else:
        seed, n = (int(v) for v in gold[f"alloc_{name}_hash"])
        C = R.hashed_C(seed, n)
    bits = float(gold[f"alloc_{name}_target"][0])
    return C.astype(np.float32), int(bits * C.size), gold[f"alloc_{name}_bits"].astype(np.int32)


@pytest.mark.parametrize("name", ALLOC_CASES)
def test_topk_allocation_matches_reference_calc_precision(gold, name):
    C, target, want = alloc_case(gold, name)
    got = R.alloc_topk(C, target)
    assert np.array_equal(got, want)
    assert got.sum() <= target or np.all(got == 1)


@pytest.mark.parametrize("seed", range(6))
def test_topk_allocation_matches_heap_greedy(seed):
    rng = np.random.default_rng(seed)
    N = int(rng.integers(1, 400))
    C = rng.random(N).astype(np.float32) * rng.choice([1e-30, 1.0, 1e20])
    C[rng.random(N) < 0.2] = 0
    C[rng.random(N) < 0.2] = C[0]
    for target in (0, N, int(2.5 * N), 5 * N, 8 * N, 9 * N):
        for b0 in (8, 4):
            assert np.array_equal(R.alloc_topk(C, target, b0), R.alloc_greedy(C, target, b0)), (N, target, b0)


@pytest.mark.parametrize("name", Q_CASES)
def test_codes_and_dequantized_values_match_reference_torch_path(gold, name):
    x, bits = gold[f"q_{name}_x"], gold[f"q_{name}_bits"]
    gs = int(name.rsplit("_g", 1)[1])
    codes, scale, mn = R.quantize(x, bits, gs)
    assert np.array_equal(codes, gold[f"q_{name}_codes"])
    assert np.array_equal(scale, gold[f"q_{name}_scale"])
    assert np.array_equal(mn, gold[f"q_{name}_mn"])
    deq = R.dequantize(codes, scale, mn, x.shape[1], gs)
    assert np.array_equal(deq, gold[f"q_{name}_deq"])


@pytest.mark.parametrize("name", Q_CASES)
def test_pack_unpack_round_trip(gold, name):
    x, bits = gold[f"q_{name}_x"], gold[f"q_{name}_bits"]
    gs = int(name.rsplit("_g", 1)[1])
    codes = R.quantize(x, bits, gs)[0]
    packed = R.pack(codes, bits)
    assert packed.size == int(np.sum(bits)) * codes.shape[1] // 8
    assert np.array_equal(R.unpack(packed, bits, *codes.shape), codes)


def test_stochastic_rounding_is_seeded_and_unbiased():
    rng = np.random.default_rng(3)
    x = rng.standard_normal((64, 256)).astype(np.float32)
    det = R.quantize(x, 2, 256)
    a = R.quantize(x, 2, 256, stochastic=True, seed=11)
    b = R.quantize(x, 2, 256, stochastic=True, seed=11)
    c = R.quantize(x, 2, 256, stochastic=True, seed=12)
    assert np.array_equal(a[0], b[0]) and not np.array_equal(a[0], c[0])
    assert np.array_equal(a[1], det[1]) and np.array_equal(a[2], det[2])
    assert np.abs(a[0] - det[0]).max() <= 1
    errs = [R.dequantize(R.quantize(x, 2, 256, True, s)[0], det[1], det[2], 256, 256) - x for s in range(64)]
    one = np.abs(errs[0]).mean()
    assert np.abs(np.mean(errs, axis=0)).mean() <= one / 4


def test_noise_draw_matches_library_generator():
    from cogdl_b200 import _cabi

    lib = _cabi.load()
    for seed, i in ((0, 0), (11, 5), (2 ** 63 + 7, 123456789)):
        assert int(R.draw(seed, [i], 0)[0]) == int(lib.cogdl_b200_sample_draw(seed, i, 0))


def test_masks():
    rng = np.random.default_rng(5)
    x = rng.standard_normal(1000).astype(np.float32)
    y, m = R.relu(x)
    assert m.size == 32 and np.array_equal(np.unpackbits(m.view(np.uint8), bitorder="little")[:1000], x > 0)
    assert np.array_equal(y, np.maximum(x, 0))
    keep = R.dropout_keep(200000, 0.3, 9)
    assert abs(keep.mean() - 0.7) < 6 * np.sqrt(0.21 / 200000)
    yd, md = R.dropout(x, 0.5, 9)
    assert np.array_equal(yd != 0, R.dropout_keep(1000, 0.5, 9) & (x != 0))
    assert np.array_equal(yd[yd != 0], (x[yd != 0] * 2).astype(np.float32))


@pytest.mark.parametrize("seed", range(3))
def test_host_allocate_perlayer_greedy_matches_heap(seed):
    """calc_precision_host (allocate_perlayer's greedy, weighted) against a heap restatement with weights."""
    import heapq

    from cogdl_b200.actnn.qscheme import calc_precision_host

    rng = np.random.default_rng(seed)
    N = 300
    C = (rng.random(N) * rng.choice([0, 1, 1, 5], N)).astype(np.float32)
    w = rng.choice([16, 64, 256], N).astype(np.int32)
    b0 = np.full(N, 8, dtype=np.int32)
    target = float(w.sum() * 2)
    got = calc_precision_host(torch.from_numpy(b0.copy()), torch.from_numpy(C), torch.from_numpy(w), target).numpy()
    b = b0.astype(np.int64)

    def key(i):
        return float(np.float32(float(C[i]) * R._coef(b[i]) / int(w[i])))

    heap = [(-key(i), -i) for i in range(N)]
    heapq.heapify(heap)
    b_sum = float((b * w).sum())
    while b_sum > target:
        _, ni = heapq.heappop(heap)
        b[-ni] -= 1
        b_sum -= int(w[-ni])
        if b[-ni] > 1:
            heapq.heappush(heap, (-key(-ni), ni))
    assert np.array_equal(got, b)
